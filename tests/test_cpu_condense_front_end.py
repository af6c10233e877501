"""The condensation has one front end: jac_gram in hb_lowrank.cu is the only caller of the int8 Gram kernels, the condensation modes are
known to hb_lowrank.cu / hb_lowrank.cuh alone, the two int8 schemes share one host driver (one cuTensorMapEncodeTiled lookup), and one
helper brackets every Gram kernel with the timing events. A new Gram kernel or scheme then touches one dispatch and one driver."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hiop_b200", "csrc")
LOWRANK = {"hb_lowrank.cu", "hb_lowrank.cuh"}


def _code(path):
    """source without comments and string literals (line structure kept)"""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    return re.sub(r'"(\\.|[^"\\\n])*"', '""', src)


def _scan(pattern):
    """(file, enclosing top-level definition) of every match on an indented line; definitions start in column 0"""
    rx = re.compile(pattern)
    found = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        owner = None
        for line in _code(path).splitlines():
            if line[:1].isalpha() or line[:1] in "_~":
                m = re.search(r"([\w:~]+)\s*\(", line)
                owner = m.group(1) if m else None
                continue
            found += [(os.path.basename(path), owner)] * len(rx.findall(line))
    return found


def test_one_function_calls_the_int8_gram_kernels():
    calls = _scan(r"\bhb_syrk_rows_(?:ozaki|crt)\s*\(")
    assert len(calls) == 2, calls  # the scan sees the two calls (a scan that finds nothing proves nothing)
    assert set(calls) == {("hb_lowrank.cu", "jac_gram")}, calls


def test_only_hb_lowrank_knows_the_condensation_modes():
    for name in ("condense_mode", "HB_CONDENSE_INT8_CRT"):
        files = {os.path.basename(p) for p in glob.glob(os.path.join(CSRC, "*.cu*")) if re.search(rf"\b{name}\b", _code(p))}
        assert files and files <= LOWRANK, (name, files)


def test_one_tensor_map_encoder_lookup():
    assert len(_scan(r"\bcudaGetDriverEntryPoint\s*\(")) == 1


def test_one_timing_bracket():
    assert len(_scan(r"\bcudaEventRecord\s*\([^;]*\bev_syrk0\b")) == 1

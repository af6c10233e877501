"""Every inline PTX instruction of the library and of the probes in tools/ is written once, in hb_ptx.cuh: no other kernel source or
probe contains an asm statement, so the memory-ordering contract of each primitive is stated and kept in one place."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "hiop_b200", "csrc", "hb_ptx.cuh")
ASM = re.compile(r"\basm\s*(volatile\s*)?\(")


def _code(path):
    """source without comments and string literals (line structure kept)"""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    return re.sub(r'"(\\.|[^"\\\n])*"', '""', src)


def _asm_statements():
    """(file, line) of every asm statement of the library's CUDA sources and the CUDA probes"""
    paths = glob.glob(os.path.join(ROOT, "hiop_b200", "csrc", "*.cu")) + glob.glob(os.path.join(ROOT, "hiop_b200", "csrc", "*.cuh"))
    paths += glob.glob(os.path.join(ROOT, "tools", "*.cu"))
    found = []
    for path in sorted(paths):
        for n, line in enumerate(_code(path).splitlines(), 1):
            if ASM.search(line):
                found.append((os.path.relpath(path, ROOT), n))
    return found


def test_inline_ptx_lives_only_in_hb_ptx():
    found = _asm_statements()
    stray = [f for f in found if f[0] != os.path.relpath(HEADER, ROOT)]
    assert not stray, f"call a primitive of hb_ptx.cuh (or add one there) instead of writing asm: {stray}"
    # the scan sees the statements it allows (a scan that finds nothing proves nothing)
    assert len(found) > 20, found


def test_the_wgmma_header_is_folded_in():
    assert not os.path.exists(os.path.join(ROOT, "hiop_b200", "csrc", "hb_wgmma.cuh"))

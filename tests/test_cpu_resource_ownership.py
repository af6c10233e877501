"""Every device buffer, pinned buffer, stream and event of the engine is held by the owner types of hb_common.cuh: outside their
implementation and the four public hb_malloc / hb_free / hb_malloc_host / hb_free_host entry points (whose memory belongs to the
caller), no source file of the library allocates, frees, creates or destroys one itself."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hiop_b200", "csrc")
RAW = re.compile(r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|cudaEventDestroy)\s*\(")
# the functions allowed to call them: the owners' implementation (hb_api.cu) and the caller-owned public allocation entry points
OWNERS = {"hb_mem_alloc", "hb_mem_free", "create_handle", "destroy_handle"}
PUBLIC = {"hb_malloc", "hb_free", "hb_malloc_host", "hb_free_host"}


def _code(path):
    """source without comments and string literals (line structure kept)"""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    return re.sub(r'"(\\.|[^"\\\n])*"', '""', src)


def _raw_calls():
    """(file, enclosing top-level definition, call) of every raw call; definitions start in column 0, their bodies are indented"""
    found = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        owner = None
        for line in _code(path).splitlines():
            if line[:1].isalpha() or line[:1] in "_~":
                m = re.search(r"([\w:~]+)\s*\(", line)
                owner = m.group(1) if m else None
            for call in RAW.findall(line):
                found.append((os.path.basename(path), owner, call))
    return found


def test_only_the_owner_types_manage_device_resources():
    calls = _raw_calls()
    stray = [c for c in calls if not (c[0] == "hb_api.cu" and c[1] in OWNERS | PUBLIC)]
    assert not stray, f"allocate / free / create / destroy through an owner type of hb_common.cuh instead: {stray}"
    # the scan sees the calls it allows (a scan that finds nothing proves nothing)
    assert {c[1] for c in calls} == OWNERS | PUBLIC

"""Every device and pinned host allocation of the library goes through the one owning buffer type (csrc/dev_buffer.h): no
other source under csrc/ calls a CUDA allocation or free function, so no buffer is freed by hand or left out of a free list."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vainplex_openclaw_b200", "csrc")
OWNER = "dev_buffer.h"
ALLOC = re.compile(r"\bcuda(?:Malloc|Free|HostAlloc)\w*")


def strip_comments(src):
    return re.sub(r"//[^\n]*|/\*.*?\*/", "", src, flags=re.S)


def test_only_the_owner_header_allocates_or_frees():
    found = {}
    for name in sorted(os.listdir(CSRC)):
        path = os.path.join(CSRC, name)
        if name == OWNER or not os.path.isfile(path):
            continue
        calls = ALLOC.findall(strip_comments(open(path, encoding="utf-8").read()))
        if calls:
            found[name] = sorted(set(calls))
    assert not found, "CUDA allocation / free calls outside %s: %r" % (OWNER, found)


def test_the_owner_header_is_a_build_dependency():
    from vainplex_openclaw_b200 import _build
    assert OWNER in _build.HEADERS
    src = strip_comments(open(os.path.join(CSRC, OWNER), encoding="utf-8").read())
    for fn in ("cudaMalloc", "cudaMallocHost", "cudaFree", "cudaFreeHost"):
        assert re.search(r"\b%s\(" % fn, src), fn

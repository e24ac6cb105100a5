"""CPU-side checks of lwf_batcher_add_headers: the library exports it, the header declares it with the argument types the
ctypes mirror uses, and it refuses NULL arguments and (on a VQ batcher) headers that do not qualify for LWB_ENTRY_VQ before
it reads the context or the setup (no device needed)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import vorbis_packer as vp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import build
    from lewton_b200 import frontend as fe
    build.build()
    return fe.lib()


def headers(seed, channels):
    from lewton_b200 import frontend as fe
    spec = vp.StreamSpec(np.random.default_rng(seed), channels=channels)
    return fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())


def test_add_headers_exported_and_declared(lib):
    from lewton_b200 import _cabi
    from lewton_b200 import frontend as fe
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lewton_frontend.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+lwf_batcher_add_headers\s*\(([^)]*)\)", hdr)
    assert m, "lwf_batcher_add_headers not declared in the header"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert params == ["lwf_batcher *b", "const lwf_headers *h", "const lwb_setup *setup"], params
    nm = subprocess.run(["nm", "-D", "--defined-only", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert "lwf_batcher_add_headers" in re.findall(r" T (lwf_[a-z0-9_]+)", nm)
    assert "lwf_batcher_add_headers" in fe.SYMBOLS
    f = lib.lwf_batcher_add_headers
    assert f.restype is C.c_int
    assert f.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p]


def test_add_headers_refuses_null_arguments_and_non_vq_headers(lib):
    """LWB_ERR_INVALID for a NULL batcher, headers or setup, and on an LWB_ENTRY_VQ batcher for 10-channel headers
    (lwf_headers_vq_capable takes at most 8).  The batcher is made on a stand-in context and the setup is a stand-in
    pointer: these refusals come before anything reads either.  set_entry(VQ) still succeeds afterwards: the refused set
    was not added."""
    from lewton_b200 import _cabi as cabi
    two, ten = headers(7, 2), headers(8, 10)
    assert two.vq_capable() and not ten.vq_capable()
    stand_in = C.create_string_buffer(64)
    b = C.c_void_p()
    assert lib.lwf_batcher_create(C.addressof(stand_in), two._h, 1, C.byref(b)) == 0
    try:
        su = C.addressof(stand_in)
        assert lib.lwf_batcher_add_headers(None, two._h, su) == cabi.ERR_INVALID
        assert lib.lwf_batcher_add_headers(b, None, su) == cabi.ERR_INVALID
        assert lib.lwf_batcher_add_headers(b, two._h, None) == cabi.ERR_INVALID
        assert lib.lwf_batcher_set_entry(b, cabi.ENTRY_VQ) == 0
        assert lib.lwf_batcher_add_headers(b, ten._h, su) == cabi.ERR_INVALID
        assert lib.lwf_batcher_set_entry(b, cabi.ENTRY_VQ) == 0
    finally:
        lib.lwf_batcher_destroy(b)
    assert lib.lwf_batcher_add_headers(None, None, None) == cabi.ERR_INVALID

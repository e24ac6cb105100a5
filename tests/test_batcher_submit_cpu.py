"""CPU-side checks of lwf_batcher_submit: the library exports it, the header declares it with the argument types the ctypes
mirror uses, and it refuses NULL handles and bad arguments before it touches the context (no device needed)."""
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


def test_submit_exported_and_declared(lib):
    from lewton_b200 import _cabi
    from lewton_b200 import frontend as fe
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lewton_frontend.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+lwf_batcher_submit\s*\(([^)]*)\)", hdr)
    assert m, "lwf_batcher_submit not declared in the header"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert params == ["lwf_batcher *b", "lwf_stream_job *jobs", "size_t n_jobs", "int out_format", "void *pcm", "int pcm_memory",
                      "uint64_t *ticket"], params
    nm = subprocess.run(["nm", "-D", "--defined-only", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert "lwf_batcher_submit" in re.findall(r" T (lwf_[a-z0-9_]+)", nm)
    assert "lwf_batcher_submit" in fe.SYMBOLS
    f = lib.lwf_batcher_submit
    assert f.restype is C.c_int
    assert f.argtypes == [C.c_void_p, C.POINTER(fe._StreamJob), C.c_size_t, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]


def test_submit_refuses_null_handles_and_bad_arguments(lib):
    """LWB_ERR_INVALID for a NULL batcher, jobs, pcm or ticket, an unknown memory space and a job without a stream or
    packet arrays.  The batcher is made on a stand-in context pointer: these refusals come before anything reads it,
    and a batcher that never submitted frees nothing on the device."""
    from lewton_b200 import frontend as fe
    spec = vp.StreamSpec(np.random.default_rng(7))
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    stand_in = C.create_string_buffer(64)
    b = C.c_void_p()
    assert lib.lwf_batcher_create(C.addressof(stand_in), hdr._h, 1, C.byref(b)) == 0
    try:
        pk = (C.c_char_p * 1)(b"\x00\x00")
        ln = (C.c_size_t * 1)(2)
        jobs = (fe._StreamJob * 1)()
        jobs[0].stream, jobs[0].n_packets, jobs[0].packets, jobs[0].lengths = C.addressof(stand_in), 1, pk, ln
        jobs[0].n_samples, jobs[0].packets_done, jobs[0].status = 77, 88, 99
        pcm = np.zeros(64, np.float32)
        t = C.c_uint64(5)
        ok = dict(b=b, jobs=jobs, n=1, fmt=0, pcm=pcm.ctypes.data, mem=0, t=C.byref(t))

        def submit(**kw):
            a = dict(ok, **kw)
            return lib.lwf_batcher_submit(a["b"], a["jobs"], a["n"], a["fmt"], a["pcm"], a["mem"], a["t"])

        assert submit(b=None) == 4
        assert submit(jobs=None) == 4
        assert submit(jobs=None, n=0, pcm=None) == 4
        assert submit(pcm=None) == 4
        assert submit(t=None) == 4
        for mem in (-1, 2, 7):
            assert submit(mem=mem) == 4
        jobs[0].stream = None
        assert submit() == 4
        jobs[0].stream = C.addressof(stand_in)
        jobs[0].packets = None
        assert submit() == 4
        assert (jobs[0].n_samples, jobs[0].packets_done, jobs[0].status) == (77, 88, 99)
        assert t.value == 5 and not pcm.any()
    finally:
        lib.lwf_batcher_destroy(b)
    assert lib.lwf_batcher_submit(None, None, 0, 0, None, 0, None) == 4

"""CPU-side checks of lwf_readers (include/lewton_frontend.h): the library exports the new calls, the ctypes mirror of
lwf_read_job has the C compiler's layout, readers share one set of headers per distinct (ident, setup) byte pair, and
lwf_readers_read refuses bad arguments before it changes a job or a reader.  No device is needed: the readers object is
made on a stand-in context pointer, which it only reads when a read makes a reader's device setup -- and every read here
is refused before that."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import vorbis_packer as vp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 4
READERS = ["lwf_readers_create", "lwf_readers_destroy", "lwf_readers_add", "lwf_readers_headers", "lwf_readers_last_absgp",
           "lwf_readers_setup_count", "lwf_readers_last_timing", "lwf_readers_read"]


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import build
    from lewton_b200 import frontend as fe
    build.build()
    return fe.lib()


def _file(seed, channels=2, bs0=8, bs1=11, comments=None, setup_tail=b"", n_packets=4):
    """An Ogg Vorbis file of the packer: headers, then n_packets long audio packets, 2 per page."""
    spec = vp.StreamSpec(np.random.default_rng(seed), channels=channels, bs0=bs0, bs1=bs1)
    if comments is not None:
        spec.comments = comments
    long_mode = [i for i, (bf, _) in enumerate(spec.modes) if bf][0]
    packets = [spec.audio_packet(long_mode)[0] for _ in range(n_packets)]
    pages = (n_packets + 1) // 2
    return vp.ogg_stream(7, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet() + setup_tail], packets,
                         [1024 * (k + 1) for k in range(pages)], packets_per_page=2)


def test_readers_exported_and_declared(lib):
    from lewton_b200 import _cabi
    from lewton_b200 import frontend as fe
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lewton_frontend.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(lwf_readers_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(READERS), declared ^ set(READERS)
    m = re.search(r"\bint\s+lwf_readers_read\s*\(([^)]*)\)", hdr)
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert params == ["lwf_readers *rs", "lwf_read_job *jobs", "size_t n_jobs", "int out_format", "void *pcm", "int pcm_memory",
                      "uint64_t *ticket"], params
    nm = subprocess.run(["nm", "-D", "--defined-only", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert set(READERS) <= set(re.findall(r" T (lwf_[a-z0-9_]+)", nm))
    assert set(READERS) <= set(fe.SYMBOLS)
    assert lib.lwf_readers_read.argtypes == [C.c_void_p, C.POINTER(fe._ReadJob), C.c_size_t, C.c_int, C.c_void_p, C.c_int,
                                             C.POINTER(C.c_uint64)]


def test_read_job_layout(lib, tmp_path):
    """sizeof(lwf_read_job) and the offset of every field, as gcc lays them out, equal the ctypes mirror's."""
    from lewton_b200 import frontend as fe
    fields = [f for f, _ in fe._ReadJob._fields_]
    src = tmp_path / "rj.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lewton_frontend.h"\nint main(void){printf("%zu", '
                   'sizeof(lwf_read_job));' + "".join('printf(" %%zu", offsetof(lwf_read_job, %s));' % f for f in fields) +
                   'return 0;}\n')
    exe = tmp_path / "rj"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(fe._ReadJob)] + [getattr(fe._ReadJob, f).offset for f in fields]


@pytest.fixture
def readers(lib):
    stand_in = C.create_string_buffer(4096)
    rs = C.c_void_p()
    assert lib.lwf_readers_create(C.addressof(stand_in), 1, C.byref(rs)) == 0
    keep = []

    def add(data):
        keep.append(data)
        i = C.c_uint32(99)
        rc = lib.lwf_readers_add(rs, data, len(data), C.byref(i))
        return rc, i.value
    yield rs, add
    lib.lwf_readers_destroy(rs)


def _comments(lib, rs, i):
    from lewton_b200 import frontend as fe
    h = fe.Headers(None, None, None, _handle=lib.lwf_readers_headers(rs, i))
    return h.vendor, h.comment_list


def test_equal_header_bytes_share_one_setup(lib, readers):
    """Two files whose ident and setup headers are byte-equal but whose comments differ make one shared set of headers;
    each reader keeps its own comments.  A setup header with one byte more (past its framing bit, so it parses the same)
    makes a second one, and so does another channel count."""
    rs, add = readers
    assert lib.lwf_readers_setup_count(rs) == 0
    assert add(_file(5, comments=[("TITLE", "a")])) == (0, 0)
    assert add(_file(5, comments=[("TITLE", "b"), ("ALBUM", "c")])) == (0, 1)
    assert lib.lwf_readers_setup_count(rs) == 1
    assert _comments(lib, rs, 0)[1] == [("TITLE", "a")]
    assert _comments(lib, rs, 1)[1] == [("TITLE", "b"), ("ALBUM", "c")]
    assert lib.lwf_readers_headers(rs, 0) != lib.lwf_readers_headers(rs, 1)
    # each reader's headers hold its comments and give the shared setup's info and packet decode
    from lewton_b200 import frontend as fe
    spec = vp.StreamSpec(np.random.default_rng(5))
    full = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    for i in range(2):
        light = fe.Headers(None, None, None, _handle=lib.lwf_readers_headers(rs, i))
        assert [getattr(light.info, f) for f, _ in fe.Info._fields_ if f != "n_comments"] == \
            [getattr(full.info, f) for f, _ in fe.Info._fields_ if f != "n_comments"]
        assert light.n_comments == (1, 2)[i]
        long_mode = [m for m, (bf, _) in enumerate(spec.modes) if bf][0]
        pk = spec.audio_packet(long_mode)[0]
        a, b = light.decode_packet(pk), full.decode_packet(pk)
        assert a.mode_number == b.mode_number and np.array_equal(a.residue.view(np.uint32), b.residue.view(np.uint32))
        assert light.decoded_sample_count(pk) == full.decoded_sample_count(pk)
    assert add(_file(5, setup_tail=b"\x00")) == (0, 2)
    assert lib.lwf_readers_setup_count(rs) == 2
    assert add(_file(5, comments=[])) == (0, 3)
    assert lib.lwf_readers_setup_count(rs) == 2
    assert add(_file(6, channels=1)) == (0, 4)
    assert lib.lwf_readers_setup_count(rs) == 3
    # a file that is not Ogg Vorbis adds no reader and no set
    rc, _ = add(b"OggS" + bytes(40))
    assert rc != 0
    assert lib.lwf_readers_setup_count(rs) == 3 and not lib.lwf_readers_headers(rs, 5)


def test_add_and_queries_refuse_null_and_unknown(lib, readers):
    rs, add = readers
    i = C.c_uint32()
    v = C.c_uint64(123)
    data = _file(9)
    assert lib.lwf_readers_add(None, data, len(data), C.byref(i)) == INVALID
    assert lib.lwf_readers_add(rs, None, 10, C.byref(i)) == INVALID
    assert lib.lwf_readers_add(rs, data, len(data), None) == INVALID
    assert lib.lwf_readers_create(None, 1, C.byref(C.c_void_p())) == INVALID
    assert add(data) == (0, 0)
    assert lib.lwf_readers_last_absgp(rs, 0, C.byref(v)) == 1 and v.value == 123     # None before the first packet
    assert lib.lwf_readers_last_absgp(rs, 1, C.byref(v)) == INVALID
    assert lib.lwf_readers_last_absgp(None, 0, C.byref(v)) == INVALID
    assert lib.lwf_readers_last_absgp(rs, 0, None) == INVALID
    assert not lib.lwf_readers_headers(rs, 1) and not lib.lwf_readers_headers(None, 0)
    assert lib.lwf_readers_setup_count(None) == 0


def test_read_refusals_change_nothing(lib, readers):
    """LWB_ERR_INVALID for a NULL readers, jobs, pcm or ticket, a memory space other than host and device, an unknown
    out_format, an unknown reader index, a reader in two jobs and a planar out_stride below what max_packets packets can
    return (max_packets * blocksize_1 / 2, and (blocksize_1 - blocksize_0) / 4 more for a long block before a short one);
    the jobs' results, the readers' absgp and headers and the PCM stay as they were, and no ticket is issued."""
    from lewton_b200 import frontend as fe
    rs, add = readers
    assert add(_file(11)) == (0, 0)
    assert add(_file(12, channels=6, bs0=9, bs1=12)) == (0, 1)
    heads = [lib.lwf_readers_headers(rs, i) for i in range(2)]
    jobs = (fe._ReadJob * 2)()
    counts = np.full(8, 77, np.uint32)
    need = [4 * 1024 + (2048 - 256) // 4, 4 * 2048 + (4096 - 512) // 4]
    for k, (r, stride) in enumerate(zip((0, 1), need)):
        jobs[k].reader, jobs[k].max_packets, jobs[k].out_offset, jobs[k].out_stride = r, 4, k * 100000, stride
        jobs[k].packet_samples = counts.ctypes.data_as(C.POINTER(C.c_uint32))
        jobs[k].n_packets, jobs[k].n_samples, jobs[k].channels, jobs[k].status = 55, 66, 9, 88
        jobs[k].next_chained, jobs[k].ended = 3, 3
    pcm = np.zeros(64, np.float32)
    t = C.c_uint64(5)
    ok = dict(rs=rs, jobs=jobs, n=2, fmt=0, pcm=pcm.ctypes.data, mem=0, t=C.byref(t))

    def read(**kw):
        a = dict(ok, **kw)
        return lib.lwf_readers_read(a["rs"], a["jobs"], a["n"], a["fmt"], a["pcm"], a["mem"], a["t"])

    assert read(rs=None) == INVALID
    assert read(jobs=None) == INVALID
    assert read(n=0) == INVALID                                 # an empty call is refused, whatever was read before
    assert read(pcm=None) == INVALID
    assert read(t=None) == INVALID
    for mem in (-1, 2, 7):
        assert read(mem=mem) == INVALID
    for fmt in (-1, 6, 100):
        assert read(fmt=fmt) == INVALID
    jobs[1].reader = 2
    assert read() == INVALID                                    # unknown index
    jobs[1].reader = 0
    assert read() == INVALID                                    # a reader in two jobs
    jobs[1].reader = 1
    for k in range(2):
        for short in (1, need[k] - 4 * (1024 << k)):            # below the most 4 packets return, and below 4 halves
            jobs[k].out_stride = need[k] - short
            for fmt in (0, 1, 4):                               # planar only: interleaved output has no planes
                assert read(fmt=fmt) == INVALID
        jobs[k].out_stride = need[k]
    for k in range(2):
        assert (jobs[k].n_packets, jobs[k].n_samples, jobs[k].channels, jobs[k].status) == (55, 66, 9, 88)
        assert (jobs[k].next_chained, jobs[k].ended) == (3, 3)
    assert (counts == 77).all() and not pcm.any() and t.value == 5
    v = C.c_uint64()
    assert all(lib.lwf_readers_last_absgp(rs, i, C.byref(v)) == 1 for i in range(2))
    assert [lib.lwf_readers_headers(rs, i) for i in range(2)] == heads

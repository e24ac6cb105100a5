"""CPU-side checks of lwf_readers_seek_absgp_pg and lwf_readers_skip_samples_linear (include/lewton_frontend.h): the
library exports and declares them, the ctypes mirror of lwf_skip_job has the C compiler's layout, every refusal of
either call changes nothing, and seeks of readers whose device stream does not exist yet complete without touching the
context.  No device is needed: the readers object is made on a stand-in context pointer, which it only reads when a
call makes a reader's device setup or stream -- seeks never do, and every skip here is refused before that."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import vorbis_packer as vp
from test_ogg_readers_cpu import INVALID, ROOT, _file

OGG = 24
NEW = ["lwf_readers_seek_absgp_pg", "lwf_readers_skip_samples_linear"]


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import build
    from lewton_b200 import frontend as fe
    build.build()
    return fe.lib()


@pytest.fixture
def readers(lib):
    stand_in = C.create_string_buffer(4096)        # not a context: any use of it would be a fault, not a refusal
    rs = C.c_void_p()
    assert lib.lwf_readers_create(C.addressof(stand_in), 2, C.byref(rs)) == 0
    keep = []

    def add(data):
        keep.append(data)
        i = C.c_uint32(99)
        assert lib.lwf_readers_add(rs, data, len(data), C.byref(i)) == 0
        return i.value
    yield rs, add
    lib.lwf_readers_destroy(rs)


def _stream(seed, serial, channels=2, bs0=8, bs1=11, n_packets=4):
    """_file's stream under another serial"""
    spec = vp.StreamSpec(np.random.default_rng(seed), channels=channels, bs0=bs0, bs1=bs1)
    long_mode = [i for i, (bf, _) in enumerate(spec.modes) if bf][0]
    packets = [spec.audio_packet(long_mode)[0] for _ in range(n_packets)]
    return vp.ogg_stream(serial, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets,
                         [1024 * (k + 1) for k in range((n_packets + 1) // 2)], packets_per_page=2)


def _chained():
    """A stereo 256/2048 stream of 4 packets, then a six-channel 512/4096 one: a skip past the first enters the second."""
    return _stream(21, 7) + _stream(22, 8, channels=6, bs0=9, bs1=12)


def _serials(data):
    out, at = [], 0
    while at < len(data):
        out.append(int.from_bytes(data[at + 14: at + 18], "little"))
        at += 27 + data[at + 26] + sum(data[at + 27: at + 27 + data[at + 26]])
    return out


def test_seek_and_skip_exported_and_declared(lib):
    from lewton_b200 import _cabi
    from lewton_b200 import frontend as fe
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lewton_frontend.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(lwf_readers_[a-z0-9_]+)\)?\s*\(", hdr))
    assert set(NEW) <= declared
    m = re.search(r"\bint\s+\(lwf_readers_seek_absgp_pg\)\s*\(([^)]*)\)", hdr)
    assert [" ".join(p.split()) for p in m.group(1).split(",")] == [
        "lwf_readers *rs", "const uint32_t *readers", "const uint64_t *absgps", "size_t n", "int32_t *status"]
    m = re.search(r"\bint\s+\(lwf_readers_skip_samples_linear\)\s*\(([^)]*)\)", hdr)
    assert [" ".join(p.split()) for p in m.group(1).split(",")] == [
        "lwf_readers *rs", "lwf_skip_job *jobs", "size_t n_jobs", "int out_format", "void *pcm", "int pcm_memory",
        "uint64_t *ticket"]
    nm = subprocess.run(["nm", "-D", "--defined-only", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert set(NEW) <= set(re.findall(r" T (lwf_[a-z0-9_]+)", nm))
    assert lib.lwf_readers_skip_samples_linear.argtypes == [C.c_void_p, C.POINTER(fe._SkipJob), C.c_size_t, C.c_int,
                                                            C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]


def test_skip_job_layout(lib, tmp_path):
    """sizeof(lwf_skip_job) and the offset of every field, as gcc lays them out, equal the ctypes mirror's."""
    from lewton_b200 import frontend as fe
    fields = [f for f, _ in fe._SkipJob._fields_]
    src = tmp_path / "sj.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lewton_frontend.h"\nint main(void){printf("%zu", '
                   'sizeof(lwf_skip_job));' + "".join('printf(" %%zu", offsetof(lwf_skip_job, %s));' % f for f in fields) +
                   'return 0;}\n')
    exe = tmp_path / "sj"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(fe._SkipJob)] + [getattr(fe._SkipJob, f).offset for f in fields]


def _seek(lib, rs, readers, absgps, status, n=None):
    n = len(readers or absgps) if n is None else n
    r = (C.c_uint32 * max(1, len(readers)))(*readers) if readers is not None else None
    g = (C.c_uint64 * max(1, len(absgps)))(*absgps) if absgps is not None else None
    return lib.lwf_readers_seek_absgp_pg(rs, r, g, n, status)


def test_seeks_complete_on_the_host(lib, readers):
    """Seeks of readers that never read (no device stream) complete on the stand-in context: a goal inside the stream
    and one past its end give LWB_OK, a goal whose page walk meets a broken page gives LWF_ERR_OGG, as the single
    reader's seek does; absgp is None after them."""
    rs, add = readers
    good = _file(31, n_packets=8)
    broken = good + b"OggS\x01" + bytes(40)               # a page of an unknown version behind the last one
    add(good)
    add(broken)
    st = (C.c_int32 * 3)(7, 7, 7)
    assert _seek(lib, rs, [0, 1], [2000, 0], st) == 0
    assert list(st)[:2] == [0, 0]
    assert _seek(lib, rs, [1, 0], [10 ** 9, 10 ** 9], st) == 0
    assert list(st)[:2] == [OGG, 0]
    v = C.c_uint64()
    assert all(lib.lwf_readers_last_absgp(rs, i, C.byref(v)) == 1 for i in range(2))


def test_seek_refusals_change_nothing(lib, readers):
    rs, add = readers
    add(_file(41))
    add(_file(42))
    st = (C.c_int32 * 3)(7, 7, 7)
    assert _seek(lib, None, [0], [5], st) == INVALID
    assert _seek(lib, rs, None, [5], st) == INVALID
    assert _seek(lib, rs, [0], None, st) == INVALID
    assert _seek(lib, rs, [0], [5], None) == INVALID
    assert _seek(lib, rs, [0], [5], st, n=0) == INVALID
    assert _seek(lib, rs, [0, 2], [5, 5], st) == INVALID            # unknown index
    assert _seek(lib, rs, [1, 1], [5, 5], st) == INVALID            # a reader listed twice
    assert list(st) == [7, 7, 7]


def test_skip_refusals_change_nothing(lib, readers):
    """LWB_ERR_INVALID for a NULL readers, jobs, pcm or ticket, n_jobs == 0, a memory space other than host and device,
    an unknown out_format, an unknown or repeated reader, a planar out_stride below what one packet can return
    (blocksize_1 / 2 + (blocksize_1 - blocksize_0) / 4), out_channels below the reader's channel count, and a walk that
    enters a chained stream with more channels than the job has room for: no job result, absgp, headers, PCM element or
    ticket changes, and a call after them walks from where the readers stood."""
    from lewton_b200 import frontend as fe
    rs, add = readers
    add(_file(51))
    add(_file(52, channels=6, bs0=9, bs1=12))
    chained = _chained()
    assert len(set(_serials(chained))) == 2
    add(chained)
    heads = [lib.lwf_readers_headers(rs, i) for i in range(3)]
    need = [1024 + (2048 - 256) // 4, 2048 + (4096 - 512) // 4, 1024 + (2048 - 256) // 4]
    jobs = (fe._SkipJob * 3)()

    def reset_jobs():
        for k in range(3):
            jobs[k].reader, jobs[k].to_skip, jobs[k].out_offset, jobs[k].out_stride = k, 3000 + k, k * 100000, need[k]
            jobs[k].out_channels = 0
            jobs[k].left_to_skip, jobs[k].n_samples, jobs[k].got_packet, jobs[k].channels, jobs[k].status = 11, 22, 33, 44, 55
    reset_jobs()
    pcm = np.zeros(64, np.float32)
    t = C.c_uint64(5)
    ok = dict(rs=rs, jobs=jobs, n=3, fmt=0, pcm=pcm.ctypes.data, mem=0, t=C.byref(t))

    def skip(**kw):
        a = dict(ok, **kw)
        return lib.lwf_readers_skip_samples_linear(a["rs"], a["jobs"], a["n"], a["fmt"], a["pcm"], a["mem"], a["t"])

    def unchanged():
        for k in range(3):
            assert (jobs[k].left_to_skip, jobs[k].n_samples, jobs[k].got_packet, jobs[k].channels, jobs[k].status) == \
                (11, 22, 33, 44, 55), k
        assert not pcm.any() and t.value == 5
        v = C.c_uint64()
        assert all(lib.lwf_readers_last_absgp(rs, i, C.byref(v)) == 1 for i in range(3))
        assert [lib.lwf_readers_headers(rs, i) for i in range(3)] == heads

    assert skip(rs=None) == INVALID
    assert skip(jobs=None) == INVALID
    assert skip(n=0) == INVALID
    assert skip(pcm=None) == INVALID
    assert skip(t=None) == INVALID
    for mem in (-1, 2, 7):
        assert skip(mem=mem) == INVALID
    for fmt in (-1, 6, 100):
        assert skip(fmt=fmt) == INVALID
    unchanged()
    jobs[1].reader = 3
    assert skip() == INVALID                                    # unknown index
    jobs[1].reader = 0
    assert skip() == INVALID                                    # a reader in two jobs
    jobs[1].reader = 1
    for k in range(2):
        jobs[k].out_stride = need[k] - 1
        for fmt in (0, 1, 4):                                   # planar only: interleaved output has no planes
            assert skip(fmt=fmt) == INVALID
        jobs[k].out_stride = need[k]
    jobs[1].out_channels = 5
    assert skip() == INVALID
    jobs[1].out_channels = 0
    unchanged()
    # the chained file's skip runs through its stereo stream into the six-channel one, which a stereo job has no room
    # for: refused after the walk, which is undone -- twice, so the second walk starts where the first did
    jobs[2].to_skip = 10 ** 9
    for _ in range(2):
        assert skip(n=3) == INVALID
        unchanged()
    jobs[2].out_channels = 6
    jobs[2].out_stride = 2048 + (4096 - 512) // 4 - 1                # room in channels but not for a 4096 block
    assert skip(n=3) == INVALID
    unchanged()
    # seeks still work after the refusals
    st = (C.c_int32 * 3)()
    assert _seek(lib, rs, [0, 1, 2], [0, 0, 0], st) == 0 and list(st) == [0, 0, 0]
    assert [lib.lwf_readers_headers(rs, i) for i in range(3)] == heads


def test_stream_shapes_and_skip_room(lib):
    """OggStreamReaders.skip_room: the room of a skip job takes every logical stream of the file into account."""
    from lewton_b200 import frontend as fe
    assert fe._stream_shapes(_chained()) == [(2, 8, 11), (6, 9, 12)]
    assert fe._stream_shapes(_file(61)) == [(2, 8, 11)]
    spec = vp.StreamSpec(np.random.default_rng(62), channels=10, bs0=8, bs1=8)
    assert fe._stream_shapes(vp.ogg_stream(3, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], [], [])) == \
        [(10, 8, 8)]

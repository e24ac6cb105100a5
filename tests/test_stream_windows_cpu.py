"""Host-side checks of the output windows (lwb_stream_set_window / lwb_stream_window), without a GPU: the library
exports both calls and the header declares them as the ctypes binding does, no existing struct or kernel id moved, a
NULL stream is refused, the Python wrapper's arguments, and the clip plus the host-memory copy planner on windowed
chains (lewton_b200/csrc/pcm_copy_plan.h, compiled for the host): the copies cover exactly the samples the windows let
through, so no dropped sample crosses to the host."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from lewton_b200 import _cabi as cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "lewton_b200.h")
NO_LIMIT = (1 << 64) - 1


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import build
    build.build()
    return cabi.lib()


def test_window_calls_declared_bound_and_exported(lib):
    hdr = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    want = {"lwb_stream_set_window": ["lwb_stream *s", "uint64_t skip", "uint64_t limit"],
            "lwb_stream_window": ["const lwb_stream *s", "uint64_t *skip_left", "uint64_t *limit_left"]}
    for name, args in want.items():
        m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, hdr)
        assert m, name
        assert [a.strip() for a in m.group(1).split(",")] == args
        res, argtypes = cabi.SYMBOLS[name]
        assert res is C.c_int and len(argtypes) == len(args)
        assert getattr(lib, name) is not None
    assert cabi.SYMBOLS["lwb_stream_set_window"][1][1:] == [C.c_uint64, C.c_uint64]
    assert lib.lwb_abi_version() == 3
    nm = subprocess.run(["nm", "-D", "--defined-only", cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert {"lwb_stream_set_window", "lwb_stream_window"} <= set(re.findall(r" T (lwb_[a-z0-9_]+)", nm))


def test_null_stream_refused(lib):
    s, l_ = C.c_uint64(7), C.c_uint64(9)
    assert lib.lwb_stream_set_window(None, 0, NO_LIMIT) == cabi.ERR_INVALID
    assert lib.lwb_stream_set_window(None, 5, 5) == cabi.ERR_INVALID
    assert lib.lwb_stream_window(None, C.byref(s), C.byref(l_)) == cabi.ERR_INVALID
    assert lib.lwb_stream_window(None, None, None) == cabi.ERR_INVALID
    assert (s.value, l_.value) == (7, 9)


def test_kernel_ids_and_chain_struct_unchanged(tmp_path):
    ids = dict((k, int(v)) for k, v in re.findall(r"\b(LWB_KERNEL_\w+)\s*=\s*(\d+)", open(HEADER).read()))
    assert ids["LWB_KERNEL_COUNT"] == 14 == len(cabi.KERNELS)
    assert ids["LWB_KERNEL_ROW_COPY"] == 5
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "lewton_b200.h"\nint main(void){printf("%zu %zu\\n", sizeof(lwb_chain), '
                   "sizeof(lwb_batch_io));return 0;}\n")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "sz")], check=True)
    got = subprocess.run([str(tmp_path / "sz")], capture_output=True, text=True, check=True).stdout.split()
    assert [int(v) for v in got] == [88, 96] == [C.sizeof(cabi.Chain), C.sizeof(cabi.BatchIo)]


def test_python_wrapper_defaults_and_arguments(lib):
    import lewton_b200 as L
    assert L.api.NO_LIMIT == NO_LIMIT
    pwr = object.__new__(L.PreviousWindowRight)      # (no device: only the argument checks run)
    for bad in ((-1, None), (0, -1), (0, NO_LIMIT + 1)):
        with pytest.raises(ValueError):
            pwr.set_window(*bad)
    import inspect
    sig = inspect.signature(L.PreviousWindowRight.set_window)
    assert sig.parameters["skip"].default == 0 and sig.parameters["limit"].default is None
    assert isinstance(L.PreviousWindowRight.window, property)


def _emu(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "window_plan_emu.cpp")
    so = str(tmp_path_factory.mktemp("window_emu") / "libwindow_plan_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    lib = C.CDLL(so)
    lib.lwb_emu_window_plan.restype = C.c_long
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _emu(tmp_path_factory)


def _plan(emu, planar, chans, offs, strides, ns, skips, limits, max_pitch=1 << 40):
    n = len(chans)
    arrs = [np.array(chans, np.uint32)] + [np.array(v, np.uint64) for v in (offs, strides, ns, skips, limits)]
    skip, written = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    cap = sum(chans) + n + 1
    out = np.zeros((cap, 4), np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    k = emu.lwb_emu_window_plan(int(planar), C.c_size_t(n), *(p(a) for a in arrs), p(skip), p(written), C.c_uint64(max_pitch), p(out),
                                C.c_size_t(cap))
    assert k >= 0
    return skip, written, [tuple(int(v) for v in row) for row in out[:k]]


@pytest.mark.parametrize("planar", [True, False], ids=["planar", "interleaved"])
@pytest.mark.parametrize("seed", range(6))
def test_copies_cover_exactly_the_written_samples(emu, planar, seed):
    rng = np.random.default_rng(seed)
    n_chains = int(rng.integers(1, 40))
    chans, offs, strides, ns, skips, limits = [], [], [], [], [], []
    at = int(rng.integers(0, 9))
    for _ in range(n_chains):
        K, n = int(rng.integers(1, 7)), int(rng.integers(0, 5000))
        stride = n + int(rng.integers(0, 3)) * int(rng.integers(0, 64))
        chans.append(K)
        offs.append(at)
        strides.append(stride)
        ns.append(n)
        kind = int(rng.integers(0, 5))
        skips.append([0, int(rng.integers(0, n + 1)), n + int(rng.integers(0, 3000)), 0, int(rng.integers(0, 2 * n + 1))][kind])
        limits.append([NO_LIMIT, NO_LIMIT, NO_LIMIT, int(rng.integers(0, n + 1)), int(rng.integers(0, 2 * n + 1))][kind])
        at += (K * stride if planar else K * n) + int(rng.integers(0, 2)) * int(rng.integers(0, 50))
    skip, written, copies = _plan(emu, planar, chans, offs, strides, ns, skips, limits)
    want = np.zeros(at + 1, np.int32)
    for i in range(n_chains):
        assert skip[i] == min(skips[i], ns[i])
        assert written[i] == min(limits[i], ns[i] - skip[i])
        w = int(written[i])
        if planar:
            for k in range(chans[i]):
                want[offs[i] + k * strides[i]: offs[i] + k * strides[i] + w] += 1
        else:
            want[offs[i]: offs[i] + w * chans[i]] += 1
    got = np.zeros(at + 1, np.int32)
    for off, width, pitch, height in copies:
        for r in range(height):
            got[off + r * pitch: off + r * pitch + width] += 1
    assert np.array_equal(got, want), "the copies must move every written sample once and nothing else"
    assert int(got.sum()) == sum(int(written[i]) * chans[i] for i in range(n_chains))


def test_window_clip_edges(emu):
    # (produced, skip_left, limit_left) -> (skip, written)
    cases = [((1024, 0, NO_LIMIT), (0, 1024)), ((1024, 100, NO_LIMIT), (100, 924)), ((1024, 5000, NO_LIMIT), (1024, 0)),
             ((1024, 0, 10), (0, 10)), ((1024, 1000, 100), (1000, 24)), ((1024, 0, 0), (0, 0)), ((0, 7, 7), (0, 0)),
             ((1024, 1024, 5), (1024, 0))]
    for (n, s, lim), want in cases:
        skip, written, _ = _plan(emu, True, [2], [0], [n], [n], [s], [lim])
        assert (int(skip[0]), int(written[0])) == want, (n, s, lim)


@pytest.mark.parametrize("seed", range(4))
def test_window_counters_over_stopped_chains(emu, seed):
    """A window over batches whose chains stop: each batch produces the samples of its decoded packets only (none for a
    chain that stops at packet 0, none for the packet after the overlap guard emptied the state).  window_clip of each
    batch, with the counters moved as commit_stream_states moves them (skip_left by the samples dropped, limit_left by
    those written), writes exactly the window's slice of everything the batches produced, whatever the stops."""
    rng = np.random.default_rng(seed)
    for _ in range(50):
        produced = [int(rng.choice([0, 0, 1, 7, 128, 1024, int(rng.integers(0, 4000))])) for _ in range(int(rng.integers(1, 8)))]
        total = sum(produced)
        skip = int(rng.integers(0, total + 50))
        limit = [NO_LIMIT, int(rng.integers(0, total + 50)), 0][int(rng.integers(0, 3))]
        skip_left, limit_left, pos, got = skip, limit, 0, []
        for n in produced:
            s, w, _ = _plan(emu, True, [2], [0], [n], [n], [skip_left], [limit_left])
            s, w = int(s[0]), int(w[0])
            got += list(range(pos + s, pos + s + w))
            skip_left -= s
            if limit_left != NO_LIMIT:
                limit_left -= w
            pos += n
        end = total if limit == NO_LIMIT else min(total, skip + limit)
        assert got == list(range(min(skip, total), max(min(skip, total), end))), (produced, skip, limit)
        assert skip_left == max(skip - total, 0)
        assert limit_left == (NO_LIMIT if limit == NO_LIMIT else limit - len(got))

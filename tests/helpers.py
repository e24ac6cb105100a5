"""Shared test helpers: random setups / packets, the oracle-driven reference decode, and which kernels ran."""
import contextlib
import os

import numpy as np
import pytest

import lewton_b200 as L
from lewton_b200 import _cabi as cabi

# kernel names (Context.kernel_launches) by the path they belong to
ALL_KERNELS = frozenset(cabi.KERNELS)
GENERIC = frozenset({"k_prologue", "k_imdct", "k_overlap", "k_save_state"})      # the four-kernel path
FRONT = frozenset({"k_floor1_segments", "k_prologue_fused"})                     # two-kernel front stages
FUSED = frozenset({"k_long", "k_long_s", "k_mid", "k_short", "k_short_g"})       # the fused synthesis kernels


@contextlib.contextmanager
def environ(env):
    """Sets the environment variables of dict `env` (None: none) for the block, then restores them."""
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@contextlib.contextmanager
def expect_kernels(ctx, ran=(), not_ran=()):
    """Checks which kernels the block launched on ctx.  ran: names that must have run (a dict: exact launch counts);
    not_ran: names that must not.  Yields a dict that holds {name: launches} of the block once it has finished."""
    unknown = (set(ran) | set(not_ran)) - ALL_KERNELS
    assert not unknown, f"no such kernels: {sorted(unknown)}"
    k0 = ctx.kernel_launches()
    delta = {}
    yield delta
    k1 = ctx.kernel_launches()
    delta.update({k: k1[k] - k0[k] for k in k1})
    launched = {k: v for k, v in delta.items() if v}
    if isinstance(ran, dict):
        wrong = {k: delta[k] for k, v in ran.items() if delta[k] != v}
        assert not wrong, f"expected launches {ran}, got {launched}"
    else:
        missing = sorted(k for k in ran if not delta[k])
        assert not missing, f"expected {missing} to run; launched {launched}"
    extra = sorted(k for k in not_ran if delta[k])
    assert not extra, f"expected {extra} not to run; launched {launched}"


@pytest.fixture(autouse=True)
def launches_are_attributed(request):
    """GPU tests (modules import this fixture): across every test, the per-kernel launch counts of the module's ctx
    grow by exactly as much as its total launch count, so a launch site that does not attribute itself fails."""
    if request.node.get_closest_marker("gpu") is None or "ctx" not in request.fixturenames:
        yield
        return
    ctx = request.getfixturevalue("ctx")
    t0, k0 = ctx.launch_count, sum(ctx.kernel_launches().values())
    yield
    t1, k1 = ctx.launch_count, sum(ctx.kernel_launches().values())
    assert k1 - k0 == t1 - t0, f"{t1 - t0} launches, {k1 - k0} of them attributed to a kernel"


def bits_equal(a, b):
    """Bit-identical float arrays, treating +0/-0 as equal and any-NaN == any-NaN
    (SURVEY.md section 8c parity rule)."""
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    if a.shape != b.shape:
        return False
    same = a.view(np.uint32) == b.view(np.uint32)
    zeros = (a == 0) & (b == 0)
    nans = np.isnan(a) & np.isnan(b)
    return bool(np.all(same | zeros | nans))


def mismatch_report(a, b):
    a = np.ascontiguousarray(a, np.float32).ravel()
    b = np.ascontiguousarray(b, np.float32).ravel()
    bad = np.nonzero(~((a.view(np.uint32) == b.view(np.uint32)) | ((a == 0) & (b == 0)) | (np.isnan(a) & np.isnan(b))))[0]
    return f"{bad.size} of {a.size} differ; first at {bad[:5]}: got {a[bad[:5]]} want {b[bad[:5]]}"


F32_GUARD = 0x7fa5a5a5        # a NaN with a fixed payload: no kernel produces it, compared bit for bit
I16_GUARD = 0x5a5a


def write_set(chains, channels_of, fmt):
    """The element intervals each chain produced, as the ABI states them (include/lewton_b200.h, lwb_chain):
    planar: [out_offset + c * out_stride, + n_samples) per channel c; interleaved: [out_offset, + n_samples * C).
    chains: ChainSpec objects after the call; channels_of(i) -> channel count of chain i.
    Returns [(chain index, [(start, length), ...])]."""
    planar = fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR)
    out = []
    for i, c in enumerate(chains):
        C, n = channels_of(i), int(c.n_samples)
        if planar:
            spans = [(int(c.out_offset) + k * int(c.out_stride), n) for k in range(C)]
        else:
            spans = [(int(c.out_offset), n * C)]
        out.append((i, [s for s in spans if s[1]]))
    return out


def _bits(buf):
    return buf.view(np.uint32 if buf.dtype == np.float32 else np.uint16)


def fill_guard(buf):
    """Fills an f32 / i16 output arena with the sentinel before a call; returns it."""
    _bits(buf)[...] = F32_GUARD if buf.dtype == np.float32 else I16_GUARD
    return buf


def assert_contained(buf, ws, what=""):
    """Every element of `buf` outside the write set `ws` (see write_set) still holds the sentinel."""
    flat = _bits(buf.reshape(-1))
    outside = np.ones(flat.size, bool)
    for _, spans in ws:
        for s, n in spans:
            assert s + n <= flat.size, f"{what}: a chain's write set ends past the arena ({s} + {n} > {flat.size})"
            outside[s:s + n] = False
    guard = F32_GUARD if buf.dtype == np.float32 else I16_GUARD
    bad = np.nonzero(outside & (flat != guard))[0]
    if bad.size:
        i = int(bad[0])
        near = [k for k, spans in ws if spans and min(s for s, _ in spans) <= i < max(s + n for s, n in spans)]
        raise AssertionError(f"{what}: {bad.size} elements outside the write set were written; first at {i} "
                             f"(value bits {int(flat[i]):#x}), inside the extent of chains {near[:4]}")


def random_floor1(rng, n2):
    mult = int(rng.integers(1, 5))
    rangebits = int(rng.integers(max(4, int(np.log2(n2)) - 2), min(15, int(np.log2(n2)) + 2) + 1))
    nposts = int(rng.integers(2, 66))
    nposts = min(nposts, 1 << rangebits)
    xs = [0, 1 << rangebits] + [int(v) for v in rng.permutation(np.arange(1, 1 << rangebits))[: nposts - 2]]
    return mult, xs


def random_floor1_y(rng, mult, nposts, wild=False):
    rng_y = [256, 128, 86, 64][mult - 1]
    y = [int(rng.integers(0, rng_y)), int(rng.integers(0, rng_y))]
    for _ in range(nposts - 2):
        r = rng.random()
        if r < 0.3:
            y.append(0)
        elif r < 0.9 or not wild:
            y.append(int(rng.integers(1, 40)))
        else:
            y.append(int(rng.integers(1, 5000)))
    return y


class RefStream:
    """Oracle-side twin of one stream: decodes packet by packet with oracle.synth_*."""

    def __init__(self, oracle, channels, bs0, bs1, modes, mappings=None, floors=None, tables=None):
        """tables: the oracle's (t0, t1) Tables the setup was given (default: generated)."""
        self.o, self.ch, self.bs0, self.bs1, self.tables = oracle, channels, bs0, bs1, tables
        self.modes = modes                      # [(blockflag, mapping)]
        self.mappings = mappings or [{"coupling": [], "floor_of_channel": [0] * channels}]
        self.floors = floors or []              # [(mult, xs)] -> oracle Floor1 objects
        self.ofloors = [oracle.make_floor1(m, xs) for (m, xs) in self.floors]
        self.pwr = oracle.Pwr(channels, bs1)

    def spectrum(self, mode, prev, nxt, spec):
        bf = self.modes[mode][0]
        return self.o.synth_spectrum(self.bs0, self.bs1, bf, prev, nxt, spec, self.pwr, tables=self.tables)

    def packet(self, mode, prev, nxt, residue, floors):
        """floors: per channel None | list y | ndarray dense"""
        bf, mi = self.modes[mode]
        mp = self.mappings[mi]
        fl = []
        for c, f in enumerate(floors):
            if f is None or (isinstance(f, np.ndarray) and f.dtype.kind == "f"):
                fl.append(f)
            else:
                fl.append((self.ofloors[mp["floor_of_channel"][c]], f))
        return self.o.synth_packet(self.bs0, self.bs1, bf, prev, nxt, mp["coupling"], fl, residue, self.pwr, tables=self.tables)


def make_setup(ctx, channels, bs0, bs1, modes=((0, 0), (1, 0)), mappings=None, floors=None, tables=None):
    """modes: [(blockflag, mapping)]; mappings: [{"coupling": [(m,a)..], "floor_of_channel": [..]}];
    floors: [(mult, xs)]"""
    mappings = mappings or [{"coupling": [], "floor_of_channel": [0] * channels}]
    floors = floors or [(1, [0, 128])]
    lf = [L.FloorTypeOne(m, xs) for (m, xs) in floors]
    lm = []
    for mp in mappings:
        # one submap per distinct floor, mux maps channel -> submap
        fo = mp["floor_of_channel"]
        uniq = sorted(set(fo))
        lm.append(L.Mapping(channels, [m for m, _ in mp["coupling"]], [a for _, a in mp["coupling"]],
                            mux=[uniq.index(f) for f in fo], submap_floors=uniq))
    lmodes = [L.ModeInfo(bf, mi) for bf, mi in modes]
    return L.Setup(ctx, channels, bs0, bs1, lf, lm, lmodes, tables=tables)


def mode_sequence(rng, n, p_short=0.3):
    """Random block-type sequence with consistent prev/next flags: returns (modes, prev, next)
    with mode 0 = short, 1 = long."""
    bf = (rng.random(n) >= p_short).astype(np.uint8)
    prev = np.ones(n, np.uint8)
    nxt = np.ones(n, np.uint8)
    for i in range(n):
        if bf[i]:
            prev[i] = bf[i - 1] if i else 1
            nxt[i] = bf[i + 1] if i + 1 < n else 1
    return bf, prev, nxt

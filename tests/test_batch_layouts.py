"""Where batch results land.  Every path of lwb_decode_chains writes exactly the samples it reports -- n_samples per
channel plane at out_offset + c * out_stride (planar), n_samples * channels at out_offset (interleaved) -- and nothing
else in the output arena, in host and device memory, for every layout the ABI allows: tight, padded, channel-major,
reversed, offsets that are not multiples of 4, empty chains and fresh streams.  The samples are bit-exact against the
oracle (f32; i16 exact) whatever mix of setups a batch holds, each chain's output equals what it gives decoded alone,
and misaligned device arenas give the same bytes as aligned ones."""

import numpy as np
import pytest

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from helpers import (ALL_KERNELS, FRONT, FUSED, GENERIC, RefStream, assert_contained, bits_equal, environ, expect_kernels, fill_guard,
                     launches_are_attributed, make_setup, mismatch_report, random_floor1_y, write_set)

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

PLANAR = (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR)
F32 = (cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED)
FORMATS = (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED)
LAYOUTS = ("tight", "padded", "channel_major", "reverse", "odd")
FLOOR = (2, [0, 128, 12, 46, 4, 8, 16, 23, 33, 70])
_COUPLING_51 = [(0, 1), (2, 3), (0, 4)]


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def flags(bf):
    """Consistent window flags for a block sequence (mode 0 short, mode 1 long)."""
    n = len(bf)
    prev, nxt = np.ones(n, np.uint8), np.ones(n, np.uint8)
    for i in range(n):
        if bf[i]:
            prev[i] = bf[i - 1] if i else 1
            nxt[i] = bf[i + 1] if i + 1 < n else 1
    return prev, nxt


class Kind:
    """A setup of the test; tables: the caller's own [(dict for bs0), (dict for bs1)], which its oracle twin gets too."""

    def __init__(self, ctx, C, bs0, bs1, coupling=None, tables=None):
        self.C, self.bs0, self.bs1, self.tables = C, bs0, bs1, tables
        if coupling is None:
            coupling = [(0, 1)] if C == 2 else []
        self.mappings = [{"coupling": list(coupling), "floor_of_channel": [0] * C}]
        self.floors = [FLOOR]
        self.su = make_setup(ctx, C, bs0, bs1, mappings=self.mappings, floors=self.floors, tables=tables)

    def n2(self, mode):
        return (1 << (self.bs1 if mode else self.bs0)) // 2


class Stream:
    """A stream, its oracle twin and the block sequence it will decode over the batches of a test."""

    def __init__(self, oracle, kind):
        self.kind = kind
        self.pwr = L.PreviousWindowRight(kind.su)
        tabs = None if kind.tables is None else tuple(oracle.Tables.from_arrays(b, **kind.tables[i])
                                                      for i, b in enumerate((kind.bs0, kind.bs1)))
        self.ref = RefStream(oracle, kind.C, kind.bs0, kind.bs1, [(0, 0), (1, 0)], kind.mappings, kind.floors, tables=tabs)
        self.bf = np.zeros(0, np.uint8)
        self.at = 0

    def plan(self, rng, n, p_short):
        self.bf = (rng.random(n) >= p_short).astype(np.uint8)
        self.prev, self.nxt = flags(self.bf)
        self.at = 0

    def take(self, n):
        a, self.at = self.at, self.at + n
        return self.bf[a:self.at], self.prev[a:self.at], self.nxt[a:self.at]


class Packets:
    """The next packets of one stream: inputs, expected sample count and (with an oracle twin) the oracle's PCM."""

    def __init__(self, rng, st, n, residue, bf=None):
        if bf is None:
            bf, prev, nxt = st.take(n)
        else:
            prev, nxt = flags(bf)
        self.bf, self.prev, self.nxt = bf, prev, nxt
        k = st.kind
        has = not (st.ref.pwr if st.ref else st.pwr).is_empty()      # (the oracle twin may run ahead of the device)
        self.n = 0
        for i in range(len(bf)):
            if has:
                self.n += L.get_decoded_sample_count(k.su, int(bf[i]), int(prev[i]), int(nxt[i]))
            has = True
        coeffs, kinds, ys, dense, parts = [], [], [], [], []
        for i in range(len(bf)):
            n2 = k.n2(bf[i])
            if residue:
                res = (rng.standard_normal((k.C, n2)) * rng.integers(0, 2, (k.C, n2))).astype(np.float32)
                fl = []
                for r in rng.random(k.C):
                    fl.append(None if r < 0.1 else rng.random(n2).astype(np.float32) if r < 0.2 else random_floor1_y(rng, FLOOR[0], len(FLOOR[1])))
                kd, y, d = L.DecodedPacket(int(bf[i]), res, fl).pack()
                kinds.append(kd)
                ys.append(y)
                dense.append(np.zeros_like(res) if d is None else d)
                if st.ref:
                    rc, o = st.ref.packet(int(bf[i]), int(prev[i]), int(nxt[i]), res, fl)
                coeffs.append(res)
            else:
                spec = (rng.standard_normal((k.C, n2)) * 0.1).astype(np.float32)
                if st.ref:
                    rc, o = st.ref.spectrum(int(bf[i]), int(prev[i]), int(nxt[i]), spec)
                coeffs.append(spec)
            if st.ref:
                assert rc == 0
                parts.append(o)
        flat = lambda xs, dt: np.concatenate([x.ravel() for x in xs]) if xs else np.zeros(0, dt)
        self.coeffs, self.dense = flat(coeffs, np.float32), flat(dense, np.float32)
        self.kinds = np.stack(kinds) if kinds else np.zeros((0, k.C), np.uint8)
        self.ys = np.stack(ys) if ys else np.zeros((0, k.C, cabi.MAX_POSTS), np.uint32)
        self.want = None
        if st.ref:
            self.want = np.concatenate(parts, axis=1) if parts else np.zeros((k.C, 0), np.float32)
            assert self.want.shape[1] == self.n


def place(layout, Cs, ns, fmt, rng):
    """Output offsets / strides of the chains under `layout`; returns (offsets, strides, arena elements)."""
    S, planar = len(Cs), fmt in PLANAR
    r4 = lambda x: (x + 3) // 4 * 4
    offs, strides = [0] * S, [0] * S
    if planar and layout == "channel_major":
        base = max(4, r4(max(ns, default=0)))
        return [s * base for s in range(S)], [S * base] * S, max(Cs) * S * base
    pos = int(rng.integers(1, 4)) if layout == "odd" else 0
    for s in (range(S - 1, -1, -1) if layout == "reverse" else range(S)):
        if layout == "tight":
            st = ns[s]
        elif layout == "odd":
            st = r4(ns[s]) + int(rng.integers(1, 4))
        else:
            st = r4(ns[s]) + 4 * int(rng.integers(1, 3))
        strides[s] = st if planar else 0
        offs[s] = pos
        pos += Cs[s] * (st if planar else ns[s])
        if layout == "odd":
            pos += int(rng.integers(1, 4))
        elif layout != "tight":
            pos += 4 * int(rng.integers(0, 3))
    return offs, strides, pos


class Batch:
    """The arenas and chain list of one lwb_decode_chains call over (stream, Packets) items."""

    def __init__(self, items, fmt, layout, rng, residue):
        self.items, self.fmt, self.residue = items, fmt, residue
        S = len(items)
        self.Cs = [st.kind.C for st, _ in items]
        offs, strides, self.total = place(layout, self.Cs, [pk.n for _, pk in items], fmt, rng)
        coff, cpos, rows = [0] * S, 0, 0
        for s in (range(S - 1, -1, -1) if layout == "reverse" else range(S)):
            cpos += int(rng.integers(1, 4)) if layout == "odd" else 0
            coff[s] = cpos
            cpos += items[s][1].coeffs.size
        self.coeffs = np.zeros(cpos, np.float32)
        self.dense = np.zeros(cpos, np.float32)
        C0 = self.Cs[0] if S else 1
        nrows = sum(len(pk.bf) for _, pk in items)
        self.kinds = np.zeros((nrows, C0), np.uint8)
        self.ys = np.zeros((nrows, C0, cabi.MAX_POSTS), np.uint32)
        self.specs = []
        for s, (st, pk) in enumerate(items):
            self.coeffs[coff[s]:coff[s] + pk.coeffs.size] = pk.coeffs
            if residue and len(pk.bf):
                self.dense[coff[s]:coff[s] + pk.coeffs.size] = pk.dense
                self.kinds[rows:rows + len(pk.bf), :pk.kinds.shape[1]] = pk.kinds
                self.ys[rows:rows + len(pk.bf), :pk.ys.shape[1]] = pk.ys
            self.specs.append(L.ChainSpec(st.pwr, pk.bf, pk.prev, pk.nxt, coeff_offset=coff[s], packet_index=rows,
                                          out_offset=offs[s], out_stride=strides[s]))
            rows += len(pk.bf)

    def run(self, ctx, memory, shift=0, env=None):
        """Runs the batch on a sentinel-filled arena; device arenas (and the dense floor) start `shift` bytes past an
        allocation.  Returns (status, whole arena as read back)."""
        dt = np.float32 if self.fmt in F32 else np.int16
        pcm = fill_guard(np.empty(max(self.total, 1), dt))
        entry = cabi.ENTRY_RESIDUE if self.residue else cabi.ENTRY_SPECTRUM
        kw = dict(floor_kind=self.kinds, floor1_y=self.ys) if self.residue else {}
        rc = 0
        with environ(env):
            if memory == cabi.MEM_HOST:
                if self.residue:
                    kw["dense_floor"] = self.dense
                try:
                    L.decode_chains(ctx, self.specs, entry, memory, self.coeffs, pcm, self.fmt, **kw)
                except L.AudioReadError as e:
                    rc = e.code
                return rc, pcm
            allocs = []

            def dev(arr):
                p = ctx.device_alloc(arr.nbytes + 16)
                allocs.append(p)
                ctx.h2d(p + shift, arr)
                return p + shift
            try:
                d_in, d_out = dev(self.coeffs), dev(pcm)
                if self.residue:
                    kw["dense_floor"] = dev(self.dense)
                try:
                    L.decode_chains(ctx, self.specs, entry, memory, d_in, d_out, self.fmt, **kw)
                except L.AudioReadError as e:
                    rc = e.code
                ctx.synchronize()
                ctx.d2h(pcm, d_out)
            finally:
                for p in allocs:
                    ctx.device_free(p)
        return rc, pcm

    def chain_pcm(self, pcm, i):
        c, C, n = self.specs[i], self.Cs[i], self.items[i][1].n
        if self.fmt in PLANAR:
            return np.stack([pcm[c.out_offset + k * c.out_stride:c.out_offset + k * c.out_stride + n] for k in range(C)])
        return np.ascontiguousarray(pcm[c.out_offset:c.out_offset + n * C].reshape(n, C).T)

    def check(self, oracle, pcm, what):
        """Per chain: status, counts, the oracle's PCM and state; then nothing outside the write set."""
        for i, (st, pk) in enumerate(self.items):
            c = self.specs[i]
            assert (c.status, c.packets_done, c.n_samples) == (0, len(pk.bf), pk.n), (what, i, c.status, c.packets_done, c.n_samples, pk.n)
            if pk.want is None:
                continue
            got = self.chain_pcm(pcm, i)
            if self.fmt in F32:
                assert bits_equal(got, pk.want), (what, i, mismatch_report(got, pk.want))
            else:
                assert np.array_equal(got, oracle.quantise_i16(pk.want)), (what, i)
            a, b = st.pwr.data(), st.ref.pwr.data()
            assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (what, i, "state")
        assert_contained(pcm, write_set(self.specs, lambda i: self.Cs[i], self.fmt), what)


# ------------------------------------------------------------------------------------------------
# every path, every layout
# ------------------------------------------------------------------------------------------------
SHAPES = {   # name: channels, blocksize_0, blocksize_1, share of short blocks, residue entry, environment, the kernels the
             # shape exists to reach (planar output, 16-byte aligned offsets)
    "long": (2, 8, 11, 0.0, False, None, {"k_long"}),
    "mid1024": (2, 10, 10, 0.0, False, None, {"k_mid"}),                               # n = 1024
    "mid512": (1, 9, 9, 0.0, False, None, {"k_mid"}),                                  # n = 512
    "short": (2, 8, 8, 0.0, False, None, {"k_short"}),
    "mixed": (2, 8, 11, 0.5, False, None, {"k_long_s", "k_short_g"}),                  # the one pass, bursts of short blocks
    "mixed_rounds": (2, 8, 11, 0.5, False, {"LWB_MIXED_ROUNDS": "1"}, {"k_long", "k_short"}),   # rounds
    "chain": (6, 8, 11, 0.3, False, {"LWB_NO_MIXED": "1"}, {"k_chain"}),
    "generic": (2, 8, 11, 0.3, False, {"LWB_FORCE_GENERIC": "1"}, {"k_imdct", "k_overlap", "k_save_state"}),   # four-kernel path
    "residue_long": (2, 8, 11, 0.0, True, None, FRONT | {"k_long"}),
    "residue_mid": (2, 10, 10, 0.0, True, None, FRONT | {"k_mid"}),
    "residue_mixed": (2, 8, 11, 0.3, True, None, FRONT | {"k_long_s"}),                # front stages + the one pass
}
# kernels a shape's environment switches off, whatever the layout
SWITCHED_OFF = {"mixed_rounds": {"k_long_s", "k_short_g", "k_row_copy"}, "chain": ALL_KERNELS - {"k_chain"},
                "generic": ALL_KERNELS - GENERIC}


def merged(*envs):
    out = {}
    for e in envs:
        out.update(e or {})
    return out or None


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_every_path_writes_exactly_its_samples_in_every_layout(ctx, oracle, shape, memory, fmt):
    """Seven chains (one without packets) over three consecutive batches -- fresh streams first, so their first packet
    emits nothing -- in each layout; host-memory batches run their third batch in three pipelined chunks."""
    C, bs0, bs1, p_short, residue, env, reach = SHAPES[shape]
    rng = np.random.default_rng(100 * list(SHAPES).index(shape) + 10 * memory + fmt)
    kind = Kind(ctx, C, bs0, bs1)
    reached = set()
    for layout in LAYOUTS:
        streams = [Stream(oracle, kind) for _ in range(7)]
        lengths = [[int(rng.integers(0, 7)) if s != 1 else 0 for s in range(7)] for _ in range(3)]
        for s, st in enumerate(streams):
            st.plan(rng, sum(lengths[b][s] for b in range(3)), p_short)
        for b in range(3):
            items = [(st, Packets(rng, st, lengths[b][s], residue)) for s, st in enumerate(streams)]
            batch = Batch(items, fmt, layout, rng, residue)
            chunks = {"LWB_E2E_CHUNKS": "3"} if memory == cabi.MEM_HOST and b == 2 else None
            with expect_kernels(ctx, not_ran=SWITCHED_OFF.get(shape, ())) as launched:
                rc, pcm = batch.run(ctx, memory, env=merged(env, chunks))
            assert rc == 0, (layout, b, rc)
            batch.check(oracle, pcm, (shape, layout, b))
            if layout != "odd":
                reached |= {k for k, v in launched.items() if v}
    if fmt in PLANAR or not reach & FUSED:             # (the fused kernels write planar output only)
        assert reach <= reached, (sorted(reach - reached), sorted(reached))


@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE])
@pytest.mark.parametrize("shape,fmt", [("long", cabi.OUT_F32_PLANAR), ("mixed", cabi.OUT_I16_PLANAR),
                                       ("mid1024", cabi.OUT_F32_PLANAR), ("short", cabi.OUT_I16_PLANAR)])
def test_prepared_batch_replays_into_a_padded_layout(ctx, oracle, shape, fmt, memory):
    """One prepared batch (lwb_plan_execute) run four times with new spectra in the same arenas: every step bit-exact and
    contained, in a padded layout and in one with offsets that are not multiples of 4."""
    C, bs0, bs1, p_short, _, _, _ = SHAPES[shape]
    for layout in ("padded", "odd"):
        rng = np.random.default_rng(77 + len(shape) + memory)
        kind = Kind(ctx, C, bs0, bs1)
        S, P = 6, 7
        streams = [Stream(oracle, kind) for _ in range(S)]
        seqs = []
        for _ in range(S):
            bf = (rng.random(P) >= p_short).astype(np.uint8)
            bf[0] = bf[-1] = 1                          # replayed: the sequence must close on itself
            seqs.append(bf)
        # the steady-state sample counts size the strides; the first step (fresh streams) emits less
        twins = [Stream(oracle, kind) for _ in range(S)]
        for tw, bf in zip(twins, seqs):
            Packets(rng, tw, P, False, bf)
        steady = Batch([(tw, Packets(rng, tw, P, False, bf)) for tw, bf in zip(twins, seqs)], fmt, layout, rng, False)
        items = [(st, Packets(rng, st, P, False, bf)) for st, bf in zip(streams, seqs)]
        first = Batch(items, fmt, layout, rng, False)
        for i, c in enumerate(first.specs):
            c.out_offset, c.out_stride = steady.specs[i].out_offset, steady.specs[i].out_stride
            c.coeff_offset = steady.specs[i].coeff_offset
        first.total, coeffs = steady.total, np.zeros_like(steady.coeffs)
        dt = np.float32 if fmt in F32 else np.int16
        pcm = np.empty(max(first.total, 1), dt)
        if memory == cabi.MEM_HOST:
            a_in, a_out = coeffs, pcm
        else:
            a_in, a_out = ctx.device_alloc(coeffs.nbytes), ctx.device_alloc(pcm.nbytes)
        plan = L.Batch(ctx, first.specs, cabi.ENTRY_SPECTRUM, memory, a_in, a_out, fmt)
        kernels = []
        for step in range(4):
            if step:
                first.items = [(st, Packets(rng, st, P, False, bf)) for st, bf in zip(streams, seqs)]
            for i, (_, pk) in enumerate(first.items):
                coeffs[first.specs[i].coeff_offset:first.specs[i].coeff_offset + pk.coeffs.size] = pk.coeffs
            fill_guard(pcm)
            if memory == cabi.MEM_DEVICE:
                ctx.h2d(a_in, coeffs)
                ctx.h2d(a_out, pcm)
            with expect_kernels(ctx) as launched:
                plan.run()
            kernels.append(launched)
            ctx.synchronize()
            if memory == cabi.MEM_DEVICE:
                ctx.d2h(pcm, a_out)
            plan.collect()
            first.check(oracle, pcm, (shape, layout, "step", step))
        # step 0 runs on fresh streams and changes their state; step 1 plans and captures, steps 2 and 3 replay
        assert kernels[1] == kernels[2] == kernels[3], (layout, kernels)      # a replay launches what the capture did
        plan.close()
        if memory == cabi.MEM_DEVICE:
            ctx.device_free(a_in)
            ctx.device_free(a_out)


# ------------------------------------------------------------------------------------------------
# one stream appended to one planar buffer, call after call
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", PLANAR)
@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE])
@pytest.mark.parametrize("shape", ["long", "mixed"])
def test_consecutive_calls_append_to_one_planar_buffer(ctx, oracle, shape, memory, fmt):
    """Three calls decode one stereo stream into one [2][total] buffer, each at out_offset = the samples so far and
    out_stride = total: the buffer must end up as the oracle's concatenation.  A call that copied back the span between
    its first and last plane would overwrite channel 1's earlier samples."""
    C, bs0, bs1, p_short, _, _, _ = SHAPES[shape]
    rng = np.random.default_rng(5150 + memory + 2 * fmt)
    st = Stream(oracle, Kind(ctx, C, bs0, bs1))
    lengths = [5, 4, 6]
    st.plan(rng, sum(lengths), p_short)
    calls = [Packets(rng, st, n, False) for n in lengths]
    ns = [pk.n for pk in calls]
    total = sum(ns)
    dt = np.float32 if fmt in F32 else np.int16
    buf = fill_guard(np.empty(C * total, dt))
    d_out = ctx.device_alloc(buf.nbytes) if memory == cabi.MEM_DEVICE else None
    if d_out:
        ctx.h2d(d_out, buf)
    pos = 0
    for pk, n in zip(calls, ns):
        spec = L.ChainSpec(st.pwr, pk.bf, pk.prev, pk.nxt, out_offset=pos, out_stride=total)
        if memory == cabi.MEM_HOST:
            L.decode_chains(ctx, [spec], cabi.ENTRY_SPECTRUM, memory, pk.coeffs, buf, fmt)
        else:
            d_in = ctx.device_alloc(pk.coeffs.nbytes + 16)
            ctx.h2d(d_in, pk.coeffs)
            L.decode_chains(ctx, [spec], cabi.ENTRY_SPECTRUM, memory, d_in, d_out, fmt)
            ctx.synchronize()
            ctx.device_free(d_in)
        assert spec.status == 0 and spec.n_samples == n, (spec.status, spec.n_samples, n)
        pos += n
    if d_out:
        ctx.d2h(buf, d_out)
        ctx.device_free(d_out)
    want = np.concatenate([pk.want for pk in calls], axis=1)
    got = buf.reshape(C, total)
    if fmt in F32:
        assert bits_equal(got, want), mismatch_report(got, want)
    else:
        assert np.array_equal(got, oracle.quantise_i16(want))


# ------------------------------------------------------------------------------------------------
# heterogeneous batches
# ------------------------------------------------------------------------------------------------
def setup_pool(ctx):
    pool = [Kind(ctx, C, b0, b1, coupling=_COUPLING_51 if C == 6 else None)
            for C, b0, b1 in [(1, 8, 11), (2, 8, 11), (6, 8, 11), (8, 8, 11), (2, 8, 8), (2, 9, 9), (1, 10, 10),
                              (2, 10, 10), (2, 8, 10), (2, 6, 13), (2, 11, 11)]]
    pool.append(Kind(ctx, 10, 8, 11))                                   # only the four-kernel path takes 10 channels
    pool.append(Kind(ctx, 2, 8, 11, tables=[L.generate_tables(8), L.generate_tables(11)]))     # the cached pack's tables
    bent = [L.generate_tables(8), L.generate_tables(11)]
    bent[1]["window"][300] = np.nextafter(bent[1]["window"][300], np.float32(2))
    bent[1]["a"][7] = np.nextafter(bent[1]["a"][7], np.float32(2))
    pool.append(Kind(ctx, 2, 8, 11, tables=bent))                       # tables of its own, the oracle twin's too
    return pool


def alone(ctx, st, pk, fmt, memory, residue):
    """The chain decoded on its own, on a clone of the stream as it was before the batch: its PCM [C][n]."""
    twin = Stream.__new__(Stream)
    twin.kind, twin.pwr, twin.ref = st.kind, st.before, None
    one = Batch([(twin, pk)], fmt, "tight", np.random.default_rng(0), residue)
    rc, pcm = one.run(ctx, memory)
    c = one.specs[0]
    assert rc == 0 and (c.status, c.n_samples) == (0, pk.n)
    return one.chain_pcm(pcm, 0)


@pytest.mark.parametrize("S,p_short,memory,fmt,seed", [
    (3, 0.0, cabi.MEM_DEVICE, cabi.OUT_F32_PLANAR, 1),
    (3, 0.5, cabi.MEM_HOST, cabi.OUT_I16_INTERLEAVED, 2),
    (40, 0.1, cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 3),
    (40, 0.5, cabi.MEM_DEVICE, cabi.OUT_I16_PLANAR, 4),
    (40, 0.0, cabi.MEM_HOST, cabi.OUT_F32_INTERLEAVED, 5),
    (300, 0.1, cabi.MEM_DEVICE, cabi.OUT_F32_PLANAR, 6),
    (300, 0.0, cabi.MEM_HOST, cabi.OUT_I16_PLANAR, 7),
    (300, 0.5, cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 8)])
def test_heterogeneous_batches(ctx, oracle, S, p_short, memory, fmt, seed):
    """Chains of random setups, lengths 0..24 and block sequences, in a random layout, over three consecutive batches:
    each chain equals the oracle and, byte for byte, itself decoded alone -- one chain's share of the batch-wide
    choices (channels, blocksizes, twiddle packs) must never reach another's."""
    rng = np.random.default_rng(4000 + seed)
    pool = setup_pool(ctx)
    streams = [Stream(oracle, pool[int(rng.integers(0, len(pool)))]) for _ in range(S)]
    lengths = rng.integers(0, 25, (3, S))
    for s, st in enumerate(streams):
        st.plan(rng, int(lengths[:, s].sum()), p_short)
    for b in range(3):
        layout = LAYOUTS[int(rng.integers(0, len(LAYOUTS)))]
        for st in streams:
            st.before = st.pwr.clone()
        items = [(st, Packets(rng, st, int(lengths[b, s]), False)) for s, st in enumerate(streams)]
        batch = Batch(items, fmt, layout, rng, False)
        rc, pcm = batch.run(ctx, memory)
        assert rc == 0, (b, rc)
        batch.check(oracle, pcm, (layout, b))
        for i, (st, pk) in enumerate(items):
            got = batch.chain_pcm(pcm, i)
            ref = alone(ctx, st, pk, fmt, memory, False)
            assert np.array_equal(got.view(np.uint8), ref.view(np.uint8)), (layout, b, i, st.kind.C, st.kind.bs0, st.kind.bs1)
            st.before.close()


@pytest.mark.parametrize("memory,fmt,seed", [(cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 11), (cabi.MEM_DEVICE, cabi.OUT_I16_PLANAR, 12),
                                             (cabi.MEM_HOST, cabi.OUT_F32_INTERLEAVED, 13)])
def test_heterogeneous_residue_batches(ctx, oracle, memory, fmt, seed):
    """The residue entry wants one channel count per batch: stereo chains of every stereo setup of the pool, as above.
    A batch that mixes channel counts is refused with LWB_ERR_INVALID and changes nothing: the arena keeps its sentinel
    and every stream its state."""
    rng = np.random.default_rng(5000 + seed)
    pool = [k for k in setup_pool(ctx) if k.C == 2]
    S = 40
    streams = [Stream(oracle, pool[int(rng.integers(0, len(pool)))]) for _ in range(S)]
    lengths = rng.integers(0, 25, (3, S))
    for s, st in enumerate(streams):
        st.plan(rng, int(lengths[:, s].sum()), 0.3)
    for b in range(3):
        layout = LAYOUTS[int(rng.integers(0, len(LAYOUTS)))]
        for st in streams:
            st.before = st.pwr.clone()
        items = [(st, Packets(rng, st, int(lengths[b, s]), True)) for s, st in enumerate(streams)]
        batch = Batch(items, fmt, layout, rng, True)
        rc, pcm = batch.run(ctx, memory)
        assert rc == 0, (b, rc)
        batch.check(oracle, pcm, (layout, b))
        for i, (st, pk) in enumerate(items):
            ref = alone(ctx, st, pk, fmt, memory, True)
            assert np.array_equal(batch.chain_pcm(pcm, i).view(np.uint8), ref.view(np.uint8)), (layout, b, i)
            st.before.close()
    # mixed channel counts: refused, nothing written, no state changed
    fresh = [Stream(oracle, k) for k in (pool[0], pool[1], Kind(ctx, 1, 8, 11))]
    for st in fresh:
        st.plan(rng, 3, 0.0)
    for st in fresh[:2]:
        held = rng.standard_normal((2, 1 << (st.kind.bs1 - 1))).astype(np.float32)
        st.pwr.set_data(held)
        st.ref.pwr.set_data(held)
    items = [(st, Packets(rng, st, 3, True)) for st in fresh]
    states = [st.pwr.data() for st, _ in items]
    batch = Batch(items, fmt, "padded", rng, True)
    rc, pcm = batch.run(ctx, memory)
    assert rc == cabi.ERR_INVALID
    assert_contained(pcm, [], "refused batch")
    for (st, _), s0 in zip(items, states):
        a = st.pwr.data()
        assert (a is None) == (s0 is None) and (a is None or bits_equal(a, s0))


# ------------------------------------------------------------------------------------------------
# misaligned device arenas
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", PLANAR)
@pytest.mark.parametrize("shape", ["long", "mid1024", "short", "mixed", "residue_long", "residue_mixed"])
def test_misaligned_device_arenas_match_aligned(ctx, oracle, shape, fmt):
    """coeffs / pcm (and the dense floor of the residue entry) 4, 8 or 12 bytes past a 16-byte boundary: the fused
    kernels' bulk copies and vector stores cannot take them, so the batch runs on the chain kernel -- with the same bytes.
    The aligned batches reach the shape's fused kernels."""
    C, bs0, bs1, p_short, residue, env, reach = SHAPES[shape]
    kind = Kind(ctx, C, bs0, bs1)
    arenas = {}
    for shift in (0, 4, 8, 12):
        rng = np.random.default_rng(6000 + len(shape) + fmt)
        streams = [Stream(oracle, kind) for _ in range(5)]
        lengths = rng.integers(1, 8, (2, 5))
        for s, st in enumerate(streams):
            st.plan(rng, int(lengths[:, s].sum()), p_short)
        reached = set()
        for b in range(2):
            items = [(st, Packets(rng, st, int(lengths[b, s]), residue)) for s, st in enumerate(streams)]
            batch = Batch(items, fmt, "padded", rng, residue)
            with expect_kernels(ctx, ran={"k_chain"} if shift else (), not_ran=ALL_KERNELS - {"k_chain"} if shift else ()) as launched:
                rc, pcm = batch.run(ctx, cabi.MEM_DEVICE, shift=shift, env=env)
            reached |= {k for k, v in launched.items() if v}
            assert rc == 0, (shift, b, rc)
            batch.check(oracle, pcm, (shape, shift, b))
            arenas[(shift, b)] = pcm
        if not shift:
            assert reach & FUSED <= reached, (sorted(reach), sorted(reached))
        for st in streams:
            st.pwr.close()
    for shift in (4, 8, 12):
        for b in range(2):
            assert np.array_equal(arenas[(shift, b)].view(np.uint8), arenas[(0, b)].view(np.uint8)), (shift, b)

"""Batches queued back to back without a synchronise, against the oracle.

A device-memory batch (LWB_MEM_DEVICE) returns once its launches are queued, and a decode server -- like bench.py's timed
loop -- submits the next one at once.  Much of the host side exists for that: the pinned descriptor staging ring, the
double-buffered k_long runs, the ticket pool, the context's scratch arenas, the copy streams of host-memory batches and
the descriptors a prepared batch replays.  Each is guarded by stream or event order only, and only a call that queues
behind unfinished work can tell whether that order is right.  So every test first closes a gate: torch.cuda._sleep on
the context's stream for about GATE_SECONDS, then an event.  The calls after it queue behind the gate, and each test
asserts that the gate was still closed when its second call returned.

Every chain is compared with an oracle twin that runs on the host, packet by packet, in the order of the queued calls:
f32 PCM bit for bit (bits_equal), i16 PCM exactly, nothing written outside a chain's write set, and every stream's final
state bit for bit.  A prepared batch writes the same arenas every step, so each step's output is snapshotted by a copy on
the context's stream: the final state alone depends on the last packet only.

The library waits on the host in these places by design; the tests work around them:
- Arena growth.  ensure() synchronises when it grows an arena.  Each sequence first runs ungated, on other streams and
  output arenas of the same sizes, so that no queued call grows one.
- Staging ring wrap.  acquire_staging waits for the copy three stagings back, so only the first two or three calls that
  stage descriptors return while the gate is closed.  The later ones wait for it to open, and they still reuse the ring.
- Host-memory batches return after their PCM has landed.
- Inputs are in device arenas before the gate closes."""
import threading
import types

import numpy as np
import pytest
import torch

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from helpers import (ALL_KERNELS, FRONT, RefStream, assert_contained, bits_equal, environ, expect_kernels, fill_guard,
                     launches_are_attributed, make_setup, mismatch_report, mode_sequence, random_floor1_y, write_set)

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

GATE_SECONDS = 0.3
FLOOR = (2, [0, 128, 12, 46, 4, 8, 16, 23, 33, 70])
STEREO = [{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}]
SETUPS = {"mixed": (8, 11, [(0, 0), (1, 0)]), "mid": (10, 10, [(1, 0)]), "short": (8, 8, [(1, 0)])}   # bs0, bs1, modes
F32P, I16P, F32I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED
RESIDUE, SPECTRUM = cabi.ENTRY_RESIDUE, cabi.ENTRY_SPECTRUM
MIXED_EXTRA = {"k_short", "k_row_copy"}      # what the one pass may add to k_long_s + k_short_g


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


class Gate:
    """Holds a context's CUDA stream for about GATE_SECONDS: work queued after close() waits behind it."""
    cycles_per_s = None

    def __init__(self, ctx):
        self.stream = torch.cuda.ExternalStream(ctx.cuda_stream, device=torch.device("cuda", ctx.device))
        self.opened = None
        if Gate.cycles_per_s is None:
            with torch.cuda.stream(self.stream):
                torch.cuda._sleep(1000)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                torch.cuda._sleep(50_000_000)
                b.record()
            b.synchronize()
            Gate.cycles_per_s = 50_000_000 / (a.elapsed_time(b) * 1e-3)

    def close(self):
        with torch.cuda.stream(self.stream):
            torch.cuda._sleep(int(Gate.cycles_per_s * GATE_SECONDS))
            self.opened = torch.cuda.Event()
            self.opened.record()

    def assert_closed(self, what):
        assert not self.opened.query(), (f"{what}: the gate had opened when the second call returned, so nothing queued "
                                         f"behind it: the gate ({GATE_SECONDS} s) was too short")

    def on_stream(self):
        """Torch work (arena copies, snapshots) in the context's stream order."""
        return torch.cuda.stream(self.stream)


class Twin:
    """A device stream and its oracle twin."""

    def __init__(self, oracle, su, kind):
        self.su = su
        self.bs0, self.bs1, self.modes = SETUPS[kind]
        self.pwr = L.PreviousWindowRight(su)
        self.ref = RefStream(oracle, 2, self.bs0, self.bs1, self.modes, STEREO, [FLOOR])

    def n2(self, mode):
        return (1 << (self.bs1 if self.modes[mode][0] else self.bs0)) // 2

    def check_state(self, what):
        a, b = self.pwr.data(), self.ref.pwr.data()
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (what, "state")


def setups(ctx):
    return {k: make_setup(ctx, 2, b0, b1, modes=m, mappings=STEREO, floors=[FLOOR]) for k, (b0, b1, m) in SETUPS.items()}


def twins(oracle, sus, kind, n):
    return [Twin(oracle, sus[kind], kind) for _ in range(n)]


def flags(bf):
    n = len(bf)
    prev, nxt = np.ones(n, np.uint8), np.ones(n, np.uint8)
    for i in range(n):
        if bf[i]:
            prev[i] = bf[i - 1] if i else 1
            nxt[i] = bf[i + 1] if i + 1 < n else 1
    return prev, nxt


def seq(rng, kind, P):
    """(mode numbers, prev flags, next flags) of P packets.  'long': long blocks; 'mixed': short and long blocks that
    start and end long, so that consecutive calls join up; 'uniform': the one mode of a 'mid' or 'short' setup."""
    if kind == "mixed":
        bf = mode_sequence(rng, P, p_short=0.3)[0]
        bf[0] = bf[-1] = 1
    else:
        bf = np.ones(P, np.uint8)
    prev, nxt = flags(bf)
    return (np.zeros(P, np.uint8) if kind == "uniform" else bf), prev, nxt


def items(rng, ts, kind, P):
    return [(t, seq(rng, kind, P)) for t in ts]


def packet_inputs(rng, tw, mode, residue, floors=None):
    """One packet's coefficients and, for the residue entry, its floors (per channel None | y list | dense curve)."""
    n2 = tw.n2(mode)
    if not residue:
        return (rng.standard_normal((2, n2)) * 0.1).astype(np.float32), None
    res = (rng.standard_normal((2, n2)) * rng.integers(0, 2, (2, n2))).astype(np.float32)
    if floors is None:
        floors = [None if r < 0.1 else rng.random(n2).astype(np.float32) if r < 0.2 else
                  random_floor1_y(rng, FLOOR[0], len(FLOOR[1])) for r in rng.random(2)]
    return res, floors


class Call:
    """One decode_chains call over (twin, sequence) items: its inputs, its arenas (on the device for MEM_DEVICE, output
    filled with the sentinel) and the oracle's output.  Building it runs the twins over its packets, so the calls of a
    test are built in the order they are submitted.  Planar strides leave room for the samples of a stream with history
    plus a gap, so calls over the same sequences have the same layout.  floors: fixed floors of every packet, [item][packet]."""

    def __init__(self, rng, items, entry=SPECTRUM, fmt=F32P, memory=cabi.MEM_DEVICE, floor_memory=cabi.MEM_HOST,
                 pinned=False, floors=None, expect=((), ())):
        self.items, self.entry, self.fmt, self.memory, self.floor_memory = items, entry, fmt, memory, floor_memory
        self.expect = expect
        residue = entry == RESIDUE
        planar = fmt in (F32P, I16P)
        coeffs, dense, kinds, ys = [], [], [], []
        self.wants, self.chains = [], []
        coff = ooff = rows = 0
        for j, (tw, (modes, prev, nxt)) in enumerate(items):
            parts, steady, c0 = [], 0, coff
            for i, m in enumerate(int(x) for x in modes):
                x, fl = packet_inputs(rng, tw, m, residue, floors[j][i] if floors else None)
                if residue:
                    k, y, d = L.DecodedPacket(m, x, fl).pack()
                    kinds.append(k)
                    ys.append(y)
                    dense.append(np.zeros_like(x) if d is None else d)
                    rc, o = tw.ref.packet(m, int(prev[i]), int(nxt[i]), x, fl)
                else:
                    rc, o = tw.ref.spectrum(m, int(prev[i]), int(nxt[i]), x)
                assert rc == 0
                parts.append(o)
                coeffs.append(x.ravel())
                coff += x.size
                steady += L.get_decoded_sample_count(tw.su, m, int(prev[i]), int(nxt[i]))
            self.wants.append(np.concatenate(parts, axis=1))
            stride = (steady + 3) // 4 * 4 + 4
            self.chains.append(L.ChainSpec(tw.pwr, modes, prev, nxt, coeff_offset=c0, packet_index=rows, out_offset=ooff,
                                           out_stride=stride if planar else 0))
            ooff += 2 * stride + 4 if planar else (2 * steady + 3) // 4 * 4 + 4
            rows += len(modes)
        self.total = ooff
        self.pcm = fill_guard(np.empty(self.total, np.float32 if fmt in (F32P, F32I) else np.int16))
        self.coeffs = np.concatenate(coeffs)
        self.kw = {}
        if residue:
            self.kinds, self.ys, self.dense = np.stack(kinds), np.stack(ys), np.concatenate([d.ravel() for d in dense])
            if pinned:          # page-locked copies: the library's uploads read them when the stream reaches the copy
                self.pinned = [torch.from_numpy(a).pin_memory() for a in (self.kinds, self.ys)]
                self.kinds, self.ys = (t.numpy() for t in self.pinned)
            self.kw = dict(floor_kind=self.kinds, floor1_y=self.ys, dense_floor=self.dense, floor_memory=floor_memory)
        if memory == cabi.MEM_DEVICE:
            self.dev = {"coeffs": torch.from_numpy(self.coeffs).cuda(), "pcm": torch.from_numpy(self.pcm).cuda()}
            if residue:
                self.dev["dense"] = torch.from_numpy(self.dense).cuda()
                self.kw["dense_floor"] = self.dev["dense"].data_ptr()
                if floor_memory == cabi.MEM_DEVICE:
                    self.dev["kinds"], self.dev["ys"] = torch.from_numpy(self.kinds).cuda(), torch.from_numpy(self.ys).cuda()
                    self.kw.update(floor_kind=self.dev["kinds"].data_ptr(), floor1_y=self.dev["ys"].data_ptr())

    def submit(self, ctx):
        if self.memory == cabi.MEM_DEVICE:
            arenas = (self.dev["coeffs"].data_ptr(), self.dev["pcm"].data_ptr())
        else:
            arenas = (self.coeffs, self.pcm)
        ran, not_ran = self.expect
        with expect_kernels(ctx, ran=ran, not_ran=not_ran):
            L.decode_chains(ctx, self.chains, self.entry, self.memory, *arenas, self.fmt, **self.kw)

    def check(self, oracle, what):
        """After the call's work has run: results, the whole output arena and the stream states."""
        pcm = self.dev["pcm"].cpu().numpy() if self.memory == cabi.MEM_DEVICE else self.pcm
        for i, c in enumerate(self.chains):
            assert (c.status, c.packets_done, c.n_samples) == (0, len(c.modes), self.wants[i].shape[1]), \
                (what, i, c.status, c.packets_done, c.n_samples)
        check_arena(oracle, pcm, self.chains, self.wants, self.fmt, what)


def check_arena(oracle, pcm, chains, wants, fmt, what):
    """A whole output arena against the oracle: chains give the layout, wants [2][n] per chain; nothing else written."""
    planar = fmt in (F32P, I16P)
    spans = []
    for i, (c, want) in enumerate(zip(chains, wants)):
        n = want.shape[1]
        if planar:
            got = np.stack([pcm[c.out_offset + k * c.out_stride:c.out_offset + k * c.out_stride + n] for k in range(2)])
        else:
            got = pcm[c.out_offset:c.out_offset + 2 * n].reshape(n, 2).T
        if fmt in (F32P, F32I):
            assert bits_equal(got, want), (what, i, mismatch_report(got, want))
        else:
            assert np.array_equal(got, oracle.quantise_i16(want)), (what, i)
        spans.append(types.SimpleNamespace(out_offset=c.out_offset, out_stride=c.out_stride, n_samples=n))
    assert_contained(pcm, write_set(spans, lambda i: 2, fmt), what)


def run_queued(ctx, gate, calls, what, sync=True):
    """Submits the calls behind the gate (None: ungated), checks that the second returned before it opened.  sync: wait
    for the device first, so that the calls' arenas have been filled."""
    if sync:
        torch.cuda.synchronize()
    if gate:
        gate.close()
    for k, call in enumerate(calls):
        call.submit(ctx)
        if gate and k == 1:
            gate.assert_closed(what)


# ------------------------------------------------------------------------------------------------
# streams handed from path to path
# ------------------------------------------------------------------------------------------------
def path_sequence(rng, oracle, sus):
    """Eight stereo 256/2048 streams through nine calls, each taken by another path, then streams of 1024-point and
    256-point blocks through k_mid and k_short.  Returns (calls, twins)."""
    g, mid, short = twins(oracle, sus, "mixed", 8), twins(oracle, sus, "mid", 4), twins(oracle, sus, "short", 4)
    mixed = {"k_long_s", "k_short_g"}
    calls = [
        Call(rng, items(rng, g, "long", 8), expect=({"k_long": 1}, ALL_KERNELS - {"k_long"})),
        Call(rng, items(rng, g, "long", 8), RESIDUE, floor_memory=cabi.MEM_DEVICE,
             expect=({"k_floor1_segments": 1, "k_prologue_fused": 1, "k_long": 1}, ALL_KERNELS - FRONT - {"k_long"})),
        Call(rng, items(rng, g, "mixed", 16), expect=(mixed, ALL_KERNELS - mixed - MIXED_EXTRA)),
        Call(rng, items(rng, g, "mixed", 16), RESIDUE, fmt=I16P,
             expect=(FRONT | {"k_long_s"}, ALL_KERNELS - FRONT - mixed - MIXED_EXTRA)),
        Call(rng, items(rng, g, "mixed", 12), fmt=F32I, expect=({"k_chain"}, ALL_KERNELS - {"k_chain"})),
        Call(rng, items(rng, g, "long", 8), expect=({"k_long": 1}, ALL_KERNELS - {"k_long"})),     # runs_buf reused
        Call(rng, items(rng, mid, "uniform", 8), expect=({"k_mid"}, ALL_KERNELS - {"k_mid"})),
        Call(rng, items(rng, mid, "uniform", 8), RESIDUE, expect=(FRONT | {"k_mid"}, ALL_KERNELS - FRONT - {"k_mid"})),
        Call(rng, items(rng, short, "uniform", 16), expect=({"k_short"}, ALL_KERNELS - {"k_short"})),
    ]
    return calls, g + mid + short


def check_all(oracle, calls, tws, what):
    for k, call in enumerate(calls):
        call.check(oracle, (what, "call", k))
    for tw in tws:
        tw.check_state(what)


def test_streams_handed_from_path_to_path(ctx, oracle):
    """Queued calls over the same streams, each taken by another batch path: the state moves from kernel to kernel on the
    device, and the k_long batch at the end reuses the descriptor half of the first while that one is still queued."""
    sus = setups(ctx)
    gate = Gate(ctx)
    for gated in (False, True):
        calls, tws = path_sequence(np.random.default_rng(1), oracle, sus)
        run_queued(ctx, gate if gated else None, calls, "path to path")
        ctx.synchronize()
        check_all(oracle, calls, tws, ("gated" if gated else "warm-up"))


def test_long_batches_back_to_back(ctx, oracle):
    """Six k_long batches of one layout, each with arenas of its own: the third reuses the first's half of the
    double-buffered runs and the sixth waits for the third's staging slot, both while the gate holds the first."""
    sus = setups(ctx)
    gate = Gate(ctx)
    for gated in (False, True):
        rng = np.random.default_rng(6)
        tws = twins(oracle, sus, "mixed", 6)
        seqs = items(rng, tws, "long", 8)
        calls = [Call(rng, seqs, expect=({"k_long": 1}, ALL_KERNELS - {"k_long"})) for _ in range(6)]
        run_queued(ctx, gate if gated else None, calls, "k_long back to back")
        ctx.synchronize()
        check_all(oracle, calls, tws, ("gated" if gated else "warm-up"))


# ------------------------------------------------------------------------------------------------
# prepared batches
# ------------------------------------------------------------------------------------------------
class Plan:
    """A prepared batch (L.Batch) over the layout of `steps[0]`, fed step k's inputs by on-stream copies and snapshotted
    after each run."""

    def __init__(self, ctx, steps, snap_steps=None):
        first = steps[0]
        self.steps, self.fmt = steps, first.fmt
        self.snap_at = {k: i for i, k in enumerate(range(len(steps)) if snap_steps is None else snap_steps)}
        sets = {}                           # distinct input arrays -> row of the pool
        self.which = [sets.setdefault(id(s.coeffs), len(sets)) for s in steps]
        uniq = {id(s.coeffs): s.coeffs for s in steps}
        self.pool = torch.from_numpy(np.stack([uniq[i] for i in sets])).cuda()
        self.arena = torch.empty_like(self.pool[0])
        self.guard = torch.from_numpy(first.pcm).cuda()
        self.pcm = self.guard.clone()
        self.snaps = torch.empty((len(self.snap_at), first.total), dtype=self.pcm.dtype, device="cuda")
        kw = dict(first.kw)
        if first.entry == RESIDUE:          # floors are the same every step; the dense floor arena is the first step's
            kw["dense_floor"] = first.dev["dense"].data_ptr()
        self.batch = L.Batch(ctx, first.chains, first.entry, cabi.MEM_DEVICE, self.arena.data_ptr(), self.pcm.data_ptr(),
                             first.fmt, **kw)

    def run(self, ctx, gate, k):
        with gate.on_stream():
            self.arena.copy_(self.pool[self.which[k]])
            self.pcm.copy_(self.guard)
        ran, not_ran = self.steps[k].expect
        with expect_kernels(ctx, ran=ran, not_ran=not_ran):
            self.batch.run()
        if k in self.snap_at:
            with gate.on_stream():
                self.snaps[self.snap_at[k]].copy_(self.pcm)

    def check(self, oracle, what):
        snaps = self.snaps.cpu().numpy()
        for k, i in self.snap_at.items():
            check_arena(oracle, snaps[i], self.steps[0].chains, self.steps[k].wants, self.fmt, (what, "step", k))
        for c, want in zip(self.batch.collect(), self.steps[-1].wants):
            assert (c.status, c.n_samples) == (0, want.shape[1]), (what, c.status, c.n_samples)


def interleaved_plans(oracle, gated, big):
    """Plans A and B run A, B, A, B, ... for eight steps each, with a plain batch of `big` streams after the fourth pair."""
    ctx = L.Context(0)
    try:
        sus = setups(ctx)
        gate = Gate(ctx)
        rng = np.random.default_rng(2)
        a_seqs = items(rng, twins(oracle, sus, "mixed", 6), "long", 8)
        b_seqs = items(rng, twins(oracle, sus, "mixed", 6), "mixed", 12)
        b_floors = [[packet_inputs(rng, tw, int(m), True)[1] for m in modes] for tw, (modes, _, _) in b_seqs]
        steps = 8
        a = [Call(rng, a_seqs, expect=({"k_long": 1}, ALL_KERNELS - {"k_long"})) for _ in range(steps)]
        b = [Call(rng, b_seqs, RESIDUE, fmt=I16P, floors=b_floors,
                  expect=(FRONT | {"k_long_s"}, ALL_KERNELS - FRONT - {"k_long_s", "k_short_g"} - MIXED_EXTRA))
             for _ in range(steps)]
        plain_twins = twins(oracle, sus, "mixed", big)
        plain = Call(rng, items(rng, plain_twins, "mixed", 24), RESIDUE, expect=(FRONT, ()))
        plans = [Plan(ctx, a), Plan(ctx, b)]
        torch.cuda.synchronize()
        if gated:
            gate.close()
        for k in range(steps):
            if k == steps // 2:
                plain.submit(ctx)                # grows ctx->spec and the segment tables: both plans must re-plan
            for p in plans:
                p.run(ctx, gate, k)
                if gated and k == 0 and p is plans[1]:
                    gate.assert_closed("plans A, B")
        ctx.synchronize()
        what = "gated" if gated else "warm-up"
        plans[0].check(oracle, (what, "A"))
        plans[1].check(oracle, (what, "B"))
        plain.check(oracle, (what, "plain"))
        for tw, _ in a_seqs + b_seqs:
            tw.check_state(what)
        for tw in plain_twins:
            tw.check_state(what)
        for p in plans:
            p.batch.close()
    finally:
        ctx.close()


def test_two_prepared_batches_interleaved(oracle):
    """A uniform-long spectrum plan (A) and a mixed residue plan whose host floor arrays its front stages upload on every
    replay (B), queued alternately on a context of their own.  The first step of each runs on fresh streams, so the
    second re-plans while the first is still queued; the plain batch halfway grows the context's scratch, so both
    re-plan again.  Every step's snapshot matches the oracle."""
    interleaved_plans(oracle, False, 12)
    interleaved_plans(oracle, True, 24)     # larger than anything before on its context: it grows the arenas


def test_prepared_k_long_across_a_ticket_pool_wrap(ctx, oracle):
    """A small k_long plan replayed until the context's k_long launches cross a multiple of the ticket pool (1024):
    the pool is zeroed on the stream at the wrap, while the replays before it are still queued."""
    sus = setups(ctx)
    gate = Gate(ctx)
    rng = np.random.default_rng(3)
    warm_seqs = items(rng, twins(oracle, sus, "mixed", 4), "long", 8)
    warm = Plan(ctx, [Call(rng, warm_seqs, expect=({"k_long": 1}, ALL_KERNELS - {"k_long"})) for _ in range(3)])
    for k in range(3):
        warm.run(ctx, gate, k)
    ctx.synchronize()
    warm.check(oracle, "warm-up")
    warm.batch.close()
    c0 = ctx.kernel_launches()["k_long"]
    before = (1024 - c0 % 1024) % 1024
    if before < 12:
        before += 1024
    n = before + 12
    tws = twins(oracle, sus, "mixed", 4)
    seqs = items(rng, tws, "long", 8)
    layout = Call(rng, seqs, expect=({"k_long": 1}, ALL_KERNELS - {"k_long"}))       # (its packets are not decoded)
    for tw in tws:
        tw.ref.pwr.reset()
    # 64 distinct input sets, used in turn (step k's output depends on the inputs of steps k - 1 and k)
    inputs = [(rng.standard_normal(layout.coeffs.shape) * 0.1).astype(np.float32) for _ in range(64)]
    steps = []
    for k in range(n):
        st = types.SimpleNamespace(coeffs=inputs[k % 64], expect=layout.expect, wants=[])
        x = inputs[k % 64]
        for (tw, (modes, prev, nxt)), c in zip(seqs, layout.chains):
            parts = []
            for i in range(len(modes)):
                off = c.coeff_offset + i * 2048
                rc, o = tw.ref.spectrum(int(modes[i]), int(prev[i]), int(nxt[i]), x[off:off + 2048].reshape(2, 1024))
                assert rc == 0
                parts.append(o)
            st.wants.append(np.concatenate(parts, axis=1))
        steps.append(st)
    for attr in ("chains", "fmt", "pcm", "total", "entry", "kw"):
        setattr(steps[0], attr, getattr(layout, attr))
    checked = sorted(set(range(before - 10, before + 10)) | {n - 1})
    plan = Plan(ctx, steps, snap_steps=checked)
    torch.cuda.synchronize()
    gate.close()
    for k in range(n):
        plan.run(ctx, gate, k)
        if k == 1:
            gate.assert_closed("ticket wrap")
    c1 = ctx.kernel_launches()["k_long"]
    assert c1 - c0 == n and c0 // 1024 < c1 // 1024, (c0, c1)
    ctx.synchronize()
    plan.check(oracle, "ticket wrap")
    for tw in tws:
        tw.check_state("ticket wrap")
    plan.batch.close()


# ------------------------------------------------------------------------------------------------
# host-memory batches behind queued device work
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("host_path,chunks", [("residue_long", None), ("long", 64), ("residue_long", 64),
                                              ("residue_mixed", 64)])
def test_host_batch_right_behind_queued_device_work(ctx, oracle, host_path, chunks):
    """Two replays of a device-memory residue plan, whose front stages upload its host floor arrays into the context's
    ctx->kinds / ctx->ys on every replay, then at once a host-memory batch whose copy_in uploads overwrite the same
    scratch: they must wait for the queued work (order_copies_behind_compute).  (Replays stage no descriptors, so the
    host batch is planned and uploaded while the gate is closed rather than after a staging-ring wait.)  With
    LWB_E2E_CHUNKS=64 and 64 chains every ev_in / ev_done slot is used."""
    sus = setups(ctx)
    gate = Gate(ctx)
    S = 64 if chunks else 8
    kind = "mixed" if host_path == "residue_mixed" else "long"
    entry = SPECTRUM if host_path == "long" else RESIDUE
    for gated in (False, True):
        rng = np.random.default_rng(4)
        seqs = items(rng, twins(oracle, sus, "mixed", 8), "long", 8)
        floors = [[packet_inputs(rng, tw, int(m), True)[1] for m in modes] for tw, (modes, _, _) in seqs]
        plan = Plan(ctx, [Call(rng, seqs, RESIDUE, floors=floors, expect=({"k_floor1_segments": 1, "k_prologue_fused": 1,
                                                                            "k_long": 1}, ALL_KERNELS - FRONT - {"k_long"}))
                          for _ in range(4)])
        host_twins = twins(oracle, sus, "mixed", S)
        host = Call(rng, items(rng, host_twins, kind, 6), entry, memory=cabi.MEM_HOST,
                    expect=({"k_long_s"} if kind == "mixed" else {"k_long"}, {"k_chain", "k_prologue"}))
        torch.cuda.synchronize()
        plan.run(ctx, gate, 0)                  # fresh streams
        plan.run(ctx, gate, 1)                  # planned and captured
        ctx.synchronize()
        if gated:
            gate.close()
        plan.run(ctx, gate, 2)
        plan.run(ctx, gate, 3)
        if gated:
            gate.assert_closed("replays")
        with environ({"LWB_E2E_CHUNKS": str(chunks)} if chunks else None):
            host.submit(ctx)
        ctx.synchronize()
        what = ("gated" if gated else "warm-up", host_path, chunks)
        plan.check(oracle, what)
        host.check(oracle, what)
        for tw in [tw for tw, _ in seqs] + host_twins:
            tw.check_state(what)
        plan.batch.close()


# ------------------------------------------------------------------------------------------------
# two contexts on two host threads
# ------------------------------------------------------------------------------------------------
def test_two_contexts_on_two_threads(oracle):
    """Each of two contexts runs the path-to-path sequence behind its own gate, from its own host thread, at once (the
    C calls release the GIL).  The sequences are built, and checked, on the main thread."""
    ctxs = [L.Context(0), L.Context(0)]
    try:
        work = []
        for i, c in enumerate(ctxs):
            sus = setups(c)
            calls, tws = path_sequence(np.random.default_rng(50 + i), oracle, sus)      # warm-up
            run_queued(c, None, calls, "warm-up")
            c.synchronize()
            check_all(oracle, calls, tws, ("warm-up", i))
            work.append((Gate(c), *path_sequence(np.random.default_rng(50 + i), oracle, sus)))
        torch.cuda.synchronize()
        start, errors = threading.Barrier(2), []

        def worker(i):
            try:
                gate, calls, _ = work[i]
                start.wait()
                run_queued(ctxs[i], gate, calls, ("thread", i), sync=False)     # (a device-wide sync would wait for the other gate)
                ctxs[i].synchronize()
            except BaseException as e:                   # re-raised on the main thread
                errors.append(e)
        threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        for i, (_, calls, tws) in enumerate(work):
            check_all(oracle, calls, tws, ("thread", i))
    finally:
        for c in ctxs:
            c.close()


# ------------------------------------------------------------------------------------------------
# host floor arrays of a device batch
# ------------------------------------------------------------------------------------------------
def test_pinned_host_floor_arrays_of_a_device_batch(ctx, oracle):
    """A device-memory batch uploads its host floor arrays by copies queued on the context's stream; from page-locked
    memory such a copy reads them only when the stream reaches it.  The header states the contract that follows: the
    arrays stay unchanged until the batch's work has run.  Kept so, pinned arrays behind the gate give the oracle's
    output."""
    sus = setups(ctx)
    gate = Gate(ctx)
    for gated in (False, True):
        rng = np.random.default_rng(5)
        tws = twins(oracle, sus, "mixed", 8)
        calls = [Call(rng, items(rng, tws, "long", 8), RESIDUE, pinned=True, expect=(FRONT | {"k_long"}, ())),
                 Call(rng, items(rng, tws, "mixed", 12), RESIDUE, pinned=True, expect=(FRONT | {"k_long_s"}, ()))]
        run_queued(ctx, gate if gated else None, calls, "pinned floors")
        ctx.synchronize()
        check_all(oracle, calls, tws, ("gated" if gated else "warm-up"))

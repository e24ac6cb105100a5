"""Asynchronous batches (lwb_submit_chains / lwb_ticket_query / lwb_ticket_wait) against the oracle.

A host-memory submit returns once its copies and kernels are queued; the library stages it in one of the context's two
host arena sets, whose uploads wait on the GPU only for the batch that used the same set before.  So the tests queue
submits behind a gate (test_queued_batches.Gate: torch.cuda._sleep on the context's stream, then an event) and check
what the contract states: every submit returned while the gate was still closed, no ticket completed and no PCM landed
before it opened, and after the tickets completed every chain matches an oracle twin that ran the same packets in
submission order -- f32 PCM bit for bit, i16 PCM exactly, nothing outside the write set of a sentinel-filled page-locked
arena changed, and every stream's final state bit for bit.  Each sequence runs ungated first, so that no arena grows in
the gated run, and every call names the kernels that must (and must not) run.

A submit still waits on the host in the places the header lists (arena growth, staging-ring wrap); must_return() says
how many submits of each path return behind the gate.  Page-locked arrays are freed before a gate closes: cudaFreeHost
waits for the device."""
import ctypes
import threading

import numpy as np
import pytest
import torch

import lewton_b200 as L
import vorbis_packer as vp
from helpers import (ALL_KERNELS, F32_GUARD, FRONT, GENERIC, RefStream, assert_contained, bits_equal, expect_kernels, fill_guard,
                     launches_are_attributed, make_setup, mismatch_report, mode_sequence, random_floor1_y, write_set)
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from test_frontend_gpu import consistent_modes, oracle_pcm
from test_queued_batches import FLOOR, MIXED_EXTRA, SETUPS, STEREO, Gate, environ, flags

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, I16P, F32I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED
RESIDUE, SPECTRUM, HOST, DEVICE = cabi.ENTRY_RESIDUE, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, cabi.MEM_DEVICE
WIDE = 10                     # channels of the four-kernel path's streams (the fused kernels and k_chain take <= 8)


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def mappings(C):
    return STEREO if C == 2 else [{"coupling": [], "floor_of_channel": [0] * C}]


def setups(ctx):
    sus = {k: make_setup(ctx, 2, b0, b1, modes=m, mappings=STEREO, floors=[FLOOR]) for k, (b0, b1, m) in SETUPS.items()}
    b0, b1, m = SETUPS["mixed"]
    sus["wide"] = make_setup(ctx, WIDE, b0, b1, modes=m, mappings=mappings(WIDE), floors=[FLOOR])
    return sus


class Twin:
    """A device stream and its oracle twin, of C channels."""

    def __init__(self, oracle, su, kind):
        self.su, self.C = su, su.audio_channels
        self.bs0, self.bs1, self.modes = SETUPS["mixed" if kind == "wide" else kind]
        self.pwr = L.PreviousWindowRight(su)
        self.ref = RefStream(oracle, self.C, self.bs0, self.bs1, self.modes, mappings(self.C), [FLOOR])

    def n2(self, mode):
        return (1 << (self.bs1 if self.modes[mode][0] else self.bs0)) // 2

    def check_state(self, what):
        a, b = self.pwr.data(), self.ref.pwr.data()
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (what, "state")


def twins(oracle, sus, kind, n):
    return [Twin(oracle, sus[kind], kind) for _ in range(n)]


def seq(rng, kind, P):
    """(modes, prev, next) of P packets: 'long', 'uniform' (the one mode of 'mid' / 'short'), or 'mixed' short and long
    blocks that start and end long, so that consecutive calls join up."""
    if kind == "mixed":
        bf = mode_sequence(rng, P, p_short=0.3)[0]
        bf[0] = bf[-1] = 1
    else:
        bf = np.ones(P, np.uint8)
    prev, nxt = flags(bf)
    return (np.zeros(P, np.uint8) if kind == "uniform" else bf), prev, nxt


class AsyncCall:
    """One batch over (twin, (modes, prev, next)) items: inputs, arenas (page-locked host arrays for HOST, device tensors
    for DEVICE; the output filled with the sentinel) and the oracle's output.  Building it runs the twins over its
    packets, so the calls of a test are built in submission order."""

    def __init__(self, ctx, rng, items, entry=SPECTRUM, fmt=F32P, memory=HOST, expect=((), ()), chunks=None, pinned=True):
        self.items, self.entry, self.fmt, self.memory, self.expect, self.chunks = items, entry, fmt, memory, expect, chunks
        residue, planar = entry == RESIDUE, fmt in (F32P, I16P)
        coeffs, dense, kinds, ys = [], [], [], []
        self.wants, self.chains, self.ticket = [], [], None
        coff = ooff = rows = 0
        for tw, (modes, prev, nxt) in items:
            parts, steady, c0 = [], 0, coff
            for i, m in enumerate(int(x) for x in modes):
                n2 = tw.n2(m)
                if residue:
                    x = (rng.standard_normal((tw.C, n2)) * rng.integers(0, 2, (tw.C, n2))).astype(np.float32)
                    fl = [None if r < 0.1 else rng.random(n2).astype(np.float32) if r < 0.2 else
                          random_floor1_y(rng, FLOOR[0], len(FLOOR[1])) for r in rng.random(tw.C)]
                    k, y, d = L.DecodedPacket(m, x, fl).pack()
                    kinds.append(k)
                    ys.append(y)
                    dense.append(np.zeros_like(x) if d is None else d)
                    rc, o = tw.ref.packet(m, int(prev[i]), int(nxt[i]), x, fl)
                else:
                    x = (rng.standard_normal((tw.C, n2)) * 0.1).astype(np.float32)
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
            ooff += tw.C * stride + 4 if planar else (tw.C * steady + 3) // 4 * 4 + 4
            rows += len(modes)
        alloc = ctx.host_alloc if pinned else (lambda shape, dt: np.empty(shape, dt))

        def host(a):
            out = alloc(a.shape, a.dtype)
            out[...] = a
            return out
        self.total = ooff
        self.pcm = fill_guard(alloc(self.total, np.float32 if fmt in (F32P, F32I) else np.int16))
        self.coeffs = host(np.concatenate(coeffs))
        self.kw = {}
        if residue:
            self.kinds, self.ys = host(np.concatenate(kinds)), host(np.concatenate(ys))
            self.dense = host(np.concatenate([d.ravel() for d in dense]))
            self.kw = dict(floor_kind=self.kinds, floor1_y=self.ys, dense_floor=self.dense)
        if memory == DEVICE:
            self.dev = {"coeffs": torch.from_numpy(self.coeffs.copy()).cuda(), "pcm": torch.from_numpy(self.pcm.copy()).cuda()}
            if residue:
                self.dev["dense"] = torch.from_numpy(self.dense.copy()).cuda()
                self.kw["dense_floor"] = self.dev["dense"].data_ptr()

    def arenas(self):
        if self.memory == DEVICE:
            return self.dev["coeffs"].data_ptr(), self.dev["pcm"].data_ptr()
        return self.coeffs, self.pcm

    def submit(self, ctx):
        ran, not_ran = self.expect
        with environ({"LWB_E2E_CHUNKS": str(self.chunks)} if self.chunks else None):
            with expect_kernels(ctx, ran=ran, not_ran=not_ran):
                self.ticket = ctx.submit_chains(self.chains, self.entry, self.memory, *self.arenas(), self.fmt, **self.kw)
        return self.ticket

    def decode(self, ctx):
        """The same batch through the synchronous entry point."""
        ran, not_ran = self.expect
        with expect_kernels(ctx, ran=ran, not_ran=not_ran):
            L.decode_chains(ctx, self.chains, self.entry, self.memory, *self.arenas(), self.fmt, **self.kw)

    def untouched(self):
        """The PCM arena holds nothing but the sentinel."""
        pcm = self.dev["pcm"].cpu().numpy() if self.memory == DEVICE else self.pcm
        return bool(np.all(pcm.view(np.uint32 if pcm.dtype == np.float32 else np.uint16) == fill_guard(pcm.copy()).view(
            np.uint32 if pcm.dtype == np.float32 else np.uint16)))

    def check(self, oracle, what):
        """After the call's work has run: results, the whole output arena."""
        if self.ticket is not None:
            assert self.ticket.done(), (what, "ticket not done")
            self.ticket.wait()
        pcm = self.dev["pcm"].cpu().numpy() if self.memory == DEVICE else self.pcm
        for i, c in enumerate(self.chains):
            assert (c.status, c.packets_done, c.n_samples) == (0, len(c.modes), self.wants[i].shape[1]), \
                (what, i, c.status, c.packets_done, c.n_samples)
        check_arena(oracle, pcm, self.chains, self.wants, [tw.C for tw, _ in self.items], self.fmt, what)


def check_arena(oracle, pcm, chains, wants, channels, fmt, what):
    """A whole output arena against the oracle: chains give the layout, wants [C][n] per chain; nothing else written."""
    planar = fmt in (F32P, I16P)
    for i, (c, want) in enumerate(zip(chains, wants)):
        C, n = channels[i], want.shape[1]
        if planar:
            got = np.stack([pcm[c.out_offset + k * c.out_stride:c.out_offset + k * c.out_stride + n] for k in range(C)])
        else:
            got = pcm[c.out_offset:c.out_offset + C * n].reshape(n, C).T
        if fmt in (F32P, F32I):
            assert bits_equal(got, want), (what, i, mismatch_report(got, want))
        else:
            assert np.array_equal(got, oracle.quantise_i16(want)), (what, i)
    assert_contained(pcm, write_set(chains, lambda i: channels[i], fmt), what)


def check_states(tws, what):
    for tw in tws:
        tw.check_state(what)


# what each batch path launches (host memory)
MIXED = {"k_long_s", "k_short_g"}
PATHS = {
    "long": ("mixed", "long", 8, SPECTRUM, F32P, ({"k_long"}, ALL_KERNELS - {"k_long"})),     # (one launch per chunk)
    "residue_long": ("mixed", "long", 8, RESIDUE, F32P, (FRONT | {"k_long"}, ALL_KERNELS - FRONT - {"k_long"})),
    "mixed": ("mixed", "mixed", 16, SPECTRUM, F32P, (MIXED, ALL_KERNELS - MIXED - MIXED_EXTRA)),
    "residue_mixed": ("mixed", "mixed", 16, RESIDUE, I16P, (FRONT | {"k_long_s"}, ALL_KERNELS - FRONT - MIXED - MIXED_EXTRA)),
    "mid": ("mid", "uniform", 8, SPECTRUM, F32P, ({"k_mid"}, ALL_KERNELS - {"k_mid"})),
    "residue_mid": ("mid", "uniform", 8, RESIDUE, I16P, (FRONT | {"k_mid"}, ALL_KERNELS - FRONT - {"k_mid"})),
    "short": ("short", "uniform", 16, SPECTRUM, F32P, ({"k_short"}, ALL_KERNELS - {"k_short"})),
    "chain": ("mixed", "mixed", 12, SPECTRUM, F32I, ({"k_chain"}, ALL_KERNELS - {"k_chain"})),
    "generic": ("wide", "mixed", 6, SPECTRUM, F32P, (GENERIC - {"k_prologue"}, ALL_KERNELS - GENERIC)),
}


def path_calls(ctx, rng, tws, path, n_calls, chunks, memory=HOST):
    kind, seq_kind, P, entry, fmt, expect = PATHS[path]
    return [AsyncCall(ctx, rng, [(tw, seq(rng, seq_kind, P)) for tw in tws], entry, fmt, memory, expect, chunks)
            for _ in range(n_calls)]


def submit_gated(ctx, gate, calls, what, must_return=3):
    """Submits the calls behind the gate (None: ungated).  After each submit that returns while the gate is closed, no
    ticket so far is done and no PCM has landed; the first `must_return` submits must return while it is closed
    (see must_return)."""
    torch.cuda.synchronize()
    if gate:
        gate.close()
    for k, call in enumerate(calls):
        call.submit(ctx)
        if not gate:
            continue
        busy = not any(c.ticket.done() for c in calls[:k + 1])
        clean = all(c.untouched() for c in calls[:k + 1] if c.memory == HOST)
        if not gate.opened.query():             # both observations were made behind the closed gate
            assert busy, (what, k, "a ticket completed behind the closed gate")
            assert clean, (what, k, "PCM landed behind the closed gate")
        if k < must_return:
            gate.assert_closed((what, "submit", k))


# ------------------------------------------------------------------------------------------------
# every path, three or four deep, with the same streams in consecutive submits
# ------------------------------------------------------------------------------------------------
def must_return(path, chunks):
    """Submits of `path` that return behind the gate, from the blocking points the header lists.  The staging ring has
    three slots, all completed after the warm-up.  Paths that stage once per submit (k_long, the one-pass and segmented
    schedules, k_mid's spectrum entry, k_chain, and the four-kernel path, whose 6-packet batches take one round)
    therefore return all three.  The residue entries of k_mid and k_long stage twice per submit, at any chunk count:
    their packet list on the compute stream, then all their runs at once.  The second submit takes the first one's
    packet list slot, which completes behind the gate."""
    return 1 if path in ("residue_long", "residue_mid") else 3


@pytest.mark.parametrize("chunks", [1, 3, 64])
@pytest.mark.parametrize("path", list(PATHS))
def test_every_path_submitted_deep(ctx, oracle, path, chunks):
    """Three host-memory submits over the same streams (the third reuses the first's arena set while the first is still
    queued), then one more once the gate has opened; each chain and each final state against the oracle."""
    sus = setups(ctx)
    gate = Gate(ctx)
    S = 64 if chunks == 64 else 8
    for gated in (False, True):
        rng = np.random.default_rng(10 + chunks)
        tws = twins(oracle, sus, PATHS[path][0], S)
        calls = path_calls(ctx, rng, tws, path, 4, chunks)
        what = (path, chunks, "gated" if gated else "warm-up")
        submit_gated(ctx, gate if gated else None, calls[:3], what, must_return(path, chunks))
        calls[3].submit(ctx)
        calls[3].ticket.wait()
        for k, call in enumerate(calls):
            call.check(oracle, (what, k))
        check_states(tws, what)


def test_vq_long_submitted_deep(ctx, oracle):
    """LWB_ENTRY_VQ k_long batches (VQ runs and entries in page-locked host arrays), four deep behind the gate over the
    same streams: the device accumulates each packet's residue from its VQ records."""
    rng = np.random.default_rng(77)
    S, P, K = 4, 6, 4          # (both passes decode the same packets, K even: each set sees the same batches, none grows)
    spec = vp.StreamSpec(rng, channels=2, residue_types=[1])
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    assert hdr.vq_capable()
    su = hdr.make_setup(ctx)
    gate = Gate(ctx)
    infos, pkts = [[] for _ in range(S)], [[] for _ in range(S)]
    for s in range(S):
        for mode, prev, nxt in consistent_modes(spec, rng, P * K, p_short=0.0):
            pk, info = spec.audio_packet(mode, prev, nxt, p_unused=0.1)
            pkts[s].append(pk)
            infos[s].append(info)
    for gated in (False, True):
        refs = [oracle_pcm(oracle, spec, infos[s]) for s in range(S)]
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        stride = P * (1 << spec.bs1) // 2
        calls = []
        for k in range(K):
            kinds, ys, runs, ents, roffs, eoffs, chains = [], [], [], [], [0], [0], []
            for s in range(S):
                modes, prevs, nexts = [], [], []
                for pk in pkts[s][k * P:(k + 1) * P]:
                    dense = hdr.decode_packet(pk)
                    dp, rr, ee = hdr.decode_packet_vq(pk)
                    kd, y, _ = dense.pack()
                    kinds.append(kd)
                    ys.append(y)
                    runs.append(rr)
                    ents.append(ee)
                    roffs.append(roffs[-1] + len(rr))
                    eoffs.append(eoffs[-1] + len(ee))
                    modes.append(dp.mode_number); prevs.append(dp.prev_window_flag); nexts.append(dp.next_window_flag)
                chains.append(L.ChainSpec(pwrs[s], np.array(modes, np.uint8), np.array(prevs, np.uint8),
                                          np.array(nexts, np.uint8), packet_index=s * P, coeff_offset=s * 2 * stride,
                                          out_offset=s * 2 * stride, out_stride=stride))

            def pinned(a):
                out = ctx.host_alloc(a.shape, a.dtype)
                out[...] = a
                return out
            arrays = [pinned(x) for x in (np.concatenate(kinds), np.concatenate(ys), np.concatenate(runs),
                                          np.array(roffs, np.uint64), np.concatenate(ents), np.array(eoffs, np.uint64))]
            pcm = fill_guard(ctx.host_alloc(S * 2 * stride, np.float32))
            calls.append((chains, arrays, pcm))
        # the previous pass's page-locked arrays go now, not behind the gate: cudaFreeHost waits for the device
        kd = y = rr = ro = ee = eo = arrays = pcm = tickets = None
        torch.cuda.synchronize()
        if gated:
            gate.close()
        tickets = []
        for chains, (kd, y, rr, ro, ee, eo), pcm in calls:
            with expect_kernels(ctx, ran={"k_floor1_segments": 1, "k_prologue_fused": 1, "k_long": 1},
                                not_ran=ALL_KERNELS - FRONT - {"k_long"}):
                tickets.append(ctx.submit_chains(chains, cabi.ENTRY_VQ, HOST, None, pcm, F32P, floor_kind=kd, floor1_y=y,
                                                 vq=(rr, ro, ee, eo)))
            if gated and len(tickets) == 1:     # (the second waits for the first's packet-list staging: ring wrap)
                assert not tickets[0].done() and np.all(pcm.view(np.uint32) == fill_guard(pcm.copy()).view(np.uint32))
                gate.assert_closed("VQ")
        tickets[-1].wait()
        for k, (chains, _, pcm) in enumerate(calls):
            assert tickets[k].done()
            tickets[k].wait()                   # (copies the chain results)
            for s in range(S):
                want = np.concatenate(refs[s][0][k * P:(k + 1) * P], axis=1)
                n = want.shape[1]
                assert (chains[s].status, chains[s].n_samples) == (0, n), (k, s)
                got = pcm[s * 2 * stride:(s + 1) * 2 * stride].reshape(2, stride)[:, :n]
                assert bits_equal(got, want), (gated, k, s, mismatch_report(got, want))
            assert_contained(pcm, write_set(chains, lambda i: 2, F32P), ("VQ", gated, k))
        for s in range(S):
            assert bits_equal(pwrs[s].data(), refs[s][1].pwr.data()), ("VQ state", s)
            pwrs[s].close()


# ------------------------------------------------------------------------------------------------
# tickets
# ------------------------------------------------------------------------------------------------
def test_ticket_order_and_repeated_waits(ctx, oracle):
    """Tickets are issued in order from 1 up; waiting on the last makes every earlier one query done; waiting again on
    an old ticket returns at once; ticket 0 and tickets never issued are refused."""
    sus = setups(ctx)
    gate = Gate(ctx)
    for gated in (False, True):
        rng = np.random.default_rng(20)
        tws = twins(oracle, sus, "mixed", 8)
        calls = path_calls(ctx, rng, tws, "long", 3, None)
        submit_gated(ctx, gate if gated else None, calls, "tickets")
        ids = [c.ticket.id for c in calls]
        assert ids[0] >= 1 and ids == list(range(ids[0], ids[0] + 3))
        lib, d = cabi.lib(), ctypes.c_int()
        assert lib.lwb_ticket_wait(ctx._h, ids[-1]) == 0
        for t in ids:
            assert lib.lwb_ticket_query(ctx._h, t, ctypes.byref(d)) == 0 and d.value == 1, t
        assert lib.lwb_ticket_wait(ctx._h, ids[0]) == 0          # again, and older than the newest: at once
        assert lib.lwb_ticket_wait(ctx._h, 1) == 0
        assert lib.lwb_ticket_query(ctx._h, 0, ctypes.byref(d)) == cabi.ERR_INVALID
        assert lib.lwb_ticket_wait(ctx._h, 0) == cabi.ERR_INVALID
        assert lib.lwb_ticket_wait(ctx._h, ids[-1] + 1) == cabi.ERR_INVALID
        for k, call in enumerate(calls):
            call.check(oracle, ("tickets", gated, k))
        check_states(tws, ("tickets", gated))


def test_completion_means_the_pcm_has_landed(ctx, oracle):
    """One host submit of 512 streams in one chunk, so that its D2H of 32 MiB comes last: the moment wait() returns the
    last sample of the last chain is in the page-locked arena, and so it is the moment done() first answers 1."""
    sus = setups(ctx)
    rng = np.random.default_rng(25)
    tws = twins(oracle, sus, "mixed", 512)
    for how in ("wait", "poll", "wait", "poll"):
        call = path_calls(ctx, rng, tws, "long", 1, 1)[0]
        c = call.chains[-1]
        last = c.out_offset + (tws[-1].C - 1) * c.out_stride + call.wants[-1].shape[1] - 1
        bits = call.pcm.view(np.uint32)
        torch.cuda.synchronize()
        t = call.submit(ctx)
        if how == "wait":
            assert cabi.lib().lwb_ticket_wait(ctx._h, t.id) == 0
        else:
            d = ctypes.c_int()
            while cabi.lib().lwb_ticket_query(ctx._h, t.id, ctypes.byref(d)) == 0 and not d.value:
                pass
        landed = int(bits[last])                 # read at once
        assert landed != F32_GUARD, (how, "the last sample had not landed")
        call.check(oracle, ("landed", how))
    check_states(tws, "landed")


# ------------------------------------------------------------------------------------------------
# mixing entry points
# ------------------------------------------------------------------------------------------------
def test_mixing_entry_points(ctx, oracle):
    """Host submits with, between them on the same streams, a device-memory submit, a synchronous host-memory
    decode_chains, and a prepared device batch run three times: the first run plans and captures it, the next two
    replay the capture (no stream changes shape and no arena grows in the gated pass), each between two host submits.
    Each run is fed its own inputs and snapshotted by copies on the context's stream; everything against the oracle in
    submission order."""
    sus = setups(ctx)
    for gated in (False, True):
        gate = Gate(ctx)
        rng = np.random.default_rng(30)
        tws = twins(oracle, sus, "mixed", 8)
        h1 = path_calls(ctx, rng, tws, "long", 1, None)[0]
        d1 = path_calls(ctx, rng, tws, "long", 1, None, memory=DEVICE)[0]
        h2 = path_calls(ctx, rng, tws, "long", 1, None)[0]
        sync = path_calls(ctx, rng, tws, "residue_mixed", 1, None)[0]
        pseq = [(tw, seq(rng, "long", 8)) for tw in tws]          # one layout for every run of the prepared batch
        host, plan_runs = [], []
        for _ in range(3):
            host.append(path_calls(ctx, rng, tws, "long", 1, None)[0])
            plan_runs.append(AsyncCall(ctx, rng, pseq, SPECTRUM, F32P, DEVICE, ({"k_long": 1}, ALL_KERNELS - {"k_long"})))
        last = path_calls(ctx, rng, tws, "residue_long", 1, None)[0]
        p0 = plan_runs[0]
        batch = L.Batch(ctx, p0.chains, SPECTRUM, DEVICE, *p0.arenas(), F32P)
        snaps = [torch.empty_like(p0.dev["pcm"]) for _ in plan_runs]
        torch.cuda.synchronize()
        if gated:
            gate.close()
        h1.submit(ctx)
        d1.submit(ctx)
        h2.submit(ctx)
        if gated:
            assert not h1.ticket.done() and h1.untouched() and h2.untouched()
            gate.assert_closed("mixing")
        sync.decode(ctx)                         # waits for everything before it
        assert h1.ticket.done() and d1.ticket.done() and h2.ticket.done()
        for k, run in enumerate(plan_runs):
            host[k].submit(ctx)
            with gate.on_stream():
                p0.dev["coeffs"].copy_(run.dev["coeffs"])
                p0.dev["pcm"].copy_(run.dev["pcm"])     # (the sentinel)
            ran, not_ran = run.expect
            with expect_kernels(ctx, ran=ran, not_ran=not_ran):
                batch.run()
            with gate.on_stream():
                snaps[k].copy_(p0.dev["pcm"])
        last.submit(ctx)
        last.ticket.wait()
        torch.cuda.synchronize()
        results = [(c.n_samples, c.packets_done, c.status) for c in batch.collect()]
        for run, snap in zip(plan_runs, snaps):
            run.dev["pcm"] = snap
            for c, r in zip(run.chains, results):
                c.n_samples, c.packets_done, c.status = r
        for k, call in enumerate([h1, d1, h2, sync] + [x for pair in zip(host, plan_runs) for x in pair] + [last]):
            call.check(oracle, ("mixing", gated, k))
        check_states(tws, ("mixing", gated))
        batch.close()


# ------------------------------------------------------------------------------------------------
# growth
# ------------------------------------------------------------------------------------------------
def test_growth_while_the_set_is_in_flight(oracle):
    """On a fresh context whose shared scratch (k_long runs, staging ring) large device batches have grown, and whose
    host sets are still empty: a small host submit (set 0) behind the gate, then a large one, which takes set 1 (a first
    allocation, nothing to free) and returns at once, then another large one, whose set 0 must grow while the first
    submit still holds it: it waits for that ticket, and every output is right."""
    ctx = L.Context(0)
    try:
        sus = setups(ctx)
        gate = Gate(ctx)
        rng = np.random.default_rng(40)
        big_tws, small_tws = twins(oracle, sus, "mixed", 64), twins(oracle, sus, "mixed", 8)
        for call in path_calls(ctx, rng, big_tws, "long", 4, None, memory=DEVICE):
            call.submit(ctx)
            call.ticket.wait()
            call.check(oracle, "device warm-up")
        small = path_calls(ctx, rng, small_tws, "long", 1, None)[0]
        big1, big2 = path_calls(ctx, rng, big_tws, "long", 2, None)
        torch.cuda.synchronize()
        gate.close()
        small.submit(ctx)
        big1.submit(ctx)
        assert small.untouched() and not small.ticket.done()
        gate.assert_closed("growth of the free set")
        big2.submit(ctx)                        # set 0 grows behind small's ticket
        assert small.ticket.done()
        big2.ticket.wait()
        for k, call in enumerate((small, big1, big2)):
            call.check(oracle, ("growth", k))
        check_states(big_tws + small_tws, "growth")
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------
# refusal
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pageable", ["coeffs", "pcm", "floor_kind", "floor1_y", "dense_floor"])
def test_pageable_arrays_are_refused(ctx, oracle, pageable):
    """A host-memory submit with one pageable array: LWB_ERR_INVALID, and the chain results, the stream states and the
    PCM arena are as they were.  The same batch from page-locked arrays then decodes right."""
    sus = setups(ctx)
    rng = np.random.default_rng(50)
    tws = twins(oracle, sus, "mixed", 4)
    first = path_calls(ctx, rng, tws, "residue_long", 1, None)[0]
    first.submit(ctx)
    first.ticket.wait()
    first.check(oracle, "first")
    call = path_calls(ctx, rng, tws, "residue_long", 1, None)[0]
    states = [tw.pwr.data() for tw in tws]
    for c in call.chains:
        c.n_samples, c.packets_done, c.status = 7, 7, 7
    arr, io = L.api._marshal(call.chains, RESIDUE, HOST, call.coeffs, call.pcm, F32P, call.kinds, call.ys, call.dense,
                             HOST, None)
    for c in range(len(call.chains)):
        arr[c].n_samples, arr[c].packets_done, arr[c].status = 7, 7, 7
    src = {"coeffs": call.coeffs, "pcm": call.pcm, "floor_kind": call.kinds, "floor1_y": call.ys, "dense_floor": call.dense}
    plain = src[pageable].copy()                # ordinary, pageable numpy memory
    setattr(io, pageable, plain.ctypes.data)
    import ctypes
    t = ctypes.c_uint64()
    launches = ctx.launch_count
    rc = cabi.lib().lwb_submit_chains(ctx._h, arr, len(call.chains), ctypes.byref(io), ctypes.byref(t))
    assert rc == cabi.ERR_INVALID, rc
    assert pageable in cabi.lib().lwb_last_error(ctx._h).decode()
    assert ctx.launch_count == launches
    assert all((arr[i].n_samples, arr[i].packets_done, arr[i].status) == (7, 7, 7) for i in range(len(call.chains)))
    ctx.synchronize()
    for tw, s in zip(tws, states):
        assert bits_equal(tw.pwr.data(), s)
    assert call.untouched() and (pageable != "pcm" or np.all(plain.view(np.uint32) == fill_guard(plain.copy()).view(np.uint32)))
    call.submit(ctx)
    call.ticket.wait()
    call.check(oracle, ("after refusal", pageable))
    check_states(tws, ("after refusal", pageable))


# ------------------------------------------------------------------------------------------------
# two contexts on two host threads
# ------------------------------------------------------------------------------------------------
def test_two_contexts_submitting_on_two_threads(oracle):
    """Each of two contexts submits host batches of three paths, three deep, from its own host thread, at once (the C
    calls release the GIL), then waits for its last ticket.  Built and checked on the main thread."""
    ctxs = [L.Context(0), L.Context(0)]
    try:
        work = []
        for i, c in enumerate(ctxs):
            sus = setups(c)
            rng = np.random.default_rng(60 + i)
            tws = twins(oracle, sus, "mixed", 16)
            calls = []
            for path in ("residue_long", "residue_mixed", "long", "chain", "residue_long", "mixed"):
                calls += path_calls(c, rng, tws, path, 1, None)
            work.append((calls, tws))
        errors = []
        start = threading.Barrier(2)

        def worker(i):
            try:
                calls, _ = work[i]
                start.wait()
                for call in calls:
                    call.submit(ctxs[i])
                calls[-1].ticket.wait()
            except BaseException as e:          # re-raised on the main thread
                errors.append(e)
        threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        for i, (calls, tws) in enumerate(work):
            for k, call in enumerate(calls):
                call.check(oracle, ("thread", i, k))
            check_states(tws, ("thread", i))
    finally:
        for c in ctxs:
            c.close()


# ------------------------------------------------------------------------------------------------
# teardown with tickets in flight
# ------------------------------------------------------------------------------------------------
def test_teardown_with_tickets_in_flight(oracle):
    """Behind the gate: three host submits, then a stream of the last batch is closed and then the context itself, while
    every ticket is still in flight.  Both return after the work, and the PCM in the page-locked arenas is right."""
    ctx = L.Context(0)
    sus = setups(ctx)
    gate = Gate(ctx)
    rng = np.random.default_rng(70)
    for step in ("warm-up", "stream", "context"):
        tws = twins(oracle, sus, "mixed", 8)
        calls = path_calls(ctx, rng, tws, "long", 3, None)
        submit_gated(ctx, None if step == "warm-up" else gate, calls, ("teardown", step))
        if step == "warm-up":
            calls[-1].ticket.wait()
        elif step == "stream":
            tws[0].pwr.close()                  # lwb_stream_destroy: returns after the kernels and the copies
            assert gate.opened.query() and not any(c.untouched() for c in calls)
            tws = tws[1:]
        else:
            for c in calls:                     # (results were written before submit returned)
                L.api._collect(c.chains, c.ticket._arr)
            ctx.close()                         # lwb_ctx_destroy (streams and setups first) with every ticket in flight
            for c in calls:
                c.ticket = None                 # (the context is gone: the PCM alone tells)
        for k, call in enumerate(calls):
            call.check(oracle, ("teardown", step, k))
        if step != "context":
            check_states(tws, ("teardown", step))

"""Output windows (lwb_stream_set_window) on chains that stop, and the window calls around batches.

A stopped chain changes everything a window is clipped from: its samples are those of the decoded packets only, the
overlap guard leaves the stream empty (so its next packet produces 0 samples), and the window's counters must move by
the samples of the decoded packets.  Each case runs the stop kinds of test_chain_errors_gpu.py -- bad mode numbers at
packet 0, in the middle and last, the guard in the middle, carried across batches and on an imported state, and a bad
mode number behind a long block -- on windowed streams and on their unwindowed twins, over the same packets (from the
stop on poisoned with NaN), in three batches: the one that stops (the second, for the carried guard), the batches after
it.  Every stream's window clips the stopped batch: it ends inside the decoded packets, exactly at the stop, starts
after it (the chain writes nothing), or spans into the next batches.  Per batch:
  * the twin's chain results, PCM and states equal the oracle's (Call.check), on the kernels pins() names;
  * the windowed chain reports the twin's status and packets_done, and n_samples what its window lets through;
  * the windowed arena holds exactly the twin's samples sliced to the windows, and the sentinel everywhere else;
  * the windowed batch launches the twin's kernels plus one k_row_copy per chunk that moves samples -- none for a
    chain that stops at packet 0 or whose window starts after its last decoded sample;
  * the window left on each stream (PreviousWindowRight.window) and its state equal what the decoded packets give."""
import numpy as np
import pytest
import torch

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from helpers import bits_equal, environ, expect_kernels, fill_guard, launches_are_attributed, make_setup, mismatch_report
from test_chain_errors_gpu import ALL_STOPS, CLEAN, UNIFORM, Call, Stream, pins
from test_stream_windows_gpu import FLOOR, PATHS, Arena, Batch, Stream as WinStream, check_batch, decode

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

F32P, F32I, I16P = cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_PLANAR
SPECTRUM, RESIDUE, HOST, DEVICE = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE, cabi.MEM_HOST, cabi.MEM_DEVICE
WINDOWS = ("inside", "at_stop", "after", "span")

# Each batch path of test_stream_windows_gpu.PATHS, as stopped batches are routed (test_chain_errors_gpu.pins): a bad
# mode number keeps a batch off k_long and k_mid, so the 2048-point shapes take the segmented path and k_mid's shapes
# (uniform 1024- and 512-point setups here) the chain kernel, until the batches after the stop go back to k_mid.
# path: (blocksize_0, blocksize_1, stream kinds, format, (pins of the three batches))
STOP_PATHS = {
    "k_long": (8, 11, ALL_STOPS, F32P, ("mixed",) * 3),
    "k_mid_1024": (10, 10, UNIFORM, I16P, ("chain", "mid", "mid")),
    "k_mid_512": (9, 9, UNIFORM, F32P, ("chain", "mid", "mid")),
    "one_pass": (8, 11, CLEAN, F32P, ("pass",) * 3),
    "rounds": (8, 11, ALL_STOPS, F32P, ("rounds",) * 3),
    "k_chain": (8, 11, ALL_STOPS, F32I, ("chain",) * 3),
    "four_kernel": (8, 11, ALL_STOPS, F32P, ("generic",) * 3),
}
assert set(STOP_PATHS) == set(PATHS)


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


class Windowed:
    """The windowed twin of a Stream: its own device stream, from the same state, and the window it runs under."""

    def __init__(self, st, variant):
        self.st, self.variant = st, variant
        self.pwr = L.PreviousWindowRight(st.su)
        if not st.pwr.is_empty():
            self.pwr.set_data(st.pwr.data())
        self.window, self.pos = None, 0       # (skip, limit or None); samples produced since it was set

    def set(self, n):
        """Sets the window of `variant` over a batch that produces n samples (its decoded packets only)."""
        s = min(7, n)
        self.window = {"inside": (n // 3, n // 3), "at_stop": (s, n - s), "after": (n + 50, None),
                       "span": (n // 2, 3000)}[self.variant]
        self.pos = 0
        self.pwr.set_window(*self.window)

    def expect(self, n):
        """[a, b) of the next n produced samples that the window writes."""
        if self.window is None:
            return 0, n
        skip, limit = self.window
        end = np.inf if limit is None else skip + limit
        a = int(min(max(skip - self.pos, 0), n))
        return a, int(max(a, min(end - self.pos, n)))

    def left(self):
        skip, limit = self.window
        return max(skip - self.pos, 0), None if limit is None else max(0, min(limit, skip + limit - self.pos))


def windowed_chains(call, wins):
    return [L.ChainSpec(w.pwr, c.modes, c.prev, c.next, coeff_offset=c.coeff_offset, packet_index=c.packet_index,
                        out_offset=c.out_offset, out_stride=c.out_stride) for c, w in zip(call.chains, wins)]


def expected_arena(call, twin_pcm, twin_chains, spans):
    """The twin's arena with every chain's output cut to [a, b) of its samples and moved to its start; sentinel elsewhere."""
    want = fill_guard(np.empty_like(twin_pcm))
    C = call.C
    for c, (a, b) in zip(twin_chains, spans):
        o, sd = int(c.out_offset), int(c.out_stride)
        if call.fmt in (F32P, I16P):
            for k in range(C):
                want[o + k * sd:o + k * sd + b - a] = twin_pcm[o + k * sd + a:o + k * sd + b]
        else:
            want[o:o + (b - a) * C] = twin_pcm[o + a * C:o + b * C]
    return want


def row_copies(moves, chunks):
    n = len(moves)
    return sum(any(moves[n * q // chunks:n * (q + 1) // chunks]) for q in range(chunks))


def run_stops(ctx, oracle, bs0, bs1, kinds, entry, fmt, memory, paths, env=None, chunks=1, seed=0):
    rng = np.random.default_rng(seed)
    su = make_setup(ctx, 2, bs0, bs1, modes=[(0, 0), (1, 0)], mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}],
                    floors=[FLOOR])
    streams = [Stream(oracle, su, kind, bs0 != bs1, rng) for kind in kinds for _ in WINDOWS]
    wins = [Windowed(st, WINDOWS[i % len(WINDOWS)]) for i, st in enumerate(streams)]
    env = dict(env or {}, **({"LWB_E2E_CHUNKS": str(chunks)} if chunks > 1 else {}))
    bits = np.uint32 if fmt == F32P or fmt == F32I else np.uint16
    with environ(env):
        for batch, path in enumerate(paths):
            if batch == 2:
                for st in streams:          # after its stop in the second batch the carried stream is an ordinary one
                    st.kind = "ok" if st.kind == "carry" else st.kind
            call = Call(rng, streams, min(batch, 1), entry, fmt, memory)
            wants = call.expect()
            if batch == 0:
                for w, (_, _, want) in zip(wins, wants):
                    w.set(want.shape[1])    # from the samples of the decoded packets of the first batch
            ran, not_ran, segmented = pins(path, entry)
            with expect_kernels(ctx, ran=ran, not_ran=not_ran) as kfull:
                call.submit(ctx)
            ctx.synchronize()
            call.check(oracle, call.chains, wants, ("twin", batch))
            if segmented:
                assert any(kfull[k] for k in ("k_long", "k_long_s", "k_short", "k_short_g")), kfull
            twin_pcm = np.array(call.output())
            call.reset_pcm()
            if memory == DEVICE:
                torch.cuda.synchronize()
            wch = windowed_chains(call, wins)
            spans = [w.expect(int(c.n_samples)) for w, c in zip(wins, call.chains)]
            saved = call.chains
            call.chains = wch
            with expect_kernels(ctx) as kwin:
                call.submit(ctx)
            ctx.synchronize()
            call.chains = saved
            for w, c, fc, (a, b) in zip(wins, wch, call.chains, spans):
                what = (batch, w.st.kind, w.variant, w.window, w.pos)
                assert (c.status, c.packets_done, c.n_samples) == (fc.status, fc.packets_done, b - a), \
                    what + ((c.status, c.packets_done, c.n_samples), (fc.status, fc.packets_done, fc.n_samples))
                w.pos += int(fc.n_samples)
                if w.window is not None:
                    assert w.pwr.window == w.left(), what + (w.pwr.window, w.left())
                assert w.pwr.is_empty() == w.st.pwr.is_empty() and len(w.pwr) == len(w.st.pwr), what
                if not w.pwr.is_empty():
                    assert bits_equal(w.pwr.data(), w.st.pwr.data()), what
            got = np.array(call.output()).view(bits)
            want = expected_arena(call, twin_pcm, call.chains, spans).view(bits)
            bad = np.nonzero(got != want)[0]
            assert not bad.size, f"batch {batch}: {bad.size} elements differ; first at {bad[:5]}: got {got[bad[:5]]} want {want[bad[:5]]}"
            clipped = [(a, b) != (0, int(c.n_samples)) for c, (a, b) in zip(call.chains, spans)]
            moves = [cl and b > a for cl, (a, b) in zip(clipped, spans)]
            want_k = dict(kfull)
            want_k["k_row_copy"] += row_copies(moves, chunks)
            assert kwin == want_k, (batch, dict((k, v) for k, v in kfull.items() if v), dict((k, v) for k, v in kwin.items() if v))


@pytest.mark.parametrize("memory", [DEVICE, HOST], ids=["device", "host"])
@pytest.mark.parametrize("entry", [SPECTRUM, RESIDUE], ids=["spectrum", "residue"])
@pytest.mark.parametrize("path", list(STOP_PATHS))
def test_windows_on_stopped_chains(ctx, oracle, path, entry, memory):
    bs0, bs1, kinds, fmt, paths = STOP_PATHS[path]
    env = PATHS[path][4]
    run_stops(ctx, oracle, bs0, bs1, kinds, entry, fmt, memory, paths, env=env, seed=sum(map(ord, path)) + 7 * entry + memory)


def test_windows_on_stopped_chains_in_chunked_host_batches(ctx, oracle):
    """A host-memory batch in three chunks (LWB_E2E_CHUNKS=3): one k_row_copy per chunk that moves samples."""
    run_stops(ctx, oracle, 8, 11, ALL_STOPS, RESIDUE, I16P, HOST, ("mixed",) * 3, chunks=3, seed=11)


# ---------------------------------------------------------------------------------------------------------------------
# the window calls between batches
# ---------------------------------------------------------------------------------------------------------------------
def k_long_streams(ctx, oracle, path, n, windows, packets):
    C, bs0, bs1, p_short, _, _ = PATHS[path]
    su = make_setup(ctx, C, bs0, bs1, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}], floors=[FLOOR])
    rng = np.random.default_rng(n)
    return [WinStream(su, oracle, C, bs0, bs1, (rng.random(packets) >= p_short).astype(np.uint8), w) for w in windows], rng


def one_batch(ctx, rng, streams, path, k, memory=DEVICE):
    """Decodes the next k packets of every stream, windowed and twin, and checks them with check_batch.  Returns the
    batch, the written counts, the twin's PCM per stream ([C][n] f32) and the windowed arena."""
    b = Batch(rng, streams, k, SPECTRUM, F32P)
    fa, wa = Arena(ctx, b.full_elems, F32P, memory), Arena(ctx, b.win_elems, F32P, memory)
    fch, wch = b.chains("full", b.full_lay), b.chains("win", b.win_lay)
    with environ(PATHS[path][4]):
        with expect_kernels(ctx) as kfull:
            decode(ctx, b, "full", memory, fa, fch)
        decode(ctx, b, "win", memory, wa, wch)
    assert kfull[PATHS[path][5]] > 0, kfull
    fbuf, wbuf = fa.read(), wa.read()
    full = [fbuf.view(np.float32)[o:o + 2 * n].reshape(2, n) for (o, n) in b.full_lay]
    return b, check_batch(b, fch, wch, fbuf, wbuf), full, wbuf


@pytest.mark.parametrize("path", ["k_long", "one_pass"])
def test_seek_between_batches(ctx, oracle, path):
    """reset() then set_window(skip) between batches: the next batch decodes from an empty state, and what the window
    writes is the oracle's decode from an empty state of the same packets, sliced."""
    streams, rng = k_long_streams(ctx, oracle, path, 31, [(0, None)] * 4, 8)
    one_batch(ctx, rng, streams, path, 4)
    skips = [0, 1, 700, 1500]
    for st, skip in zip(streams, skips):
        for p in (st.win, st.full):
            p.reset()
        st.ref.pwr = oracle.Pwr(st.C, st.bs1)            # the oracle seeks too: an empty state
        st.oracle_pcm, st.pos = [], 0
        st.window = (skip, None)
        st.win.set_window(skip)
    _, counts, full, _ = one_batch(ctx, rng, streams, path, 4)
    for st, skip, n, f in zip(streams, skips, counts, full):
        want = np.concatenate(st.oracle_pcm, axis=1)
        assert bits_equal(f, want), mismatch_report(f, want)
        assert n == max(want.shape[1] - skip, 0)
        assert st.win.window == (max(skip - want.shape[1], 0), None)


def test_clone_copies_the_remaining_window(ctx, oracle):
    """clone() takes the window as it stands (part used up) and the state; the clone, run over the same packets in
    another batch, writes the samples the original wrote."""
    streams, rng = k_long_streams(ctx, oracle, "k_long", 32, [(1500, 2500), (100, 50), (5000, None), (2100, 1)], 8)
    one_batch(ctx, rng, streams, "k_long", 3)
    for st in streams:
        st.clone = st.win.clone()
        assert st.clone.window == st.win.window and st.clone.window != st.window
        assert bits_equal(st.clone.data(), st.win.data())
    b, counts, _, wbuf = one_batch(ctx, rng, streams, "k_long", 3)
    ca = Arena(ctx, b.win_elems, F32P, DEVICE)
    cch = b.chains("clone", b.win_lay)
    decode(ctx, b, "clone", DEVICE, ca, cch)
    assert [c.n_samples for c in cch] == counts
    assert np.array_equal(ca.read(), wbuf)
    for st in streams:
        assert st.clone.window == st.win.window
        assert bits_equal(st.clone.data(), st.win.data())


def test_load_states_leaves_the_window(ctx, oracle):
    """save_states then load_states into streams that have windows: the windows stay as they were, and the next batch
    writes what they let through."""
    streams, rng = k_long_streams(ctx, oracle, "k_long", 33, [(300, 900), (5000, None), (0, 7), (2500, None)], 6)
    one_batch(ctx, rng, streams, "k_long", 3)
    before = [st.win.window for st in streams]
    offsets, total = L.state_offsets([st.win for st in streams])
    buf = torch.zeros(max(total, 1), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    slots, t = ctx.save_states([st.win for st in streams], buf.data_ptr(), DEVICE, offsets)
    t.wait()
    ctx.load_states(slots, buf.data_ptr(), DEVICE).wait()
    assert [st.win.window for st in streams] == before
    one_batch(ctx, rng, streams, "k_long", 3)


@pytest.mark.parametrize("memory", [DEVICE, HOST], ids=["device", "host"])
def test_exhausted_limits_write_nothing(ctx, oracle, memory):
    """A prepared batch whose windows' limits have all run out to 0 writes nothing, reports 0 samples, moves no row
    and leaves every sentinel; after set_window(0, None) it decodes exactly what an unprepared batch over the same
    packets and states does."""
    C, bs0, bs1, S, k, n2 = 2, 8, 11, 3, 3, 1024
    su = make_setup(ctx, C, bs0, bs1, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}], floors=[FLOOR])
    rng = np.random.default_rng(34)
    win = [L.PreviousWindowRight(su) for _ in range(S)]
    ref = [L.PreviousWindowRight(su) for _ in range(S)]
    for w, lim in zip(win, (0, 10, 2047)):          # the first execution produces 2048 samples per stream
        w.set_window(0, lim)
    modes = np.ones(k, np.uint8)
    stride = k * n2 + 4
    n_el = S * C * stride
    coeffs = ctx.host_alloc(S * k * C * n2, np.float32)
    wa, ra = Arena(ctx, n_el, F32P, memory, pinned=True), Arena(ctx, n_el, F32P, memory, pinned=True)
    dco = torch.zeros(coeffs.size, dtype=torch.float32, device="cuda") if memory == DEVICE else None
    co = dco.data_ptr() if dco is not None else coeffs

    def specs(pw):
        return [L.ChainSpec(pw[i], modes, coeff_offset=i * k * C * n2, packet_index=i * k, out_offset=i * C * stride, out_stride=stride)
                for i in range(S)]
    wb = L.Batch(ctx, specs(win), SPECTRUM, memory, co, wa.ptr, F32P)
    for ex in range(4):
        coeffs[...] = (rng.standard_normal(coeffs.size) * 0.1).astype(np.float32)
        if dco is not None:
            dco.copy_(torch.from_numpy(np.array(coeffs)))
            torch.cuda.synchronize()
        if ex < 2:
            wb.run()
            ctx.synchronize()
            assert [c.n_samples for c in wb.collect()] == ([0, 10, 2047] if ex == 0 else [0] * S)
            continue
        if ex == 2:
            assert all(w.window == (0, 0) for w in win)
            sentinel = wa.read()
            with expect_kernels(ctx) as d:
                wb.run()
                ctx.synchronize()
            assert [c.n_samples for c in wb.collect()] == [0] * S
            assert np.array_equal(wa.read(), sentinel), "an exhausted window wrote"
            assert d["k_row_copy"] == 0, d
            for w in win:
                w.set_window(0, None)
            continue
        for r, w in zip(ref, win):
            r.set_data(w.data())
        ref_chains = specs(ref)
        L.decode_chains(ctx, ref_chains, SPECTRUM, memory, co, ra.ptr, F32P)
        wb.run()
        ctx.synchronize()
        assert [c.n_samples for c in wb.collect()] == [c.n_samples for c in ref_chains] == [k * n2] * S
        assert np.array_equal(wa.read(), ra.read())
        for r, w in zip(ref, win):
            assert bits_equal(r.data(), w.data()) and w.window == (0, None)
    wb.close()

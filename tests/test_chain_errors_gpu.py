"""Chains that stop on a packet the reference refuses, on every batch path and entry, against the oracle.

The reference refuses a packet in two places, and they leave the stream in different states:
  * a mode number >= the number of modes (audio.rs:925-929) returns before the state is taken (:1083): the chain reports
    ERR_BAD_FORMAT with packets_done = k, and the stream keeps the right half of packet k - 1 (or the state the chain
    started from, k = 0);
  * the overlap guard -- a left slope shorter than the saved right half (audio.rs:1107-1111) -- fires after :1083 has
    taken the state: ERR_BAD_FORMAT, packets_done = k, and the stream is empty, so its next packet emits 0 samples.

walk_chain decides both on the host, and every batch path sizes its uploads, descriptors, front-stage packet lists,
segments and PCM copy-back from the walk's numbers.  So every packet from the stop on is poisoned -- NaN coefficients
and dense floors, floor_kind 0xFF on host floor arrays (scan_floor_kinds must only look at decoded rows), garbage floor
posts -- and each batch is checked against oracle twins that run the packets before the stop (and, for the guard, the
stopped packet, which the oracle refuses with rc 1 and an empty state):
  * status, packets_done and n_samples of every chain;
  * f32 PCM bit for bit (bits_equal), i16 PCM against oracle.quantise_i16;
  * nothing written outside the chains' write sets (a sentinel-filled arena);
  * every stream's state afterwards, bit for bit, and a second batch that continues every stream (kept or emptied);
  * which kernels ran (expect_kernels), as the routing of such batches stands: try_long and try_mid refuse a batch that
    holds a bad mode number, so uniform 1024- and 512-point batches go to k_chain, 256/2048 and uniform 256-point ones
    to the segmented path (try_mixed), more than 8 channels to the four-kernel path."""
import numpy as np
import pytest
import torch

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from helpers import (ALL_KERNELS, FRONT, FUSED, GENERIC, RefStream, assert_contained, bits_equal, environ, expect_kernels,
                     fill_guard, launches_are_attributed, make_setup, mismatch_report, random_floor1_y, write_set)
from test_frontend_cpu import floor0_expected
from test_vq_shapes_gpu import Streams, vq_kernels

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, I16P, F32I, I16I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED
SPECTRUM, RESIDUE, VQ = cabi.ENTRY_SPECTRUM, cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ
HOST, DEVICE = cabi.MEM_HOST, cabi.MEM_DEVICE
BAD = 7                     # a mode number past every setup's modes
POISON_KIND = 0xFF          # a floor_kind no decoded row may carry
FLOOR = (2, [0, 128, 12, 46, 4, 8, 16, 23, 33, 70])
MODES = [(0, 0), (1, 0)]    # mode 0: short block, mode 1: long block
P = 6                       # packets per chain and batch

# What each stream does in the first batch (A) of a case; the second (B) continues every stream with healthy packets.
#   ok        healthy
#   bad0 / badmid / badlast   bad mode number at packet 0 / P // 2 / P - 1
#   guardmid  a long block with next flag 1, then a short block: the guard stops packet P // 2
#   carry     A ends on a long block with next flag 1; B starts with a short block: the guard stops B's packet 0
#   import    a 1024-sample state set by PreviousWindowRight.set_data; A starts with a short block: the guard at packet 0
#   badlong0  a long block with next flag 0, then a bad mode number: the stream keeps that block's short right half
UNIFORM = ("ok", "bad0", "badmid", "badlast")
CLEAN = UNIFORM + ("carry", "import", "badlong0")
ALL_STOPS = CLEAN + ("guardmid",)


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def planar(fmt):
    return fmt in (F32P, I16P)


def consistent_flags(bf):
    n = len(bf)
    prev, nxt = np.ones(n, np.uint8), np.ones(n, np.uint8)
    for i in range(n):
        if bf[i]:
            prev[i] = bf[i - 1] if i else 1
            nxt[i] = bf[i + 1] if i + 1 < n else 1
    return prev, nxt


def sequence(rng, mixed, kind, batch, first_long=False):
    """(mode numbers, prev flags, next flags, designed stop or None) of one chain of P packets.  first_long: the chain
    starts with a long block (prev flag 1), which no state trips the guard on."""
    if not mixed:
        modes = rng.integers(0, 2, P).astype(np.uint8)            # (both modes are one blocksize)
        prev, nxt = np.ones(P, np.uint8), np.ones(P, np.uint8)
    else:
        bf = (rng.random(P) >= 0.3).astype(np.uint8)
        k = P // 2
        if batch == 0 and kind in ("guardmid", "badlong0"):
            bf[k - 1], bf[k] = 1, 0
        if batch or first_long:
            bf[0] = kind != "carry"         # a chain ends on a full right half: a short block next trips the guard
        elif kind == "carry":
            bf[-1] = 1
        if kind == "import" and batch == 0:
            bf[0] = 0
        prev, nxt = consistent_flags(bf)
        if batch == 0 and kind == "guardmid":
            nxt[k - 1] = 1
        modes = bf.copy()
    stop = None
    if batch == 0:
        stop = {"bad0": 0, "badmid": P // 2, "badlast": P - 1, "badlong0": P // 2, "guardmid": P // 2, "import": 0}.get(kind)
        if kind.startswith("bad"):
            modes[stop] = BAD
    elif kind == "carry":
        stop = 0
    return modes, prev, nxt, stop


class Stream:
    """A device stream, its oracle twin and its stop plan."""

    def __init__(self, oracle, su, kind, mixed, rng):
        self.su, self.kind, self.mixed = su, kind, mixed
        C = su.audio_channels
        self.mappings = [{"coupling": [(0, 1)], "floor_of_channel": [0] * C}]
        self.pwr = L.PreviousWindowRight(su)
        self.last_long = 1
        self.ref = RefStream(oracle, C, su.blocksize_0, su.blocksize_1, MODES, self.mappings, [FLOOR])
        if kind == "import":
            state = (rng.standard_normal((C, 1024)) * 0.1).astype(np.float32)
            self.pwr.set_data(state)
            self.ref.pwr.set_data(state)

    def check_state(self, what):
        a, b = self.pwr.data(), self.ref.pwr.data()
        assert self.pwr.is_empty() == self.ref.pwr.is_empty(), (what, self.kind, "emptiness")
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (what, self.kind, "state")


def make_streams(ctx, oracle, rng, C, bs0, bs1, kinds):
    su = make_setup(ctx, C, bs0, bs1, modes=MODES, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0] * C}],
                    floors=[FLOOR])
    return [Stream(oracle, su, k, bs0 != bs1, rng) for k in kinds]


class Call:
    """One batch over `streams`: every chain's packets, with everything from its designed stop on poisoned, in arenas laid
    out 4-aligned with gaps (device arenas as torch tensors for MEM_DEVICE, page-locked ones for pinned host batches)."""

    def __init__(self, rng, streams, batch, entry=SPECTRUM, fmt=F32P, memory=HOST, floor_memory=HOST, pinned_ctx=None,
                 first_long=False):
        self.streams, self.entry, self.fmt, self.memory, self.floor_memory = streams, entry, fmt, memory, floor_memory
        su = streams[0].su
        C, self.C = su.audio_channels, su.audio_channels
        residue = entry == RESIDUE
        coeffs, dense, kinds, ys = [], [], [], []
        self.plans, self.chains = [], []
        coff = ooff = rows = 0
        stride = (P * (1 << su.blocksize_1) // 2 + 3) // 4 * 4 + 4
        for st in streams:
            modes, prev, nxt, stop = sequence(rng, st.mixed, st.kind, batch, first_long)
            if batch and st.mixed and modes[0] == 1:
                prev[0] = st.last_long          # the block the stream's state came from
            pk, c0 = [], coff
            for i, m in enumerate(int(x) for x in modes):
                n2 = (1 << (su.blocksize_1 if m < len(MODES) and MODES[m][0] else su.blocksize_0)) // 2
                if m >= len(MODES):
                    n2 = (1 << su.blocksize_0) // 2       # (a bad mode's packet occupies the arena as a short block)
                poisoned = stop is not None and i >= stop
                if residue:
                    x = (rng.standard_normal((C, n2)) * rng.integers(0, 2, (C, n2))).astype(np.float32)
                    fl = [None if r < 0.1 else rng.random(n2).astype(np.float32) if r < 0.25 else
                          random_floor1_y(rng, FLOOR[0], len(FLOOR[1])) for r in rng.random(C)]
                    k, y, d = L.DecodedPacket(0, x, fl).pack()
                    d = np.zeros_like(x) if d is None else d
                    if poisoned:
                        x[...] = np.nan
                        d[...] = np.nan
                        y[...] = rng.integers(0, 1 << 32, y.shape, dtype=np.uint64).astype(np.uint32)
                        # device floor arrays are trusted, not scanned: there the poison is a NaN dense floor
                        k[...] = POISON_KIND if floor_memory == HOST else cabi.FLOOR_DENSE
                    kinds.append(k)
                    ys.append(y)
                    dense.append(d.ravel())
                else:
                    x = (rng.standard_normal((C, n2)) * 0.1).astype(np.float32)
                    fl = None
                    if poisoned:
                        x[...] = np.nan
                pk.append((m, int(prev[i]), int(nxt[i]), x.copy(), fl))
                coeffs.append(x.ravel())
                coff += x.size
            self.plans.append((pk, stop))
            self.chains.append(L.ChainSpec(st.pwr, modes, prev, nxt, coeff_offset=c0,
                                           packet_index=rows, out_offset=ooff, out_stride=stride if planar(fmt) else 0))
            ooff += C * stride + 4
            rows += P
        self.total = ooff
        dt = np.float32 if fmt in (F32P, F32I) else np.int16
        self.coeffs = np.concatenate(coeffs)
        self.pcm = fill_guard(np.empty(self.total, dt))
        self.kw = {}
        if residue:
            self.kinds, self.ys, self.dense = np.stack(kinds), np.stack(ys), np.concatenate(dense)
        if pinned_ctx is not None:          # page-locked copies, as a host-memory submit needs
            def pin(a):
                out = pinned_ctx.host_alloc(a.shape, a.dtype)
                out[...] = a
                return out
            self.coeffs, self.pcm = pin(self.coeffs), pin(self.pcm)
            if residue:
                self.kinds, self.ys, self.dense = pin(self.kinds), pin(self.ys), pin(self.dense)
        if residue:
            self.kw = dict(floor_kind=self.kinds, floor1_y=self.ys, dense_floor=self.dense, floor_memory=floor_memory)
        self.dev = {}
        if memory == DEVICE:
            self.dev = {"coeffs": torch.from_numpy(self.coeffs).cuda(), "pcm": torch.from_numpy(self.pcm).cuda()}
            self.dev["guard"] = self.dev["pcm"].clone()
            if residue:
                self.dev["dense"] = torch.from_numpy(self.dense).cuda()
                self.kw["dense_floor"] = self.dev["dense"].data_ptr()
        if residue and floor_memory == DEVICE:
            self.dev["kinds"], self.dev["ys"] = torch.from_numpy(self.kinds).cuda(), torch.from_numpy(self.ys).cuda()
            self.kw.update(floor_kind=self.dev["kinds"].data_ptr(), floor1_y=self.dev["ys"].data_ptr())

    def arenas(self):
        if self.memory == DEVICE:
            return self.dev["coeffs"].data_ptr(), self.dev["pcm"].data_ptr()
        return self.coeffs, self.pcm

    def expect(self):
        """Runs the twins over the packets up to each chain's stop: [(status, packets_done, want [C][n])]."""
        out = []
        for st, (pk, stop) in zip(self.streams, self.plans):
            parts, found, status = [], None, cabi.OK
            for i, (m, pf, nf, x, fl) in enumerate(pk):
                if m >= len(MODES):                     # audio.rs:925-929: the state stays as it is
                    found, status = i, cabi.ERR_BAD_FORMAT
                    break
                if self.entry == RESIDUE:
                    rc, o = st.ref.packet(m, pf, nf, x, fl)
                else:
                    rc, o = st.ref.spectrum(m, pf, nf, x)
                if rc:                                  # audio.rs:1107-1111, after the state was taken
                    assert rc == 1 and st.ref.pwr.is_empty(), (st.kind, i, rc)
                    found, status = i, cabi.ERR_BAD_FORMAT
                    break
                parts.append(o)
                st.last_long = MODES[m][0]
            assert found == stop, (st.kind, "the oracle stops at", found, "the case was built to stop at", stop)
            want = np.concatenate(parts, axis=1) if parts else np.zeros((self.C, 0), np.float32)
            out.append((status, len(parts), want))
        return out

    def submit(self, ctx):
        L.decode_chains(ctx, self.chains, self.entry, self.memory, *self.arenas(), self.fmt, **self.kw)

    def reset_pcm(self):
        if self.memory == DEVICE:
            self.dev["pcm"].copy_(self.dev["guard"])
        else:
            fill_guard(self.pcm)

    def output(self):
        return self.dev["pcm"].cpu().numpy() if self.memory == DEVICE else self.pcm

    def check(self, oracle, chains, wants, what, states=True):
        """Chain results, the whole output arena and (states) every stream's state against the oracle."""
        pcm, C = self.output(), self.C
        for i, (c, (status, done, want)) in enumerate(zip(chains, wants)):
            n = want.shape[1]
            kind = self.streams[i].kind
            assert (c.status, c.packets_done, c.n_samples) == (status, done, n), \
                (what, kind, "got", (c.status, c.packets_done, c.n_samples), "want", (status, done, n))
            o, sd = int(c.out_offset), int(c.out_stride)
            got = (np.stack([pcm[o + k * sd:o + k * sd + n] for k in range(C)]) if planar(self.fmt)
                   else pcm[o:o + n * C].reshape(n, C).T)
            if pcm.dtype == np.float32:
                assert bits_equal(got, want), (what, kind, mismatch_report(got, want))
            else:
                assert np.array_equal(got, oracle.quantise_i16(want)), (what, kind)
        assert_contained(pcm, write_set(chains, lambda i: C, self.fmt), what)
        for st in self.streams if states else ():
            st.check_state(what)


# ---------------------------------------------------------------------------------------------------------------------
# the kernels a batch must and must not run
# ---------------------------------------------------------------------------------------------------------------------
SEGMENTED = {"k_long", "k_long_s", "k_short", "k_short_g"}


def pins(path, entry):
    """(ran, not_ran, segmented): the kernels of `path` for a batch of `entry`; segmented: some fused kernel must run.
    paths: 'mixed' (try_mixed, any schedule), 'pass' (its one pass: k_long_s), 'rounds' (rounds only: k_long, no
    k_long_s), 'short' (uniform 256-point: k_short alone), 'chain' (k_chain once), 'mid' (k_mid once), 'generic' (the
    four-kernel path)."""
    front = entry != SPECTRUM
    f0 = {"k_floor0_curves"}
    if path in ("mixed", "pass", "rounds"):
        ran = {"pass": {"k_long_s"}, "rounds": {"k_long"}}.get(path, set()) | (FRONT if front else set())
        not_ran = GENERIC | {"k_mid"} | ({"k_long_s"} if path == "rounds" else set()) | (set() if front else FRONT | f0)
        return ran, not_ran, True
    if path == "short":
        ran = {"k_short"} | (FRONT if front else set())
        return ran, ALL_KERNELS - ran - f0 - {"k_chain"}, False
    if path == "chain":
        return {"k_chain": 1}, ALL_KERNELS - {"k_chain"} - f0, False
    if path == "mid":
        ran = {"k_mid": 1, **({"k_floor1_segments": 1, "k_prologue_fused": 1} if front else {})}
        return ran, ALL_KERNELS - set(ran) - f0, False
    assert path == "generic", path
    return {"k_imdct", "k_overlap", "k_save_state"}, FUSED | {"k_chain", "k_row_copy"}, False


def run_pinned(ctx, call, path):
    ran, not_ran, segmented = pins(path, call.entry)
    with expect_kernels(ctx, ran=ran, not_ran=not_ran) as d:
        call.submit(ctx)
    if segmented:
        assert sum(d[k] for k in SEGMENTED), f"no fused kernel ran on the segmented path: {d}"


# ---------------------------------------------------------------------------------------------------------------------
# 1: stopped chains on every batch path, then a batch that continues every stream
# ---------------------------------------------------------------------------------------------------------------------
# id: (channels, bs0, bs1, stream kinds, entry, format, memory, floor memory, env, (path of batch A, path of batch B))
ROWS = {
    # 256/2048 stereo, clean flags: the one pass; inconsistent ones (guardmid): rounds behind it
    "spectrum-8/11-pass": (2, 8, 11, CLEAN, SPECTRUM, F32P, HOST, HOST, None, ("pass", "pass")),
    "spectrum-8/11-guard": (2, 8, 11, ALL_STOPS, SPECTRUM, I16P, DEVICE, HOST, None, ("mixed", "mixed")),
    "residue-8/11": (2, 8, 11, ALL_STOPS, RESIDUE, F32P, HOST, HOST, None, ("mixed", "mixed")),
    "residue-8/11-6ch": (6, 8, 11, ALL_STOPS, RESIDUE, I16P, DEVICE, DEVICE, None, ("mixed", "mixed")),
    "residue-8/11-chunks": (2, 8, 11, ALL_STOPS, RESIDUE, I16P, HOST, HOST, {"LWB_E2E_CHUNKS": "3"}, ("mixed", "mixed")),
    "spectrum-8/8": (2, 8, 8, UNIFORM, SPECTRUM, F32P, DEVICE, HOST, None, ("short", "short")),
    # uniform 1024 / 512: k_mid's shape, but for the bad mode numbers
    "spectrum-10/10": (2, 10, 10, UNIFORM, SPECTRUM, I16P, HOST, HOST, None, ("chain", "mid")),
    "residue-9/9": (2, 9, 9, UNIFORM, RESIDUE, F32P, DEVICE, HOST, None, ("chain", "mid")),
    "spectrum-6/13": (2, 6, 13, ALL_STOPS, SPECTRUM, F32I, HOST, HOST, None, ("chain", "chain")),
    "residue-7/12": (2, 7, 12, ALL_STOPS, RESIDUE, I16I, DEVICE, DEVICE, None, ("chain", "chain")),
    "spectrum-8/11-interleaved": (2, 8, 11, ALL_STOPS, SPECTRUM, I16I, HOST, HOST, None, ("chain", "chain")),
    "spectrum-8/11-10ch": (10, 8, 11, ALL_STOPS, SPECTRUM, F32P, HOST, HOST, None, ("generic", "generic")),
    "residue-8/11-10ch": (10, 8, 11, ALL_STOPS, RESIDUE, I16I, DEVICE, HOST, None, ("generic", "generic")),
}
# the reference schedules of one spectrum and one residue row
for _name, _base in (("spectrum", "spectrum-8/11-guard"), ("residue", "residue-8/11")):
    for _env, _path in ((("LWB_FORCE_GENERIC", "1"), "generic"), (("LWB_FORCE_GENERIC", "2"), "chain"),
                        (("LWB_NO_MIXED", "1"), "chain"), (("LWB_MIXED_ROUNDS", "1"), "rounds")):
        ROWS[f"{_name}-8/11-{_env[0]}={_env[1]}"] = ROWS[_base][:8] + (dict([_env]), (_path, _path))


@pytest.mark.parametrize("row", list(ROWS))
def test_stopped_chains_and_the_batch_after(ctx, oracle, row):
    C, bs0, bs1, kinds, entry, fmt, memory, floor_memory, env, paths = ROWS[row]
    rng = np.random.default_rng(sum(map(ord, row)))
    streams = make_streams(ctx, oracle, rng, C, bs0, bs1, kinds)
    with environ(env):
        for batch, path in enumerate(paths):
            call = Call(rng, streams, batch, entry, fmt, memory, floor_memory)
            wants = call.expect()
            run_pinned(ctx, call, path)
            ctx.synchronize()
            call.check(oracle, call.chains, wants, (row, "batch", batch))


# ---------------------------------------------------------------------------------------------------------------------
# 2: prepared batches and tickets
# ---------------------------------------------------------------------------------------------------------------------
# stops that do not depend on the state a run starts from (the chains start with a long block: see first_long)
PREPARED = ("ok", "bad0", "badmid", "guardmid", "badlong0", "badlast")
RESULT_SENTINEL = (-99, 0xFFFFFFFF, 0xFFFFFFFF)     # (status, packets_done, n_samples) no batch reports


@pytest.mark.parametrize("entry", [SPECTRUM, RESIDUE])
def test_prepared_batch_with_stopped_chains(ctx, oracle, entry):
    """A device-memory Batch over 256/2048 stereo chains that stop on both kinds of error, run three times on the same
    streams: the first run changes the streams' state shapes, the second plans the batch anew and captures it (the
    residue entry with its front stages, whose host floor arrays carry the poisoned rows), the third replays the
    capture -- the same launches as the second.  Which of the two the library did shows in the chain array: planning
    writes every chain's results, a replay leaves them as the capture found them (lwb_plan_execute), so they are
    overwritten with RESULT_SENTINEL before the second and third runs.  After each run the chain results, the PCM and
    the states equal the oracle's, the twins continuing over the same packets."""
    rng = np.random.default_rng(70 + entry)
    streams = make_streams(ctx, oracle, rng, 2, 8, 11, PREPARED)
    call = Call(rng, streams, 0, entry, F32P, DEVICE, HOST, first_long=True)
    coeffs, pcm = call.arenas()
    batch = L.Batch(ctx, call.chains, entry, DEVICE, coeffs, pcm, F32P, **call.kw)
    ran, not_ran, _ = pins("mixed", entry)
    launches, planned = [], None
    for run in range(3):
        call.reset_pcm()
        torch.cuda.synchronize()
        wants = call.expect()
        if run:
            for c in batch._arr:
                c.status, c.packets_done, c.n_samples = RESULT_SENTINEL
        with expect_kernels(ctx, ran=ran if run < 2 else launches[1], not_ran=not_ran) as d:
            batch.run()
        launches.append({k: v for k, v in d.items() if v})
        ctx.synchronize()
        results = [(c.status, c.packets_done, c.n_samples) for c in batch._arr]
        if run == 1:
            assert RESULT_SENTINEL not in results, ("the second run did not plan the batch", results)
            planned = results
        if run == 2:
            assert all(r == RESULT_SENTINEL for r in results), ("the third run planned the batch instead of replaying", results)
            for c, r in zip(batch._arr, planned):
                c.status, c.packets_done, c.n_samples = r
        call.check(oracle, batch.collect(), wants, ("prepared", entry, "run", run))
    assert sum(launches[2].get(k, 0) for k in SEGMENTED), launches
    batch.close()


@pytest.mark.parametrize("entry,fmt,path", [(SPECTRUM, F32I, "chain"), (RESIDUE, I16P, "mixed")])
def test_submitted_batches_with_stopped_chains(ctx, oracle, entry, fmt, path):
    """Two host-memory batches (page-locked arrays) submitted back to back through Context.submit_chains, the second
    continuing every stream of the first, which holds the stopped chains: each ticket's wait() returns the chains with
    their results, and once both are done the PCM, the write sets and the states equal the oracle's."""
    rng = np.random.default_rng(80 + entry)
    streams = make_streams(ctx, oracle, rng, 2, 8, 11, ALL_STOPS)
    calls, wants = [], []
    for batch in range(2):
        calls.append(Call(rng, streams, batch, entry, fmt, HOST, HOST, pinned_ctx=ctx))
        wants.append(calls[-1].expect())
    tickets = []
    for call in calls:
        ran, not_ran, _ = pins(path, entry)
        with expect_kernels(ctx, ran=ran, not_ran=not_ran):
            tickets.append(ctx.submit_chains(call.chains, entry, HOST, call.coeffs, call.pcm, fmt, **call.kw))
    done = [t.wait() for t in tickets]
    for batch, (call, chains) in enumerate(zip(calls, done)):
        for c, (status, n_done, want) in zip(chains, wants[batch]):
            assert (c.status, c.packets_done, c.n_samples) == (status, n_done, want.shape[1]), ("ticket", batch)
    # (the states are the second batch's)
    calls[0].check(oracle, done[0], wants[0], ("submitted", entry, "batch", 0), states=False)
    calls[1].check(oracle, done[1], wants[1], ("submitted", entry, "batch", 1))


# ---------------------------------------------------------------------------------------------------------------------
# 3: the per-packet API
# ---------------------------------------------------------------------------------------------------------------------
def test_per_packet_bad_mode_number_keeps_the_state(ctx, oracle):
    """read_audio_packet_generic and decode_spectrum with a bad mode number raise AudioReadError(ERR_BAD_FORMAT), and so
    do the library's own lwb_decode_packet / lwb_decode_spectrum behind them; the stream's state stays bit for bit what
    it was."""
    import ctypes as C
    rng = np.random.default_rng(90)
    su = make_setup(ctx, 2, 8, 11, modes=MODES, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}],
                    floors=[FLOOR])
    pwr = L.PreviousWindowRight(su)
    for _ in range(2):
        L.decode_spectrum(su, 1, (rng.standard_normal((2, 1024)) * 0.1).astype(np.float32), pwr)
    before = pwr.data()
    assert before is not None and before.shape == (2, 1024)
    spec = (rng.standard_normal((2, 128)) * 0.1).astype(np.float32)
    packet = L.DecodedPacket(BAD, spec, [[10, 20] + [0] * 8, None])
    for call in (lambda: L.decode_spectrum(su, BAD, spec, pwr),
                 lambda: L.read_audio_packet_generic(su, packet, pwr),
                 lambda: L.read_audio_packet_generic(su, packet, pwr, sample="i16", interleaved=True)):
        with pytest.raises(L.AudioReadError) as e:
            call()
        assert e.value.code == cabi.ERR_BAD_FORMAT and e.value.kind == "AudioBadFormat"
        assert bits_equal(pwr.data(), before)
    out, n = np.zeros((2, 2048), np.float32), C.c_size_t(12345)
    rc = cabi.lib().lwb_decode_spectrum(pwr._h, BAD, 1, 1, spec.ctypes.data_as(C.c_void_p), F32P,
                                        out.ctypes.data_as(C.c_void_p), 2048, C.byref(n))
    assert rc == cabi.ERR_BAD_FORMAT
    assert bits_equal(pwr.data(), before)
    kinds, ys, _ = packet.pack()
    p = cabi.Packet()
    p.mode_number, p.prev_window_flag, p.next_window_flag = BAD, 1, 1
    p.floor_kind, p.floor1_y = kinds.ctypes.data_as(cabi.u8p), ys.ctypes.data_as(cabi.u32p)
    p.residue = spec.ctypes.data_as(cabi.fp)
    rc = cabi.lib().lwb_decode_packet(pwr._h, C.byref(p), F32P, out.ctypes.data_as(C.c_void_p), 2048, C.byref(n))
    assert rc == cabi.ERR_BAD_FORMAT
    assert bits_equal(pwr.data(), before) and not pwr.is_empty()


# ---------------------------------------------------------------------------------------------------------------------
# 4: the VQ entry and floor-0 records
# ---------------------------------------------------------------------------------------------------------------------
class PackerCall:
    """One batch of packer-made packets (tests/vorbis_packer.py) decoded by the host front half: the dense residue entry
    (floor-0 records in the floor rows) or the VQ entry.  The chains follow the stop plans of sequence(): each position
    takes a packet of the block size it asks for, with the window flags of the plan (the flags are the chain's, not the
    packet's).  From the stop on: floor_kind 0xFF, garbage floor words, NaN residues and, VQ entry, the poisoned rows'
    run and entry offsets zeroed (out of order, so a path that read them would fail the library's offset check) and
    their codebook entries zeroed."""

    def __init__(self, rng, st, streams, batch, entry, fmt):
        self.streams, self.entry, self.fmt, self.st, self.C = streams, entry, fmt, st, st.C
        hdr, spec, C = st.hdr, st.spec, st.C
        mixed = spec.bs0 != spec.bs1
        pool = {0: [], 1: []}
        for s in range(st.S):
            for p in st.packets[s]:
                pool[p[1]["blockflag"] if mixed else 0].append(p)
        coeffs, kinds, ys, runs, ents, roffs, eoffs, poisoned_rows = [], [], [], [], [], [0], [0], set()
        self.plans, self.chains = [], []
        coff = ooff = row = 0
        stride = (P * (1 << spec.bs1) // 2 + 3) // 4 * 4 + 4
        for tw in streams:
            modes, prev, nxt, stop = sequence(rng, mixed, tw.kind, batch)
            if batch and mixed and modes[0] == 1:
                prev[0] = tw.last_long
            pk, c0 = [], coff
            for i in range(P):
                bad = modes[i] == BAD
                choice = pool[int(modes[i]) if mixed and not bad else 0]
                pkt, info, nbytes = choice[int(rng.integers(len(choice)))]
                if not bad:
                    modes[i] = info["mode"]
                d = hdr.decode_packet(pkt, floor0_records=st.records)
                _, rr, ee = hdr.decode_packet_vq(pkt, floor0_records=st.records)
                k, y, _ = d.pack()
                x = d.residue.copy()
                if stop is not None and i >= stop:
                    x[...] = np.nan
                    k[...] = POISON_KIND
                    y[...] = rng.integers(0, 1 << 32, y.shape, dtype=np.uint64).astype(np.uint32)
                    ee = np.zeros_like(ee)
                    poisoned_rows.add(row + i)
                pk.append((int(modes[i]), int(prev[i]), int(nxt[i]), info, nbytes))
                coeffs.append(x.ravel())
                kinds.append(k)
                ys.append(y)
                runs.append(rr)
                ents.append(ee)
                roffs.append(roffs[-1] + len(rr))
                eoffs.append(eoffs[-1] + len(ee))
                coff += x.size
            self.plans.append((pk, stop))
            self.chains.append(L.ChainSpec(tw.pwr, modes, prev, nxt, coeff_offset=c0, packet_index=row, out_offset=ooff,
                                           out_stride=stride if planar(fmt) else 0))
            ooff += C * stride + 4
            row += P
        self.total = ooff
        roffs, eoffs = np.array(roffs, np.uint64), np.array(eoffs, np.uint64)
        # offsets[r] is where row r starts: the first poisoned row's start ends the decoded rows, and the next chain's
        # first row starts where a chain ends; every other offset of a poisoned row is garbage
        for r in poisoned_rows:
            for j in (r, r + 1):
                if r - 1 in poisoned_rows if j == r else (r + 1 in poisoned_rows or j == row):
                    roffs[j] = eoffs[j] = 0
        self.kinds, self.ys = np.concatenate(kinds), np.concatenate(ys)
        self.has_records = {i for i, (pk, stop) in enumerate(self.plans)
                            if np.any(self.kinds[self.chains[i].packet_index * C:
                                                 (self.chains[i].packet_index + (P if stop is None else stop)) * C]
                                      == cabi.FLOOR_ZERO)}
        self.coeffs = np.concatenate(coeffs)
        self.vq = (np.concatenate(runs) if roffs.max() else np.zeros(1, fe.VQ_RUN_DTYPE), roffs,
                   np.concatenate(ents).astype(np.uint16) if eoffs.max() else np.zeros(1, np.uint16), eoffs)
        self.pcm = fill_guard(np.empty(self.total, np.float32 if fmt in (F32P, F32I) else np.int16))

    def expect(self):
        spec, out = self.st.spec, []
        for tw, (pk, stop) in zip(self.streams, self.plans):
            parts, found, status = [], None, cabi.OK
            for i, (m, pf, nf, info, nbytes) in enumerate(pk):
                if m >= len(spec.modes):
                    found, status = i, cabi.ERR_BAD_FORMAT
                    break
                fl_exp, res = spec.expected(info, nbytes)
                fl = [None if f is None else list(f[1]) if f[0] == "one" else
                      floor0_expected(f[3], f[1], f[2], info["blockflag"], info["n"] // 2, spec.bs0, spec.bs1) for f in fl_exp]
                rc, o = tw.ref.packet(m, pf, nf, res, fl)
                if rc:
                    assert rc == 1 and tw.ref.pwr.is_empty(), (tw.kind, i, rc)
                    found, status = i, cabi.ERR_BAD_FORMAT
                    break
                parts.append(o)
                tw.last_long = spec.modes[m][0]
            assert found == stop, (tw.kind, "the oracle stops at", found, "the case was built to stop at", stop)
            out.append((status, len(parts), np.concatenate(parts, axis=1) if parts else np.zeros((self.C, 0), np.float32)))
        return out

    def submit(self, ctx):
        kw = dict(floor_kind=self.kinds, floor1_y=self.ys)
        if self.entry == VQ:
            kw["vq"] = self.vq
        L.decode_chains(ctx, self.chains, self.entry, HOST, None if self.entry == VQ else self.coeffs, self.pcm, self.fmt, **kw)

    def output(self):
        return self.pcm

    check = Call.check


class PackerStream:
    """A device stream of a packer setup, its oracle twin and its stop plan."""

    def __init__(self, st, su, twin, kind, rng):
        self.kind, self.pwr, self.ref, self.last_long = kind, L.PreviousWindowRight(su), twin, 1
        if kind == "import":
            state = (rng.standard_normal((st.C, 1024)) * 0.1).astype(np.float32)
            self.pwr.set_data(state)
            self.ref.pwr.set_data(state)

    check_state = Stream.check_state


# id: (channels, bs0, bs1, floor-0 records, entry, format, (path of batch A, path of batch B))
PACKER_ROWS = {
    "vq-8/11": (2, 8, 11, False, VQ, I16I, ("chain", "chain")),
    "vq-8/11-records": (2, 8, 11, True, VQ, F32I, ("chain", "chain")),
    "vq-10/10": (2, 10, 10, False, VQ, F32P, ("chain", "mid")),
    "records-8/11": (2, 8, 11, True, RESIDUE, F32I, ("chain", "chain")),
    "records-10/10": (2, 10, 10, True, RESIDUE, I16P, ("chain", "mid")),
}


@pytest.mark.parametrize("row", list(PACKER_ROWS))
def test_stopped_vq_and_floor0_record_chains(ctx, oracle, row):
    """Stopped chains on the VQ entry and on the residue entry with floor-0 records, two batches as above.  The VQ
    arrays' uploads are sized by the offsets of the decoded rows only, and k_floor0_curves (chain_floor0_curves, or the
    front stages before k_mid) runs over the decoded packets -- pinned to run exactly when a decoded row holds a record."""
    C, bs0, bs1, records, entry, fmt, paths = PACKER_ROWS[row]
    seed = sum(map(ord, row))
    st = Streams(seed, C, bs0, bs1, None, records, 3, 12, p_short=0.3)
    assert len(st.spec.modes) <= BAD
    su = st.hdr.make_setup(ctx, floor0=records)
    rng = np.random.default_rng(seed)
    kinds = ALL_STOPS if bs0 != bs1 else UNIFORM
    streams = [PackerStream(st, su, st.twins(oracle)[0], kind, rng) for kind in kinds]
    try:
        for batch, path in enumerate(paths):
            call = PackerCall(rng, st, streams, batch, entry, fmt)
            wants = call.expect()
            ran, not_ran = vq_kernels(path, bool(call.has_records))
            with expect_kernels(ctx, ran=ran, not_ran=not_ran):
                call.submit(ctx)
            ctx.synchronize()
            call.check(oracle, call.chains, wants, (row, "batch", batch))
    finally:
        st.hdr.close()

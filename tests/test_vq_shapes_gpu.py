"""LWB_ENTRY_VQ batches of every shape the fused long-block kernels do not take, on the GPU, against the oracle.

A VQ batch carries each packet's residue as the VQ runs and codebook entries the front half decoded, not as dense
vectors.  Interleaved output at any blocksize, uniform 1024- and 512-point streams and every other blocksize pair run in
one k_chain launch (which accumulates each packet's vectors in shared memory) or, planar 1024 / 512, through the front
stages and k_mid -- the same kernels as the dense residue entry of the same packets.  The tests feed packer-made
bitstreams (tests/vorbis_packer.py) through the host front half and check, per batch of three that carry state:

  * the PCM equals the oracle's decode of what the packer encoded (f32 bit for bit up to +-0 / NaN, i16 exactly),
    also for packets cut inside their residue;
  * it is byte-identical to the dense residue entry of the same packets, and to the same VQ batch on the four-kernel
    path (LWB_FORCE_GENERIC=1), which stays the reference schedule, up to the sign of NaNs (same_but_nan_signs);
  * nothing outside the chains' write sets changes, the end states equal the oracle's, and the batch ran the kernels
    named for its shape."""
import numpy as np
import pytest
import torch

import lewton_b200 as L
import vorbis_packer as vp
from helpers import (ALL_KERNELS, FRONT, GENERIC, RefStream, assert_contained, bits_equal, environ, expect_kernels, fill_guard,
                     launches_are_attributed, mismatch_report, write_set)
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from test_frontend_cpu import floor0_expected
from test_frontend_gpu import consistent_modes
from test_queued_batches import Gate

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, I16P, F32I, I16I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED
HOST, DEVICE, VQ, RESIDUE = cabi.MEM_HOST, cabi.MEM_DEVICE, cabi.ENTRY_VQ, cabi.ENTRY_RESIDUE
FOUR_KERNEL = GENERIC - {"k_prologue"}         # (VQ records: the four-kernel path's front stages are FRONT)


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def planar(fmt):
    return fmt in (F32P, I16P)


def same_but_nan_signs(a, b):
    """Byte-identical PCM, except that where both are NaN the sign may differ.  k_chain / k_mid and the four-kernel path
    can give one NaN (say an infinite floor-0 curve times a zero residue) opposite signs, for the dense residue entry as
    for the VQ entry: the parity rule treats any NaN as equal, and the kernels were never held to NaN signs."""
    if a.dtype != np.float32:
        return a.tobytes() == b.tobytes()
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


# ---------------------------------------------------------------------------------------------------------------------
# streams, batches and the oracle
# ---------------------------------------------------------------------------------------------------------------------
class Streams:
    """S packer streams of one VQ-capable setup, their packets (the last stream's cut inside the residue) and oracle
    twins.  Redrawn until lwf_headers_vq_capable accepts the setup and, records, until a packet carries a floor-0 record."""

    def __init__(self, seed, channels, bs0, bs1, rtype, records, S, n_packets, p_short=0.2):
        for k in range(40):
            rng = np.random.default_rng(seed + 1000 * k)
            spec = vp.StreamSpec(rng, channels=channels, bs0=bs0, bs1=bs1, floor0=records,
                                 residue_types=None if rtype is None else [rtype])
            hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
            if not hdr.vq_capable():
                hdr.close()
                continue
            packets = []
            for s in range(S):
                st = []
                for mode, prev, nxt in consistent_modes(spec, rng, n_packets, p_short):
                    pk, info = spec.audio_packet(mode, prev, nxt, p_unused=0.15)
                    nbytes = None
                    lo = (max(info["floor_ends"]) + 7) // 8 + 1          # past every floor: the cut lands in the residue
                    if s == S - 1 and lo < len(pk):
                        nbytes = int(rng.integers(lo, len(pk)))
                        pk = pk[:nbytes]
                    st.append((pk, info, nbytes))
                packets.append(st)
            if records and not any(f is not None and f[0] == "zero" for st in packets for _, info, nb in st
                                   for f in spec.expected(info, nb)[0]):
                hdr.close()
                continue
            self.spec, self.hdr, self.packets, self.records = spec, hdr, packets, records
            self.C, self.S = channels, S
            return
        raise AssertionError("no VQ-capable draw")

    def twins(self, oracle):
        spec = self.spec
        floors = [(f.multiplier, f.x_list) if isinstance(f, vp.Floor1) else (1, [0, 128]) for f in spec.floors]
        mappings = [{"coupling": m["coupling"], "floor_of_channel": [m["floors"][m["mux"][c]] for c in range(spec.channels)]}
                    for m in spec.mappings]
        return [RefStream(oracle, spec.channels, spec.bs0, spec.bs1, spec.modes, mappings, floors) for _ in range(self.S)]

    def oracle_packet(self, ref, info, nbytes):
        spec = self.spec
        fl_exp, res = spec.expected(info, nbytes)
        fl = []
        for f in fl_exp:
            if f is None:
                fl.append(None)
            elif f[0] == "one":
                fl.append(list(f[1]))
            else:
                fl.append(floor0_expected(f[3], f[1], f[2], info["blockflag"], info["n"] // 2, spec.bs0, spec.bs1))
        rc, pcm = ref.packet(info["mode"], info["prev"], info["next"], res, fl)
        assert rc == 0
        return pcm


class Batch:
    """Packets [p0, p1) of every stream as one batch: the dense and the VQ decode of the same bytes, the arenas' layout
    (4-aligned, with gaps between chains) and the oracle's PCM (twins advanced over the packets)."""

    def __init__(self, st, p0, p1, fmt, twins=None):
        self.st, self.fmt = st, fmt
        C, hdr = st.C, st.hdr
        coeffs, dense, kinds, ys, runs, ents, roffs, eoffs = [], [], [], [], [], [], [0], [0]
        self.layout, self.wants = [], []
        coff = ooff = row = 0
        any_dense = False
        for s in range(st.S):
            modes, prevs, nexts, steady, c0, parts = [], [], [], 0, coff, []
            for pk, info, nbytes in st.packets[s][p0:p1]:
                d = hdr.decode_packet(pk, floor0_records=st.records)
                v, rr, ee = hdr.decode_packet_vq(pk, floor0_records=st.records)
                k, y, dn = d.pack()
                kinds.append(k)
                ys.append(y)
                any_dense |= dn is not None
                dense.append(np.zeros(d.residue.size, np.float32) if dn is None else dn.ravel())
                coeffs.append(d.residue.ravel())
                runs.append(rr)
                ents.append(ee)
                roffs.append(roffs[-1] + len(rr))
                eoffs.append(eoffs[-1] + len(ee))
                modes.append(v.mode_number); prevs.append(v.prev_window_flag); nexts.append(v.next_window_flag)
                coff += d.residue.size
                steady += st.hdr.decoded_sample_count(pk)
                if twins is not None:
                    parts.append(st.oracle_packet(twins[s], info, nbytes))
            stride = (steady + 3) // 4 * 4 + 4
            self.layout.append((np.array(modes, np.uint8), np.array(prevs, np.uint8), np.array(nexts, np.uint8), c0, row, ooff,
                                stride if planar(fmt) else 0))
            ooff += C * stride + 4 if planar(fmt) else (C * steady + 3) // 4 * 4 + 4
            row += p1 - p0
            if twins is not None:
                self.wants.append(np.concatenate(parts, axis=1))
        self.coeffs, self.kinds, self.ys = np.concatenate(coeffs), np.concatenate(kinds), np.concatenate(ys)
        self.dense = np.concatenate(dense) if any_dense else None
        self.vq = (np.concatenate(runs) if roffs[-1] else np.zeros(1, fe.VQ_RUN_DTYPE), np.array(roffs, np.uint64),
                   np.concatenate(ents).astype(np.uint16) if eoffs[-1] else np.zeros(1, np.uint16), np.array(eoffs, np.uint64))
        self.n_out = ooff
        self.has_records = bool(np.any(self.kinds == cabi.FLOOR_ZERO))
        # k_mid's shape (planar output aside): every packet a full-window block of the long size, on top of no state or
        # the right half of one
        n, n0 = 1 << st.spec.bs1, 1 << st.spec.bs0
        full = [all(info["n"] == n and (info["prev"] or n == n0 or k < p0) and (info["next"] or n == n0)
                    for k, (_, info, _) in enumerate(st.packets[s][:p1]) if k >= p0 - 1) for s in range(st.S)]
        self.uniform = n <= 1024 and all(full)

    def chains(self, pwrs):
        return [L.ChainSpec(pwrs[s], m, p, n, coeff_offset=c0, packet_index=r, out_offset=o, out_stride=sd)
                for s, (m, p, n, c0, r, o, sd) in enumerate(self.layout)]

    def run(self, ctx, pwrs, entry, memory, floor_mem, expect=None):
        """One lwb_decode_chains over a sentinel-filled output arena: (pcm, chains)."""
        dt = np.float32 if self.fmt in (F32P, F32I) else np.int16
        pcm = fill_guard(np.empty(self.n_out, dt))
        chains = self.chains(pwrs)
        frees = []

        def dev(a):
            a = np.ascontiguousarray(a)
            p = ctx.device_alloc(max(a.nbytes, 16))
            ctx.h2d(p, a)
            frees.append(p)
            return p

        try:
            kw = dict(floor_kind=self.kinds, floor1_y=self.ys)
            if entry == VQ:
                kw["vq"] = self.vq
            if floor_mem == DEVICE:
                kw = {k: dev(a) if k != "vq" else tuple(dev(x) for x in a) for k, a in kw.items()}
                kw["floor_memory"] = DEVICE
            coeffs = None if entry == VQ else self.coeffs
            dense, out = self.dense, pcm
            if memory == DEVICE:
                coeffs = None if coeffs is None else dev(coeffs)
                dense = None if dense is None else dev(dense)
                out = dev(pcm)
            with expect_kernels(ctx, *(expect or ((), ()))):
                L.decode_chains(ctx, chains, entry, memory, coeffs, out, self.fmt, dense_floor=dense, **kw)
            ctx.synchronize()
            if memory == DEVICE:
                ctx.d2h(pcm, out)
        finally:
            for p in frees:
                ctx.device_free(p)
        return pcm, chains

    def check_oracle(self, oracle, pcm, chains, what):
        C = self.st.C
        for s, (w, c) in enumerate(zip(self.wants, chains)):
            n = w.shape[1]
            assert (c.status, c.n_samples) == (0, n), (what, s, c.status, c.n_samples, n)
            _, _, _, _, _, o, sd = self.layout[s]
            got = pcm[o:o + C * sd].reshape(C, sd)[:, :n] if planar(self.fmt) else pcm[o:o + n * C].reshape(n, C).T
            if pcm.dtype == np.float32:
                assert bits_equal(got, w), (what, s, mismatch_report(got, w))
            else:
                assert np.array_equal(got, oracle.quantise_i16(w)), (what, s)
        assert_contained(pcm, write_set(chains, lambda i: C, self.fmt), what)


def vq_kernels(shape, floor0):
    """(ran, not_ran) of a VQ batch: 'chain' -> k_chain alone; 'mid' -> the front stages and k_mid; plus the floor-0
    curves when the batch may carry records."""
    f0 = {"k_floor0_curves": 1 if floor0 else 0}
    if shape == "chain":
        return {"k_chain": 1, **f0}, ALL_KERNELS - {"k_chain", "k_floor0_curves"}
    return {"k_floor1_segments": 1, "k_prologue_fused": 1, "k_mid": 1, **f0}, ALL_KERNELS - FRONT - {"k_mid", "k_floor0_curves"}


# ---------------------------------------------------------------------------------------------------------------------
# 1, 2: parity and kernels on every newly covered shape
# ---------------------------------------------------------------------------------------------------------------------
# channels, bs0, bs1, residue type (None: the packer's random mix), floor-0 records, format, memory, floor / VQ memory
CASES = [
    (2, 8, 11, 1, False, I16I, HOST, HOST),      # the player's shape: 256/2048 stereo, interleaved i16
    (2, 8, 11, 2, True, F32I, DEVICE, DEVICE),
    (1, 8, 11, 0, False, F32I, HOST, DEVICE),
    (8, 8, 11, None, False, I16I, DEVICE, HOST),
    (2, 10, 10, 1, False, F32P, HOST, HOST),     # uniform 1024 planar: k_mid
    (6, 10, 10, 0, False, I16P, DEVICE, DEVICE),
    (8, 10, 10, 2, True, F32P, HOST, DEVICE),
    (2, 9, 9, 2, False, I16P, DEVICE, HOST),     # uniform 512 planar: k_mid
    (1, 9, 9, 1, True, F32P, HOST, HOST),
    (2, 10, 10, 0, False, I16I, HOST, HOST),     # uniform 1024 / 512 interleaved: k_chain
    (6, 9, 9, 1, False, F32I, DEVICE, DEVICE),
    (2, 8, 10, 0, True, F32P, HOST, HOST),       # other blocksize pairs
    (6, 8, 10, 2, False, I16I, DEVICE, DEVICE),
    (8, 8, 10, 1, True, I16P, HOST, DEVICE),
    (1, 7, 12, 1, False, I16P, HOST, DEVICE),
    (6, 7, 12, 2, True, F32P, DEVICE, HOST),     # 6 x 2048 accumulators: the VQ limit
    (2, 6, 13, None, False, F32I, HOST, HOST),
    (1, 6, 13, 2, True, I16P, DEVICE, DEVICE),
]


@pytest.mark.parametrize("channels,bs0,bs1,rtype,records,fmt,memory,floor_mem", CASES)
def test_vq_batches_match_the_oracle_and_the_dense_entry(ctx, oracle, channels, bs0, bs1, rtype, records, fmt, memory, floor_mem):
    seed = 9000 + 97 * channels + 13 * bs0 + bs1 + 5 * fmt + (7 if records else 0)
    S, P, K = 3, 4, 3
    st = Streams(seed, channels, bs0, bs1, rtype, records, S, P * K, p_short=0.1 if bs0 == 8 and planar(fmt) else 0.3)
    su = st.hdr.make_setup(ctx, floor0=records)
    twins = st.twins(oracle)
    batches = [Batch(st, k * P, (k + 1) * P, fmt, twins) for k in range(K)]
    runs = {}
    generic = {"LWB_FORCE_GENERIC": "1"}
    for name, entry, env in (("vq", VQ, None), ("residue", RESIDUE, None), ("four-kernel", VQ, generic),
                             ("four-kernel residue", RESIDUE, generic)):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        outs = []
        with environ(env):
            for k, b in enumerate(batches):
                # device floor arrays cannot be looked at: the batch may carry records whenever the setup has them
                floor0 = records and (floor_mem == DEVICE or b.has_records)
                # (a batch of an 8/10 stream whose packets are all long and full-window is k_mid's as well)
                shape = "mid" if b.uniform and bs1 >= 9 and planar(fmt) else "chain"
                expect = (vq_kernels(shape, floor0) if name == "vq" else
                          (FOUR_KERNEL, {"k_chain", "k_mid"}) if env else None)
                pcm, chains = b.run(ctx, pwrs, entry, memory, floor_mem, expect)
                b.check_oracle(oracle, pcm, chains, (name, k))
                outs.append(pcm)
        states = [p.data() for p in pwrs]
        for s, (p, tw) in enumerate(zip(states, twins)):
            w = tw.pwr.data()
            assert (p is None) == (w is None) and (p is None or bits_equal(p, w)), (name, "state", s)
        runs[name] = outs
        for p in pwrs:
            p.close()
    for k in range(K):
        assert runs["vq"][k].tobytes() == runs["residue"][k].tobytes(), ("VQ and dense residue entry differ", k)
        assert runs["four-kernel"][k].tobytes() == runs["four-kernel residue"][k].tobytes(), ("the entries differ on the four-kernel path", k)
        assert same_but_nan_signs(runs["vq"][k], runs["four-kernel"][k]), ("VQ batch differs on the four-kernel path", k)


# ---------------------------------------------------------------------------------------------------------------------
# 3: a host-memory VQ submit with interleaved output does not wait for the device
# ---------------------------------------------------------------------------------------------------------------------
def test_vq_interleaved_submits_return_behind_queued_work(ctx, oracle):
    """Three host-memory VQ batches (256/2048 stereo, i16 interleaved, page-locked arrays) submitted behind a gate on the
    context's stream: every lwb_submit_chains returns while the gate is closed, before the first ticket completes; the
    tickets complete in order, with the PCM of the synchronous calls and the oracle's.  (An ungated pass first, so
    that no arena grows in the gated one.)"""
    S, P, K = 4, 5, 3
    st = Streams(9500, 2, 8, 11, None, False, S, P * K, p_short=0.1)
    su = st.hdr.make_setup(ctx)
    twins = st.twins(oracle)
    batches = [Batch(st, k * P, (k + 1) * P, I16I, twins) for k in range(K)]
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    sync = []
    for b in batches:
        pcm, chains = b.run(ctx, pwrs, VQ, HOST, HOST, ({"k_chain": 1}, ALL_KERNELS - {"k_chain"}))
        b.check_oracle(oracle, pcm, chains, "synchronous")
        sync.append(pcm)
    for p in pwrs:
        p.close()

    def pinned(a):
        out = ctx.host_alloc(a.shape, a.dtype)
        out[...] = a
        return out

    def submit_pass(gate):
        # (one call per pass: its page-locked arrays are freed when it returns, not behind the next gate -- cudaFreeHost
        # waits for the device)
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        calls = []
        for b in batches:
            calls.append((b, b.chains(pwrs), [pinned(x) for x in (b.kinds, b.ys, *b.vq)],
                          fill_guard(ctx.host_alloc(b.n_out, np.int16))))
        torch.cuda.synchronize()
        if gate:
            gate.close()
        tickets = []
        for b, chains, (kd, y, rr, ro, ee, eo), pcm in calls:
            with expect_kernels(ctx, ran={"k_chain": 1}, not_ran=ALL_KERNELS - {"k_chain"}):
                tickets.append(ctx.submit_chains(chains, VQ, HOST, None, pcm, I16I, floor_kind=kd, floor1_y=y, vq=(rr, ro, ee, eo)))
        if gate:
            gate.assert_closed("VQ interleaved")
            assert not tickets[0].done(), "the first ticket completed before the gate opened"
            for _, _, _, pcm in calls:
                assert np.all(pcm.view(np.uint16) == fill_guard(pcm.copy()).view(np.uint16)), "PCM landed before the gate opened"
        for k, t in enumerate(tickets):
            t.wait()
            assert all(u.done() for u in tickets[:k + 1])
        for k, (b, chains, _, pcm) in enumerate(calls):
            b.check_oracle(oracle, pcm, chains, ("submitted", gate is not None, k))
            assert pcm.tobytes() == sync[k].tobytes(), ("submitted batch differs from the synchronous call", gate is not None, k)
        for s, tw in enumerate(twins):
            assert bits_equal(pwrs[s].data(), tw.pwr.data()), ("state", gate is not None, s)
        for p in pwrs:
            p.close()

    submit_pass(None)
    submit_pass(Gate(ctx))


# ---------------------------------------------------------------------------------------------------------------------
# 4: prepared device-memory VQ batches on k_mid
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bs,floor_mem", [(10, DEVICE), (9, HOST)])
def test_prepared_vq_mid_batch_replays(ctx, oracle, bs, floor_mem):
    """A device-memory VQ Batch of uniform 1024- (512-) point streams, run five times on the same streams: the first
    two runs plan (the streams change shape after the first), the rest replay the captured front stages and k_mid,
    FRONT | {k_mid} once each.  Every run's PCM equals a fresh lwb_decode_chains of the same packets on twin streams,
    and the oracle's."""
    S, P, R = 3, 5, 5
    st = Streams(9600 + bs, 2, bs, bs, None, False, S, P)
    su = st.hdr.make_setup(ctx)
    twins = st.twins(oracle)
    b = Batch(st, 0, P, F32P)
    # the fresh decodes first (and the oracle's), so that the prepared runs find every arena grown
    fresh = [L.PreviousWindowRight(su) for _ in range(S)]
    wants = []
    for r in range(R):
        pcm, fresh_chains = b.run(ctx, fresh, VQ, HOST, HOST, vq_kernels("mid", False))
        b.wants = [np.concatenate([st.oracle_packet(twins[s], info, nb) for _, info, nb in st.packets[s]], axis=1)
                   for s in range(S)]
        b.check_oracle(oracle, pcm, fresh_chains, ("fresh", r))
        wants.append((pcm, [(c.status, c.n_samples) for c in fresh_chains]))
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    chains = b.chains(pwrs)
    frees = []

    def dev(a):
        a = np.ascontiguousarray(a)
        p = ctx.device_alloc(max(a.nbytes, 16))
        ctx.h2d(p, a)
        frees.append(p)
        return p

    try:
        d_pcm = ctx.device_alloc(b.n_out * 4)
        frees.append(d_pcm)
        kw = dict(floor_kind=b.kinds, floor1_y=b.ys, vq=b.vq)
        if floor_mem == DEVICE:
            kw = dict(floor_kind=dev(b.kinds), floor1_y=dev(b.ys), vq=tuple(dev(x) for x in b.vq), floor_memory=DEVICE)
        prepared = L.Batch(ctx, chains, VQ, DEVICE, None, d_pcm, F32P, **kw)
        for r in range(R):
            ctx.h2d(d_pcm, fill_guard(np.empty(b.n_out, np.float32)))
            steady = r >= 2
            with expect_kernels(ctx, *(({"k_floor1_segments": 1, "k_prologue_fused": 1, "k_mid": 1},
                                        ALL_KERNELS - FRONT - {"k_mid"}) if steady else ((), ()))):
                prepared.run()
            ctx.synchronize()
            prepared.collect()
            got = np.empty(b.n_out, np.float32)
            ctx.d2h(got, d_pcm)
            assert got.tobytes() == wants[r][0].tobytes(), ("prepared run differs from a fresh decode", r)
            assert [(c.status, c.n_samples) for c in chains] == wants[r][1], r
        prepared.close()
    finally:
        for p in frees:
            ctx.device_free(p)
    for s in range(S):
        assert bits_equal(pwrs[s].data(), twins[s].pwr.data()), ("state", s)


# ---------------------------------------------------------------------------------------------------------------------
# 5: the front half's batcher
# ---------------------------------------------------------------------------------------------------------------------
def test_stream_batcher_vq_interleaved_i16(ctx, oracle):
    """StreamBatcher(entry=VQ) on a 256/2048 stream with i16 interleaved output: the same bytes as the dense-entry
    batcher and the oracle's, synthesised by k_chain alone."""
    S, P = 6, 9
    st = Streams(9700, 2, 8, 11, None, False, 3, P)
    su = st.hdr.make_setup(ctx)
    want = []
    for s in range(3):
        tw = st.twins(oracle)[0]
        want.append(np.concatenate([st.oracle_packet(tw, info, nb) for _, info, nb in st.packets[s]], axis=1))
    stride = P * 1024
    out = {}
    for entry in (VQ, RESIDUE):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        jobs = [(pwrs[j], [pk for pk, _, _ in st.packets[j % 3]]) for j in range(S)]
        pcm = fill_guard(np.empty(S * 2 * stride, np.int16))
        bt = fe.StreamBatcher(ctx, st.hdr, threads=2, entry=entry)
        with expect_kernels(ctx, ran=("k_chain",), not_ran=ALL_KERNELS - {"k_chain"}):
            res = bt.decode(jobs, pcm, stride, out_format=I16I)
        bt.close()
        for j in range(S):
            w = want[j % 3]
            n = w.shape[1]
            assert res[j] == (n, P, 0), (entry, j, res[j])
            got = pcm[j * 2 * stride:j * 2 * stride + 2 * n].reshape(n, 2).T
            assert np.array_equal(got, oracle.quantise_i16(w)), (entry, j)
        out[entry] = pcm
        for p in pwrs:
            p.close()
    assert out[VQ].tobytes() == out[RESIDUE].tobytes()

"""Inverse coupling at every site that decouples (coupling_cases.py), on the GPU, against the oracle and the numpy
restatement:

  * every batch site (S1-S3, S6-S9): a batch of one stream per mapping of its case, the residues carrying probe columns
    that give every coupling step every finite (magnitude, angle) class pair and, one per packet, non-finite ones;
    floor 1, dense and unused floors mixed within packets.  f32 PCM bit for bit (bits_equal), i16 exactly, end states
    bit for bit, and the kernels of the site's row ran;
  * the cross-packet hand-over of k_prologue_fused's pipelined loop (S1, S2): more than 2 x grid packets in one launch,
    consecutive packets of each CTA differing in mapping, block size and floor kinds;
  * lwb_debug_packet_taps' post_inverse (S10) bit for bit against the restatement at 1-12 channels, on a fresh context
    and after a larger batch has used the context's IMDCT scratch;
  * lwb_setup_create refuses a mapping with magnitude == angle, a channel index past the channels or more than
    LWB_MAX_COUPLING steps, and creates no setup."""
import ctypes as C

import numpy as np
import pytest
import torch

import coupling_cases as cc
import lewton_b200 as L
from helpers import FUSED, RefStream, bits_equal, environ, expect_kernels, launches_are_attributed, make_setup, mismatch_report
import vorbis_packer as vp
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

FLOORS = [(1, [0, 256, 64, 128, 16, 200]), (3, [0, 128, 40, 90])]


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def _mappings(case):
    return [{"coupling": mp, "floor_of_channel": [c % 2 for c in range(case.C)]} for mp in case.mappings]


def _modes(case):
    return [(bf, i) for i in range(len(case.mappings)) for bf in (0, 1)]      # mode 2i short, 2i + 1 long, mapping i


def _packet(rng, case, n2, kinds, res):
    """floors of one packet (per channel: y values, a dense curve or None) for kinds [C]."""
    fl = []
    for c, k in enumerate(kinds):
        if k == cc.FLOOR_ONE:
            mult, xs = FLOORS[c % 2]
            fl.append([int(v) for v in rng.integers(0, [256, 128, 86, 64][mult - 1], len(xs))])
        elif k == cc.FLOOR_DENSE:
            fl.append((rng.random(n2) + 0.1).astype(np.float32))
        else:
            fl.append(None)
    return fl


class Streams:
    """Chains of packets of one case: per chain its modes, flags, residues, floors, the oracle's PCM and end state."""

    def __init__(self, ctx, oracle, case, chains):
        """chains: per chain [(mode, residue [C][n/2], floor kinds [C])]."""
        self.case = case
        self.su = make_setup(ctx, case.C, case.bs0, case.bs1, modes=_modes(case), mappings=_mappings(case), floors=FLOORS)
        self.refs, self.seqs, self.wants = [], [], []
        self.coeffs, self.dense, self.kinds, self.ys, self.sizes = [], [], [], [], []
        self.hit = {"unused over nonzero": False, "kinds differ within a step": False}
        modes = _modes(case)
        rng = np.random.default_rng(len(case.name) * 31 + case.C)
        for chain in chains:
            mids = [m for m, _, _ in chain]
            bf = np.array([modes[m][0] for m in mids], np.uint8)
            prev, nxt = cc.window_flags(bf)
            ref = RefStream(oracle, case.C, case.bs0, case.bs1, modes, _mappings(case), FLOORS)
            parts, size = [], 0
            for i, (m, res, kinds) in enumerate(chain):
                n2 = (1 << (case.bs1 if bf[i] else case.bs0)) // 2
                assert res.shape == (case.C, n2)
                mp = case.mappings[modes[m][1]]
                fl = _packet(rng, case, n2, kinds, res)
                self.hit["unused over nonzero"] |= any(k == cc.FLOOR_UNUSED and np.any(res[c] != 0) for c, k in enumerate(kinds))
                self.hit["kinds differ within a step"] |= any(kinds[a] != kinds[b] for a, b in mp)
                rc, o = ref.packet(int(m), int(prev[i]), int(nxt[i]), res, fl)
                assert rc == 0
                parts.append(o)
                k_, y_, d_ = L.DecodedPacket(int(m), res, fl).pack()
                self.kinds.append(k_)
                self.ys.append(y_)
                self.dense.append((d_ if d_ is not None else np.zeros_like(res)).ravel())
                self.coeffs.append(res.ravel())
                size += res.size
            self.refs.append(ref)
            self.wants.append(np.concatenate(parts, axis=1))
            self.seqs.append((np.array(mids, np.uint8), prev, nxt))
            self.sizes.append(size)
        self.n_pk = sum(len(c) for c in chains)

    def run(self, ctx, fmt, ran, not_ran, env=None):
        """Decodes every chain from empty streams in device memory (the residue arena one element past a 16-byte boundary
        when the case asks) and checks the PCM and end states against the oracle's."""
        case, Cn = self.case, self.case.C
        planar = fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR)
        pwrs = [L.PreviousWindowRight(self.su) for _ in self.seqs]
        chains, coff, ooff, row = [], 1 if case.misalign else 0, 0, 0
        for s, (mids, prev, nxt) in enumerate(self.seqs):
            n = self.wants[s].shape[1]
            stride = (n + 3) & ~3
            chains.append(L.ChainSpec(pwrs[s], mids, prev, nxt, coeff_offset=coff, packet_index=row, out_offset=ooff,
                                      out_stride=stride if planar else 0))
            coff += self.sizes[s]
            ooff += Cn * (stride if planar else n)
            row += len(mids)
        pad = np.zeros(1 if case.misalign else 0, np.float32)
        coeffs, dense = np.concatenate([pad] + self.coeffs), np.concatenate([pad] + self.dense)
        dt = np.float32 if fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED) else np.int16
        pcm = np.zeros(max(ooff, 4), dt)
        bufs = [ctx.device_alloc(a.nbytes) for a in (coeffs, dense, pcm)]
        try:
            for p, a in zip(bufs, (coeffs, dense, pcm)):
                ctx.h2d(p, a)
            with environ(env), expect_kernels(ctx, ran=ran, not_ran=not_ran):
                L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_DEVICE, bufs[0], bufs[2], fmt,
                                floor_kind=np.concatenate(self.kinds), floor1_y=np.concatenate(self.ys), dense_floor=bufs[1])
            ctx.synchronize()
            ctx.d2h(pcm, bufs[2])
        finally:
            for p in bufs:
                ctx.device_free(p)
        for s, c in enumerate(chains):
            w = self.wants[s]
            n = w.shape[1]
            assert (c.status, c.n_samples) == (0, n), (case, s, c.status, c.n_samples, n)
            got = (np.stack([pcm[c.out_offset + k * c.out_stride:][:n] for k in range(Cn)]) if planar
                   else pcm[c.out_offset:c.out_offset + n * Cn].reshape(n, Cn).T)
            if dt == np.float32:
                assert bits_equal(got, w), (case, s, case.mappings[s % len(case.mappings)], mismatch_report(got, w))
            else:
                assert np.array_equal(got, self.refs[0].o.quantise_i16(w)), (case, s)
            a, b = pwrs[s].data(), self.refs[s].pwr.data()
            assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (case, s, "state")
        for p in pwrs:
            p.close()


# ---------------------------------------------------------------------------------------------------------------------
# every batch site
# ---------------------------------------------------------------------------------------------------------------------
def site_chains(case, rng):
    """Per mapping of the case: a chain of its finite probes (floor 1 and dense floors only, every bin finite after
    decoupling, so every probe shows in the PCM) and a chain of its non-finite probes, one per packet, with unused
    floors among the others."""
    n0, n1 = (1 << case.bs0) // 2, (1 << case.bs1) // 2
    chains, j = [], 0
    for i, mp in enumerate(case.mappings):
        fin, nf = cc.mapping_pool(case.C, mp)
        for packets, unused in ((cc.finite_chain(rng, case.C, fin, n0, n1), False), (cc.nonfinite_chain(rng, case.C, nf, n0, n1), True)):
            if packets:
                chains.append([(2 * i + bf, res, [cc.floor_kind(j + k, c, unused) for c in range(case.C)])
                               for k, (bf, res) in enumerate(packets)])
                j += len(packets)
    return chains


@pytest.mark.parametrize("case", cc.cases(), ids=repr)
def test_site_matches_the_oracle(ctx, oracle, case):
    _, ran, not_ran = cc.SITES[case.site]
    st = Streams(ctx, oracle, case, site_chains(case, np.random.default_rng(case.C * 7 + len(case.mappings))))
    assert all(st.hit.values()) or case.C == 1, (case, st.hit)
    f32 = cabi.OUT_F32_INTERLEAVED if case.interleaved else cabi.OUT_F32_PLANAR
    i16 = cabi.OUT_I16_INTERLEAVED if case.interleaved else cabi.OUT_I16_PLANAR
    for fmt in (f32, i16):
        st.run(ctx, fmt, set(ran), set(not_ran), case.env)


# ---------------------------------------------------------------------------------------------------------------------
# the pipelined loop's hand-over from packet to packet
# ---------------------------------------------------------------------------------------------------------------------
def handover_layout(C, mappings):
    """(packets, grid, modes, n_chains) of a hand-over batch over the device's SM count: more than 2 x grid packets,
    modes dealt by coupling_cases.handover_modes."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    S = 16
    n_pk = 2 * sm * 8 + 16 * S
    grid = cc.pf_grid(n_pk, C, sm)
    assert n_pk > 2 * grid
    return n_pk, grid, cc.handover_modes(n_pk, grid, 2 * len(mappings)), S


def assert_cta_neighbours_differ(case, modes, grid, kinds=None, min_kinds=0.9):
    """Entries j and j + grid of the packet list (CTA j % grid decodes both, one after the other) differ in mapping and
    block size in over 90 % of pairs, and in floor kinds (a row's) in more than min_kinds of them."""
    md = _modes(case)
    maps, bfs = np.array([md[m][1] for m in modes]), np.array([md[m][0] for m in modes])
    a, b = slice(0, len(modes) - grid), slice(grid, len(modes))
    assert ((maps[a] != maps[b]) & (bfs[a] != bfs[b])).mean() > 0.9
    if kinds is not None:
        frac = np.any(kinds[a] != kinds[b], axis=1).mean()
        assert frac > min_kinds, frac
    steps = {len(case.mappings[m]) for m in maps}
    assert 0 in steps and 1 in steps and max(steps) >= 2, "test should run both branches of k_prologue_fused"


def test_pipelined_loop_hands_every_packet_its_own_header_and_residue(ctx, oracle):
    """Stereo 256/2048 packets of every S1 and S2 mapping through the four-kernel path on aligned arenas: one front-stage
    launch over the batch.  run_generic lists the packets chain by chain, each chain's in order
    (path_generic.cuh:897-936), so packet j is entry j of the list and CTA b of k_prologue_fused's grid decodes entries
    b, b + grid, ...  Modes and floor kinds are dealt so that entries j and j + grid differ in mapping (and with it the
    step count or orientation), block size and every channel's floor kind.  Every bin is finite (the finite probes of
    each mapping, cycled), so a packet decoded with another packet's header or residue shows in the PCM."""
    case = cc.Case("handover", "S1", 2, cc.STEREO + cc.STEREO_MULTI)
    n_pk, grid, modes, S = handover_layout(2, case.mappings)
    kinds = np.array([[cc.floor_kind(j % grid + j // grid, c, unused=False) for c in range(2)] for j in range(n_pk)])
    assert_cta_neighbours_differ(case, modes, grid, kinds, 0.99)
    md = _modes(case)
    pools = [cc.mapping_pool(2, mp)[0] for mp in case.mappings]
    rng = np.random.default_rng(77)
    packets = []
    for j, m in enumerate(modes):
        bf, i = md[m]
        n2 = (1 << (case.bs1 if bf else case.bs0)) // 2
        fin = pools[i]
        res = (rng.standard_normal((2, n2)) * 0.5).astype(np.float32)
        if fin.shape[1]:
            k = min(n2 - 8, fin.shape[1])
            res[:, 4:4 + k] = np.roll(fin, -(j * 37) % fin.shape[1], axis=1)[:, :k]
        assert np.isfinite(cc.decouple(res, case.mappings[i])).all()
        packets.append((int(m), res, kinds[j].tolist()))
    per = n_pk // S
    st = Streams(ctx, oracle, case, [packets[s * per:(s + 1) * per if s + 1 < S else n_pk] for s in range(S)])
    assert st.n_pk == n_pk
    st.run(ctx, cabi.OUT_F32_PLANAR, {"k_floor1_segments": 1, "k_prologue_fused": 1, "k_imdct": 1},
           FUSED | {"k_prologue", "k_chain"}, cc.GENERIC_ENV)


# ---------------------------------------------------------------------------------------------------------------------
# the debug tap
# ---------------------------------------------------------------------------------------------------------------------
def _tap_all(su, case, pwr):
    """post_inverse of every mapping's probe columns (all 64 class pairs a step can take), long blocks, vs numpy."""
    n2 = (1 << case.bs1) // 2
    for i, mp in enumerate(case.mappings):
        probes = cc.probe_columns(case.C, mp)
        cols = [col for s in probes for col in probes[s].values()]
        cols = np.stack(cols, axis=1) if cols else np.zeros((case.C, 0), np.float32)
        rng = np.random.default_rng(i)
        for k0 in range(0, max(cols.shape[1], 1), n2):
            res = (rng.standard_normal((case.C, n2)) * 0.5).astype(np.float32)
            part = cols[:, k0:k0 + n2]
            res[:, :part.shape[1]] = part
            post, _, _ = L.debug_taps(su, L.DecodedPacket(2 * i + 1, res, [None] * case.C), pwr)
            want = cc.decouple(res, mp)
            assert np.all(cc.same_bits(post, want)), (case, i, k0, int((~cc.same_bits(post, want)).sum()))


@pytest.mark.parametrize("case", cc.tap_cases(), ids=repr)
def test_debug_tap_post_inverse_on_a_fresh_context_and_after_a_batch(oracle, case):
    c = L.Context(0)
    try:
        su = make_setup(c, case.C, case.bs0, case.bs1, modes=_modes(case), mappings=_mappings(case), floors=FLOORS)
        pwr = L.PreviousWindowRight(su)
        _tap_all(su, case, pwr)
        # a spectrum batch of 6 long blocks on the four-kernel path grows and fills the IMDCT scratch the tap reuses
        n2 = (1 << case.bs1) // 2
        spec = np.random.default_rng(1).standard_normal(6 * case.C * n2).astype(np.float32)
        pcm = np.zeros(6 * case.C * n2, np.float32)
        other = L.PreviousWindowRight(su)
        with environ(cc.GENERIC_ENV):
            L.decode_chains(c, [L.ChainSpec(other, np.ones(6, np.uint8), out_stride=6 * n2)], cabi.ENTRY_SPECTRUM,
                            cabi.MEM_HOST, spec, pcm, cabi.OUT_F32_PLANAR)
        assert np.isfinite(pcm).all() and np.any(pcm != 0)
        _tap_all(su, case, pwr)
        assert pwr.is_empty()
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# mappings lwb_setup_create refuses
# ---------------------------------------------------------------------------------------------------------------------
def _create(ctx, channels, coupling, steps=None):
    d = cabi.SetupDesc()
    d.audio_channels, d.blocksize_0, d.blocksize_1 = channels, 8, 11
    fl = (cabi.FloorDesc * 1)()
    fl[0].floor_type, fl[0].floor1_multiplier, fl[0].floor1_values = cabi.FLOOR_TYPE_ONE, 1, 2
    fl[0].floor1_x_list[0], fl[0].floor1_x_list[1] = 0, 128
    mp = (cabi.MappingDesc * 1)()
    mp[0].coupling_steps = len(coupling) if steps is None else steps
    mp[0].submaps = 1
    for k, (m, a) in enumerate(coupling):
        mp[0].magnitudes[k], mp[0].angles[k] = m, a
    md = (cabi.ModeDesc * 1)()
    md[0].blockflag, md[0].mapping = 1, 0
    d.n_floors, d.floors, d.n_mappings, d.mappings, d.n_modes, d.modes = 1, fl, 1, mp, 1, md
    h = C.c_void_p()
    rc = cabi.lib().lwb_setup_create(ctx._h, C.byref(d), C.byref(h))
    return rc, h


def test_setup_create_refuses_bad_coupling_steps(ctx):
    good = cc.max_steps(np.random.default_rng(3), 8)
    rc, h = _create(ctx, 8, good)
    assert rc == cabi.OK and h.value
    cabi.lib().lwb_setup_destroy(h)
    for channels, coupling, steps in ((2, [(0, 1), (1, 1)], None),          # magnitude == angle
                                      (2, [(0, 2)], None),                  # angle past the channels
                                      (3, [(3, 0), (0, 1)], None),          # magnitude past the channels
                                      (8, good, cc.MAX_COUPLING + 1)):      # one step too many
        rc, h = _create(ctx, channels, coupling, steps)
        assert rc == cabi.ERR_BAD_FORMAT and not h.value, (channels, coupling[:3], steps, rc)


# ---------------------------------------------------------------------------------------------------------------------
# the VQ entry (S4, S5)
# ---------------------------------------------------------------------------------------------------------------------
class VqStreams:
    """Packer-made streams of one VQ case (tests/vorbis_packer.py, its coupling lists fixed to the case's, mode 2i short
    and 2i + 1 long of mapping i).  Packets are packed per (mode, flags) into a pool of `pool` and reused, so that long
    chains stay cheap to build; chains: per chain its mode numbers.  Holds per packet the frontend's dense decode and VQ
    records and the oracle's PCM of what the packer encoded."""

    def __init__(self, ctx, oracle, case, chains, seed, pool=4):
        for k in range(40):
            rng = np.random.default_rng(seed + 1000 * k)
            spec = vp.StreamSpec(rng, channels=case.C, bs0=case.bs0, bs1=case.bs1, residue_types=[1 + k % 2],
                                 couplings=case.mappings)
            hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
            if hdr.vq_capable():
                break
            hdr.close()
        else:
            raise AssertionError("no VQ-capable draw")
        assert [m["coupling"] for m in spec.mappings] == case.mappings and spec.modes == _modes(case)
        self.case, self.hdr, self.spec = case, hdr, spec
        self.su = hdr.make_setup(ctx)
        floors = [(f.multiplier, f.x_list) for f in spec.floors]
        maps = [{"coupling": m["coupling"], "floor_of_channel": [m["floors"][m["mux"][c]] for c in range(case.C)]}
                for m in spec.mappings]
        cache = {}
        coeffs, kinds, ys, runs, ents, roffs, eoffs = [], [], [], [], [], [0], [0]
        self.refs, self.seqs, self.wants, self.sizes, self.raw = [], [], [], [], []
        j = 0
        for mids in chains:
            bf = np.array([spec.modes[m][0] for m in mids], np.uint8)
            prev, nxt = cc.window_flags(bf)
            ref = RefStream(oracle, case.C, case.bs0, case.bs1, spec.modes, maps, floors)
            parts, size = [], 0
            for i, m in enumerate(mids):
                key = (int(m), int(prev[i]), int(nxt[i]), j % pool)
                if key not in cache:
                    pk, info = spec.audio_packet(*key[:3], p_unused=0.3)
                    fl_exp, res = spec.expected(info)
                    cache[key] = (hdr.decode_packet(pk), hdr.decode_packet_vq(pk)[1:], [None if f is None else list(f[1]) for f in fl_exp], res)
                d, (rr, ee), fl, res = cache[key]
                rc, o = ref.packet(int(m), int(prev[i]), int(nxt[i]), res, fl)
                assert rc == 0
                parts.append(o)
                k_, y_, dn = d.pack()
                assert dn is None
                kinds.append(k_)
                ys.append(y_)
                coeffs.append(d.residue.ravel())
                self.raw.append((int(m), d.residue))
                runs.append(rr)
                ents.append(ee)
                roffs.append(roffs[-1] + len(rr))
                eoffs.append(eoffs[-1] + len(ee))
                size += d.residue.size
                j += 1
            self.refs.append(ref)
            self.wants.append(np.concatenate(parts, axis=1))
            self.seqs.append((np.array(mids, np.uint8), prev, nxt))
            self.sizes.append(size)
        self.coeffs, self.kinds, self.ys = np.concatenate(coeffs), np.concatenate(kinds), np.concatenate(ys)
        self.vq = (np.concatenate(runs) if roffs[-1] else np.zeros(1, fe.VQ_RUN_DTYPE), np.array(roffs, np.uint64),
                   np.concatenate(ents).astype(np.uint16) if eoffs[-1] else np.zeros(1, np.uint16), np.array(eoffs, np.uint64))

    def run(self, ctx, entry):
        """One planar f32 batch from empty streams, device memory, on the four-kernel path: the PCM, checked against the
        oracle (and the end states)."""
        Cn = self.case.C
        pwrs = [L.PreviousWindowRight(self.su) for _ in self.seqs]
        chains, coff, ooff, row = [], 0, 0, 0
        for s, (mids, prev, nxt) in enumerate(self.seqs):
            stride = (self.wants[s].shape[1] + 3) & ~3
            chains.append(L.ChainSpec(pwrs[s], mids, prev, nxt, coeff_offset=coff, packet_index=row, out_offset=ooff, out_stride=stride))
            coff += self.sizes[s]
            ooff += Cn * stride
            row += len(mids)
        pcm = np.zeros(max(ooff, 4), np.float32)
        bufs = [ctx.device_alloc(a.nbytes) for a in (self.coeffs, pcm)]
        try:
            ctx.h2d(bufs[0], self.coeffs)
            ctx.h2d(bufs[1], pcm)
            kw = dict(floor_kind=self.kinds, floor1_y=self.ys)
            if entry == cabi.ENTRY_VQ:
                kw["vq"] = self.vq
            with environ(cc.GENERIC_ENV), expect_kernels(ctx, ran={"k_floor1_segments": 1, "k_prologue_fused": 1, "k_imdct": 1},
                                                         not_ran=FUSED | {"k_prologue", "k_chain", "k_floor0_curves"}):
                L.decode_chains(ctx, chains, entry, cabi.MEM_DEVICE, None if entry == cabi.ENTRY_VQ else bufs[0], bufs[1],
                                cabi.OUT_F32_PLANAR, **kw)
            ctx.synchronize()
            ctx.d2h(pcm, bufs[1])
        finally:
            for p in bufs:
                ctx.device_free(p)
        for s, c in enumerate(chains):
            w = self.wants[s]
            n = w.shape[1]
            assert (c.status, c.n_samples) == (0, n), (self.case, s, c.status, c.n_samples, n)
            got = np.stack([pcm[c.out_offset + k * c.out_stride:][:n] for k in range(Cn)])
            assert bits_equal(got, w), (self.case, entry, s, mismatch_report(got, w))
            a, b = pwrs[s].data(), self.refs[s].pwr.data()
            assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (self.case, s, "state")
        for p in pwrs:
            p.close()
        return pcm

    def step_input_problems(self):
        """What the accumulators give each step: the sums start at +0, so no step input may be -0 (nor inf / NaN).
        Returns the steps that get one, or that see no nonzero value or no zero (the signs of the nonzero values are
        the codebooks' draw), as [(mapping, step, class pairs)]."""
        out = []
        for i, mp in enumerate(self.case.mappings):
            res = [r for m, r in self.raw if self.spec.modes[m][1] == i]
            if not res:
                out.append((i, None, "no packet"))
                continue
            for s, pairs in cc.step_classes(np.concatenate(res, axis=1), mp).items():
                if (not pairs <= {(a, b) for a in (0, 1, 2) for b in (0, 1, 2)} or not any(0 in p or 1 in p for p in pairs)
                        or not any(2 in p for p in pairs)):
                    out.append((i, s, sorted(pairs)))
        return out

    def close(self):
        self.hdr.close()


def _vq_both_entries(ctx, st):
    """The VQ batch and the dense residue entry of the same packets: each equal to the oracle, and byte for byte to each
    other."""
    vq = st.run(ctx, cabi.ENTRY_VQ)
    dense = st.run(ctx, cabi.ENTRY_RESIDUE)
    assert vq.tobytes() == dense.tobytes(), (st.case, "VQ and dense residue entry differ")


@pytest.mark.parametrize("case", cc.vq_cases(), ids=repr)
def test_vq_site_matches_the_oracle_and_the_dense_entry(ctx, oracle, case):
    # two chains per mapping, 8 packets each (long, short, long, long, short, ...)
    chains = [[2 * i + cc._block(k) for k in range(8)] for i in range(len(case.mappings)) for _ in range(2)]
    for k in range(8):           # a draw whose codebooks and submaps give every step nonzero values
        st = VqStreams(ctx, oracle, case, chains, seed=12000 + 17 * case.C + len(case.mappings) + 101 * k)
        bad = st.step_input_problems()
        if not bad:
            break
        st.close()
    assert not bad, (case, bad)
    try:
        _vq_both_entries(ctx, st)
    finally:
        st.close()


def test_vq_serial_loop_hands_every_packet_its_own_header(ctx, oracle):
    """The hand-over batch of the VQ entry: stereo 256/2048 packets of every S4 and S5 mapping, more than 2 x grid in one
    k_prologue_fused<true> launch (the four-kernel path lists them as in the dense hand-over test).  The packer draws the
    floors (30 % unused), so the floor kinds of CTA neighbours differ only by chance."""
    case = cc.Case("vq_handover", "S4", 2, cc.STEREO + cc.STEREO_MULTI, env=cc.GENERIC_ENV)
    n_pk, grid, modes, S = handover_layout(2, case.mappings)
    per = n_pk // S
    st = VqStreams(ctx, oracle, case, [modes[s * per:(s + 1) * per if s + 1 < S else n_pk].tolist() for s in range(S)], seed=13000)
    try:
        assert len(st.raw) == n_pk
        # the accumulators start at +0: no step input is -0, inf or NaN
        assert all(p <= {(a, b) for a in (0, 1, 2) for b in (0, 1, 2)} for i, mp in enumerate(case.mappings)
                   for p in cc.step_classes(np.concatenate([r for m, r in st.raw if m // 2 == i], axis=1), mp).values())
        assert_cta_neighbours_differ(case, modes, grid, st.kinds.reshape(n_pk, 2), 0.25)
        _vq_both_entries(ctx, st)
    finally:
        st.close()

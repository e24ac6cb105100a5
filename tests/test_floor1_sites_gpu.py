"""Floor type 1 at every site that builds the curve on the device (floor1_cases.py, F1-F6), on the post layouts that
reach each site's edges, against the oracle:

  * every batch site: one setup whose floors are the layouts (mapping i puts layout i + c on channel c), batches of
    packets cycling through the mappings and both block sizes; f32 PCM bit for bit (bits_equal), i16 exactly, end states
    bit for bit, and the kernels of the site ran (expect_kernels);
  * F1: SHIFT and non-SHIFT rows, short and long rows in one front-stage launch of more than 2 x grid packets, the
    64/8192 extremes, and the one-pass 256/2048 schedule;  F2 / F4: the VQ entry on packer-made streams whose floors are
    the layouts a header can carry, its PCM equal byte for byte to the dense residue entry's on the same packets;
  * the curve itself: lwb_debug_packet_taps' pre_mdct under a residue of 1.0 and no coupling equals
    inverse_db[walk] exactly, at 1 to 8 channels (F5) and 9 to 12 (F6);
  * lwb_setup_create refuses x lists whose post 0 is not at x = 0, creates no setup, and takes every list the header
    parser makes."""
import ctypes as C

import numpy as np
import pytest
import torch

import coupling_cases as cc
import floor1_cases as fc
import lewton_b200 as L
import vorbis_packer as vp
from helpers import FUSED, RefStream, bits_equal, environ, expect_kernels, launches_are_attributed, mismatch_report
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

FLOOR_UNUSED, FLOOR_ONE, FLOOR_DENSE = cc.FLOOR_UNUSED, cc.FLOOR_ONE, cc.FLOOR_DENSE


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def site_layouts(bs0, bs1, seed=0):
    """The layouts of a setup of blocksizes (bs0, bs1): every layout built for the long block's n/2, and the long x list
    built for the short block's too (its segment over the short block's last bin longer than 4096 bins)."""
    n0, n1 = (1 << bs0) // 2, (1 << bs1) // 2
    lays = fc.layouts(n1, seed)
    if n0 != n1:
        lays += fc.long_x_list(np.random.default_rng(seed + n0), n0)
    return lays


def _setup_parts(lays, C_):
    floors = [(lay.mult, lay.xs) for lay in lays]
    mappings = [{"coupling": [], "floor_of_channel": [(i + c) % len(lays) for c in range(C_)]} for i in range(len(lays))]
    modes = [(bf, i) for i in range(len(lays)) for bf in (0, 1)]        # mode 2i short, 2i + 1 long, mapping i
    return floors, mappings, modes


def _make_setup(ctx, C_, bs0, bs1, floors, mappings, modes):
    lf = [L.FloorTypeOne(m, xs) for m, xs in floors]
    lm = []
    for mp in mappings:
        fo = mp["floor_of_channel"]
        uniq = sorted(set(fo))
        lm.append(L.Mapping(C_, [m for m, _ in mp["coupling"]], [a for _, a in mp["coupling"]], mux=[uniq.index(f) for f in fo],
                            submap_floors=uniq))
    return L.Setup(ctx, C_, bs0, bs1, lf, lm, [L.ModeInfo(bf, mi) for bf, mi in modes])


class Batch:
    """Chains of packets over one setup: per packet its mode, residue and floors (per channel y values, a dense curve or
    None), the oracle's PCM and end state of every chain."""

    def __init__(self, ctx, oracle, C_, bs0, bs1, floors, mappings, modes, su=None):
        self.C, self.bs0, self.bs1 = C_, bs0, bs1
        self.floors, self.mappings, self.modes = floors, mappings, modes
        self.su = su or _make_setup(ctx, C_, bs0, bs1, floors, mappings, modes)
        self.oracle = oracle
        self.refs, self.seqs, self.wants, self.sizes = [], [], [], []
        self.coeffs, self.dense, self.kinds, self.ys = [], [], [], []

    def add_chain(self, packets):
        """packets: [(mode, residue [C][n/2], floors [C])]."""
        mids = [m for m, _, _ in packets]
        bf = np.array([self.modes[m][0] for m in mids], np.uint8)
        prev, nxt = cc.window_flags(bf)
        ref = RefStream(self.oracle, self.C, self.bs0, self.bs1, self.modes, self.mappings, self.floors)
        parts, size = [], 0
        for i, (m, res, fl) in enumerate(packets):
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

    @property
    def n_pk(self):
        return sum(len(s[0]) for s in self.seqs)

    def run(self, ctx, fmt, ran, not_ran, env=None, misalign=False, entry=cabi.ENTRY_RESIDUE, vq=None):
        """Decodes every chain from empty streams in device memory and checks PCM and end states against the oracle's.
        Returns the PCM arena."""
        Cn = self.C
        planar = fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR)
        pwrs = [L.PreviousWindowRight(self.su) for _ in self.seqs]
        chains, coff, ooff, row = [], 1 if misalign else 0, 0, 0
        for s, (mids, prev, nxt) in enumerate(self.seqs):
            n = self.wants[s].shape[1]
            stride = (n + 3) & ~3
            chains.append(L.ChainSpec(pwrs[s], mids, prev, nxt, coeff_offset=coff, packet_index=row, out_offset=ooff,
                                      out_stride=stride if planar else 0))
            coff += self.sizes[s]
            ooff += Cn * (stride if planar else n)
            row += len(mids)
        pad = np.zeros(1 if misalign else 0, np.float32)
        coeffs, dense = np.concatenate([pad] + self.coeffs), np.concatenate([pad] + self.dense)
        dt = np.float32 if fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED) else np.int16
        pcm = np.zeros(max(ooff, 4), dt)
        bufs = [ctx.device_alloc(a.nbytes) for a in (coeffs, dense, pcm)]
        try:
            for p, a in zip(bufs, (coeffs, dense, pcm)):
                ctx.h2d(p, a)
            kw = dict(floor_kind=np.concatenate(self.kinds), floor1_y=np.concatenate(self.ys), dense_floor=bufs[1])
            if vq is not None:
                kw["vq"] = vq
            with environ(env), expect_kernels(ctx, ran=ran, not_ran=not_ran):
                L.decode_chains(ctx, chains, entry, cabi.MEM_DEVICE, None if entry == cabi.ENTRY_VQ else bufs[0], bufs[2], fmt, **kw)
            ctx.synchronize()
            ctx.d2h(pcm, bufs[2])
        finally:
            for p in bufs:
                ctx.device_free(p)
        for s, c in enumerate(chains):
            w = self.wants[s]
            n = w.shape[1]
            assert (c.status, c.n_samples) == (0, n), (s, c.status, c.n_samples, n)
            got = (np.stack([pcm[c.out_offset + k * c.out_stride:][:n] for k in range(Cn)]) if planar
                   else pcm[c.out_offset:c.out_offset + n * Cn].reshape(n, Cn).T)
            if dt == np.float32:
                assert bits_equal(got, w), (s, mismatch_report(got, w))
            else:
                assert np.array_equal(got, self.oracle.quantise_i16(w)), s
            a, b = pwrs[s].data(), self.refs[s].pwr.data()
            assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), (s, "state")
        for p in pwrs:
            p.close()
        return pcm


def _floors_of(lays, mapping, kinds):
    """Per channel: the coded y values of its layout (floor 1), a dense curve or None."""
    return [lays[mapping["floor_of_channel"][c]].y if k == FLOOR_ONE else None for c, k in enumerate(kinds)]


def layout_batch(ctx, oracle, C_, bs0, bs1, n_pk, chains, kinds_of=None, seed=0):
    """A Batch over the layouts of (bs0, bs1): n_pk packets in `chains` chains, packet j in mode j % (2 x layouts), so
    that every layout sits on every channel in short and long blocks.  kinds_of(c): the floor kind of channel c
    (default floor 1)."""
    lays = site_layouts(bs0, bs1, seed)
    floors, mappings, modes = _setup_parts(lays, C_)
    b = Batch(ctx, oracle, C_, bs0, bs1, floors, mappings, modes)
    rng = np.random.default_rng(seed + 17 * C_ + bs1)
    per = -(-n_pk // chains)
    for s in range(chains):
        packets = []
        for j in range(s * per, min(n_pk, (s + 1) * per)):
            m = j % len(modes)
            n2 = (1 << (bs1 if modes[m][0] else bs0)) // 2
            res = (rng.standard_normal((C_, n2)) * 0.5).astype(np.float32)
            kinds = [kinds_of(c) if kinds_of else FLOOR_ONE for c in range(C_)]
            fl = _floors_of(lays, mappings[modes[m][1]], kinds)
            fl = [(rng.random(n2) + 0.1).astype(np.float32) if k == FLOOR_DENSE else f for k, f in zip(kinds, fl)]
            packets.append((m, res, fl))
        b.add_chain(packets)
    return b, lays


def _formats(interleaved):
    return ((cabi.OUT_F32_INTERLEAVED, cabi.OUT_I16_INTERLEAVED) if interleaved else (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR))


def _shift_rows(b, lays):
    """(rows that need the post-shift, rows that do not) among the batch's floor-1 rows."""
    shift = sum(1 for lay in lays if any(x1 - x0 > 4096 for x0, _, x1, _ in lay.segments()))
    return shift, len(lays) - shift


# ---------------------------------------------------------------------------------------------------------------------
# F1: the residue entry's front stages
# ---------------------------------------------------------------------------------------------------------------------
def test_f1_front_stages_over_more_than_two_grids_of_packets(ctx, oracle):
    """Stereo 256/2048 on the four-kernel path: one k_floor1_segments + k_prologue_fused<false> launch over more than
    2 x grid packets (the pipelined loop), short and long rows, SHIFT and non-SHIFT rows in it."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_pk = 2 * cc.pf_grid(1 << 30, 2, sm) + 200
    assert n_pk > 2 * cc.pf_grid(n_pk, 2, sm)
    b, lays = layout_batch(ctx, oracle, 2, 8, 11, n_pk, 16)
    shift, plain = _shift_rows(b, lays)
    assert shift >= 2 and plain >= 2, (shift, plain)
    _, ran, not_ran = fc.SITES["F1"]
    for fmt in _formats(False):
        b.run(ctx, fmt, {"k_floor1_segments": 1, "k_prologue_fused": 1, "k_imdct": 1}, set(not_ran) | FUSED, cc.GENERIC_ENV)


@pytest.mark.parametrize("bs", [(6, 13), (8, 11)], ids=["64_8192", "256_2048_one_pass"])
def test_f1_front_stages_at_the_extremes_and_in_the_one_pass_schedule(ctx, oracle, bs):
    """64/8192 on the four-kernel path (rows of 32 and 4096 bins, 128 bitmap words), and 256/2048 on the default paths
    (the one-pass schedule: k_long_s and k_short_g behind the front stages)."""
    bs0, bs1 = bs
    b, lays = layout_batch(ctx, oracle, 2, bs0, bs1, 4 * len(site_layouts(bs0, bs1)), 6)
    _, ran, not_ran = fc.SITES["F1"]
    env = cc.GENERIC_ENV if bs == (6, 13) else None
    for fmt in _formats(False):
        b.run(ctx, fmt, set(ran) | ({"k_imdct"} if env else set()), set(not_ran) | (FUSED if env else set()), env)


# ---------------------------------------------------------------------------------------------------------------------
# F3, F5, F6: k_chain's front half and k_prologue
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C_, bs0, bs1", [(1, 6, 13), (8, 7, 12)], ids=["1ch_64_8192", "8ch_128_4096"])
def test_f3_chain_kernel(ctx, oracle, C_, bs0, bs1):
    b, _ = layout_batch(ctx, oracle, C_, bs0, bs1, 2 * len(site_layouts(bs0, bs1)), 4)
    _, ran, not_ran = fc.SITES["F3"]
    for fmt in _formats(True):
        b.run(ctx, fmt, set(ran), set(not_ran) | FUSED)


@pytest.mark.parametrize("C_", [2, 8])
def test_f5_prologue_dda(ctx, oracle, C_):
    """The four-kernel path on a residue arena one element off 16 bytes: k_prologue renders every curve with the DDA."""
    b, _ = layout_batch(ctx, oracle, C_, 6, 13, 2 * len(site_layouts(6, 13)), 4)
    _, ran, not_ran = fc.SITES["F5"]
    for fmt in _formats(False):
        b.run(ctx, fmt, set(ran) | {"k_imdct"}, set(not_ran) | FUSED, cc.GENERIC_ENV, misalign=True)


def _f6_kind(c):
    """Channels 0-7 floor 1, then at the group boundary an unused and a dense floor, then floor 1 again."""
    return FLOOR_ONE if c < 8 or c > 9 else FLOOR_UNUSED if c == 8 else FLOOR_DENSE


def test_f6_prologue_groups(ctx, oracle):
    b, _ = layout_batch(ctx, oracle, 11, 7, 10, 2 * len(site_layouts(7, 10)), 3, kinds_of=_f6_kind)
    _, ran, not_ran = fc.SITES["F6"]
    for fmt in _formats(False):
        b.run(ctx, fmt, set(ran), set(not_ran))


# ---------------------------------------------------------------------------------------------------------------------
# the curve itself, through the debug tap
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C_", list(range(1, 13)))
def test_debug_tap_pre_mdct_is_the_walked_curve(oracle, C_):
    """pre_mdct = floor x residue with a residue of 1.0 and no coupling: inverse_db[walk] exactly, every layout on
    every channel, short (n/2 = 32) and long (n/2 = 4096) blocks."""
    db = oracle.inverse_db_table()
    c = L.Context(0)
    try:
        lays = site_layouts(6, 13)
        floors, mappings, modes = _setup_parts(lays, C_)
        su = _make_setup(c, C_, 6, 13, floors, mappings, modes)
        pwr = L.PreviousWindowRight(su)
        ran = fc.SITES["F5" if C_ <= 8 else "F6"][1]
        for i in range(0, len(lays), C_ if C_ < len(lays) else 1):
            for bf in (0, 1):
                n2 = (1 << (13 if bf else 6)) // 2
                fl = [lays[mappings[i]["floor_of_channel"][k]].y for k in range(C_)]
                with expect_kernels(c, ran=ran):
                    _, pre, _ = L.debug_taps(su, L.DecodedPacket(2 * i + bf, np.ones((C_, n2), np.float32), fl), pwr)
                for k in range(C_):
                    lay = lays[mappings[i]["floor_of_channel"][k]]
                    want = db[np.array(lay.walk(n2))]
                    assert bits_equal(pre[k], want), (C_, lay, n2, k, mismatch_report(pre[k], want))
        assert pwr.is_empty()
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# F2, F4: the VQ entry
# ---------------------------------------------------------------------------------------------------------------------
def _header_layouts(bs0, bs1):
    """The layouts a header can carry (post 1 at a power of two, 3 or more posts: one partition at least)."""
    return [lay for lay in site_layouts(bs0, bs1) if len(lay.xs) > 2 and lay.xs[1] & (lay.xs[1] - 1) == 0]


def _packer_floor(rng, spec, lay):
    """A packer floor with lay's multiplier and x list: its classes cover len(xs) - 2 posts (8 per partition)."""
    rb = lay.xs[1].bit_length() - 1
    f = vp.Floor1(rng, spec.books, spec.n_scalar, rangebits=rb, multiplier=lay.mult)
    n = len(lay.xs) - 2
    f.class_dims = [8] * (n >= 8) + [n % 8] * (n % 8 != 0)
    f.partition_class = [0] * (n // 8) + [len(f.class_dims) - 1] * (n % 8 != 0)
    f.class_sub, f.master, f.sub_books = [0] * len(f.class_dims), [0] * len(f.class_dims), [[0] for _ in f.class_dims]
    f.x_list = list(lay.xs)
    return f


class VqLayouts:
    """Packer-made streams (tests/vorbis_packer.py) whose floors are `lays`, mapping i (one submap, no coupling) on floor
    i: per packet the frontend's VQ records and dense residue, the floor-1 rows given the layouts' y values."""

    def __init__(self, ctx, oracle, C_, bs0, bs1, lays, n_chains, per_chain, seed):
        for k in range(40):
            rng = np.random.default_rng(seed + 1000 * k)
            spec = vp.StreamSpec(rng, channels=C_, bs0=bs0, bs1=bs1, residue_types=[1 + k % 2], couplings=[[]] * len(lays))
            spec.floors = [_packer_floor(rng, spec, lay) for lay in lays]
            for i, m in enumerate(spec.mappings):
                m.update(submaps=1, mux=[0] * C_, floors=[i], residues=[0])
            hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
            if hdr.vq_capable():
                break
            hdr.close()
        else:
            raise AssertionError("no VQ-capable draw")
        self.hdr = hdr
        floors = [(lay.mult, lay.xs) for lay in lays]
        mappings = [{"coupling": [], "floor_of_channel": [i] * C_} for i in range(len(lays))]
        self.batch = Batch(ctx, oracle, C_, bs0, bs1, floors, mappings, spec.modes, su=hdr.make_setup(ctx))
        runs, ents, roffs, eoffs = [], [], [0], [0]
        j = 0
        for s in range(n_chains):
            packets = []
            for _ in range(per_chain):
                m = j % len(spec.modes)
                pk, _info = spec.audio_packet(m, 1, 1, p_unused=0.2)
                d = hdr.decode_packet(pk)
                rr, ee = hdr.decode_packet_vq(pk)[1:]
                kinds, _, dn = d.pack()
                assert dn is None
                lay = lays[spec.modes[m][1]]
                packets.append((m, d.residue, [lay.y if k == FLOOR_ONE else None for k in kinds]))
                runs.append(rr)
                ents.append(ee)
                roffs.append(roffs[-1] + len(rr))
                eoffs.append(eoffs[-1] + len(ee))
                j += 1
            self.batch.add_chain(packets)
        assert sum(int(k.sum()) for k in self.batch.kinds) > 0
        self.vq = (np.concatenate(runs) if roffs[-1] else np.zeros(1, fe.VQ_RUN_DTYPE), np.array(roffs, np.uint64),
                   np.concatenate(ents).astype(np.uint16) if eoffs[-1] else np.zeros(1, np.uint16), np.array(eoffs, np.uint64))

    def both_entries(self, ctx, fmts, ran, not_ran, env=None):
        """Each format: the VQ entry and the dense residue entry on the same packets, each equal to the oracle and to
        each other byte for byte."""
        for fmt in fmts:
            vq = self.batch.run(ctx, fmt, ran, not_ran, env, entry=cabi.ENTRY_VQ, vq=self.vq)
            dense = self.batch.run(ctx, fmt, ran, not_ran, env)
            assert vq.tobytes() == dense.tobytes(), fmt

    def close(self):
        self.hdr.close()


def test_f2_vq_front_stages_match_the_dense_entry(ctx, oracle):
    lays = _header_layouts(8, 11)
    assert {"full_table", "end_at_n2+0", "long_x_list"} <= {lay.name for lay in lays}
    st = VqLayouts(ctx, oracle, 2, 8, 11, lays, 4, 3 * len(lays), 21000)
    try:
        _, ran, not_ran = fc.SITES["F2"]
        st.both_entries(ctx, _formats(False), {"k_floor1_segments": 1, "k_prologue_fused": 1, "k_imdct": 1},
                        set(not_ran) | FUSED, cc.GENERIC_ENV)
    finally:
        st.close()


@pytest.mark.parametrize("C_, bs0, bs1", [(1, 6, 13), (8, 7, 11)], ids=["1ch_64_8192", "8ch_128_2048"])
def test_f4_vq_chain_kernel_matches_the_dense_entry(ctx, oracle, C_, bs0, bs1):
    """The chain kernel keeps the VQ accumulators in shared memory (C x n/2 <= 12288): 8 channels reach 2048."""
    lays = _header_layouts(bs0, bs1)
    st = VqLayouts(ctx, oracle, C_, bs0, bs1, lays, 3, 2 * len(lays), 22000 + C_)
    try:
        _, ran, not_ran = fc.SITES["F4"]
        st.both_entries(ctx, _formats(True), set(ran), set(not_ran) | FUSED)
    finally:
        st.close()


# ---------------------------------------------------------------------------------------------------------------------
# x lists lwb_setup_create refuses
# ---------------------------------------------------------------------------------------------------------------------
def _create(ctx, xs):
    d = cabi.SetupDesc()
    d.audio_channels, d.blocksize_0, d.blocksize_1 = 1, 8, 11
    fl = (cabi.FloorDesc * 1)()
    fl[0].floor_type, fl[0].floor1_multiplier, fl[0].floor1_values = cabi.FLOOR_TYPE_ONE, 1, len(xs)
    for k, x in enumerate(xs):
        fl[0].floor1_x_list[k] = x
    mp = (cabi.MappingDesc * 1)()
    mp[0].submaps = 1
    md = (cabi.ModeDesc * 1)()
    md[0].blockflag, md[0].mapping = 1, 0
    d.n_floors, d.floors, d.n_mappings, d.mappings, d.n_modes, d.modes = 1, fl, 1, mp, 1, md
    h = C.c_void_p()
    rc = cabi.lib().lwb_setup_create(ctx._h, C.byref(d), C.byref(h))
    return rc, h


def test_setup_create_refuses_x_lists_not_starting_at_zero(ctx):
    """Posts 0 and 1 bracket the others in every refused list: only post 0 away from x = 0 is wrong with them."""
    for xs in ([5, 100, 50], [1, 2], [1, 32768, 2, 16384], [32767, 32768]):
        rc, h = _create(ctx, xs)
        assert rc == cabi.ERR_BAD_FORMAT and not h.value, (xs, rc)
    rng = np.random.default_rng(5)
    for rb in range(16):                   # what the header parser makes: [0, 1 << rangebits, distinct x below]
        for n in sorted({2, min(65, (1 << rb) + 1), min(33, (1 << rb) + 1)}):
            xs = [0, 1 << rb] + [int(v) for v in rng.choice(np.arange(1, 1 << rb), n - 2, replace=False)] if n > 2 else [0, 1 << rb]
            rc, h = _create(ctx, xs)
            assert rc == cabi.OK and h.value, (rb, n, rc)
            cabi.lib().lwb_setup_destroy(h)

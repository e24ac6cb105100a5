"""Floor type 0 on the device: packets whose floor-0 channels arrive as LWB_FLOOR_ZERO records (amplitude + coefficient
cosines) decode to exactly the PCM the same packets give with host-computed dense curves (LWB_FLOOR_DENSE), and to the
oracle fed floor0_expected curves -- on every batch path, memory space, floor-array space and output format, through
plans, submit tickets, the single-packet call and the debug taps; k_floor0_curves provably runs, and only where a batch
can hold a record."""
import numpy as np
import pytest

import lewton_b200 as L
import vorbis_packer as vp
from helpers import bits_equal, expect_kernels, launches_are_attributed, mismatch_report
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from test_floor0_emu import coeff_cosines
from test_frontend_cpu import floor0_expected
from test_frontend_gpu import consistent_modes, oracle_pcm

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

FORMATS = [(cabi.OUT_F32_PLANAR, np.float32, True), (cabi.OUT_I16_PLANAR, np.int16, True),
           (cabi.OUT_F32_INTERLEAVED, np.float32, False), (cabi.OUT_I16_INTERLEAVED, np.int16, False)]


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def make_setup(ctx, spec, describe=True):
    floors = []
    for f in spec.floors:
        if isinstance(f, vp.Floor0):
            floors.append(L.FloorTypeZero(f.order, f.rate, f.bark_map_size, f.amplitude_bits, f.amplitude_offset) if describe
                          else L.FloorTypeZero())
        else:
            floors.append(L.FloorTypeOne(f.multiplier, f.x_list))
    maps = [L.Mapping(spec.channels, [a for a, _ in m["coupling"]], [b for _, b in m["coupling"]], m["mux"], m["floors"])
            for m in spec.mappings]
    modes = [L.ModeInfo(bf, mi) for bf, mi in spec.modes]
    return L.Setup(ctx, spec.channels, spec.bs0, spec.bs1, floors, maps, modes)


class Case:
    """n_streams chains of n_packets packer packets (one setup with a type-0 floor, alone or beside floor-1 floors in
    other submaps), as both a dense-curve batch and a record batch, and the oracle's PCM of every stream."""

    def __init__(self, oracle, seed, channels, bs0, bs1, n_streams=3, n_packets=5):
        rng = np.random.default_rng(seed)
        self.spec = spec = vp.StreamSpec(rng, channels=channels, bs0=bs0, bs1=bs1, floor0=True)
        self.C = C = channels
        self.streams = []                    # per stream: (modes, prevs, nexts)
        coeffs, kinds_d, kinds_r, ys_r, ys_d, dense = [], [], [], [], [], []
        self.want, self.n_rec, self.records = [], 0, {}
        for s in range(n_streams):
            seq = consistent_modes(spec, rng, n_packets)
            infos = []
            for mode, prev, nxt in seq:
                _, info = spec.audio_packet(mode, prev, nxt, p_unused=0.15)
                infos.append(info)
                fl_exp, res = spec.expected(info)
                n2 = info["n"] // 2
                coeffs.append(res.ravel())
                kd, kr = np.zeros(C, np.uint8), np.zeros(C, np.uint8)
                yd, yr = np.zeros((C, 65), np.uint32), np.zeros((C, 65), np.uint32)
                dn = np.zeros((C, n2), np.float32)
                for c, f in enumerate(fl_exp):
                    if f is None:
                        continue
                    if f[0] == "one":
                        kd[c] = kr[c] = cabi.FLOOR_ONE
                        yd[c, : len(f[1])] = yr[c, : len(f[1])] = f[1]
                    else:
                        kd[c], kr[c] = cabi.FLOOR_DENSE, cabi.FLOOR_ZERO
                        dn[c] = floor0_expected(f[3], f[1], f[2], info["blockflag"], n2, spec.bs0, spec.bs1)
                        rec = L.Floor0Record(f[1], coeff_cosines(f[3].order, f[2]))
                        self.records[(len(kinds_d), c)] = rec
                        yr[c] = rec.words()
                        self.n_rec += 1
                kinds_d.append(kd); kinds_r.append(kr); ys_d.append(yd); ys_r.append(yr); dense.append(dn.ravel())
            pcm, _ = oracle_pcm(oracle, spec, infos)
            self.want.append(np.concatenate(pcm, axis=1))
            self.streams.append(([m for m, _, _ in seq], [p for _, p, _ in seq], [x for _, _, x in seq]))
        self.coeffs = np.concatenate(coeffs)
        self.dense = np.concatenate(dense)
        self.kinds = {False: np.concatenate(kinds_d), True: np.concatenate(kinds_r)}
        self.ys = {False: np.concatenate(ys_d), True: np.concatenate(ys_r)}
        self.n_packets = n_packets
        self.stride = (max(w.shape[1] for w in self.want) + 11) // 4 * 4       # (multiples of 4: the fused paths take it)

    def chains(self, setup):
        out, coff = [], 0
        for s, (modes, prevs, nexts) in enumerate(self.streams):
            out.append(L.ChainSpec(L.PreviousWindowRight(setup), modes, prevs, nexts, coeff_offset=coff, packet_index=s * self.n_packets,
                                   out_offset=s * self.C * self.stride, out_stride=self.stride))
            coff += sum(self.C * (setup.blocksize(m) // 2) for m in modes)
        return out

    def decode(self, ctx, setup, records, fmt, memory=cabi.MEM_HOST, floor_memory=cabi.MEM_HOST, batch=None):
        """PCM of every stream, [stream][channel][samples] (interleaved formats transposed back)."""
        code, dt, planar = fmt
        chains = self.chains(setup)
        pcm = np.zeros(len(chains) * self.C * self.stride, dt)
        kinds, ys = self.kinds[records], self.ys[records]
        dense = None if records else self.dense
        bufs = []

        def dev(a):
            p = ctx.device_alloc(max(a.nbytes, 16))
            ctx.h2d(p, a)
            bufs.append(p)
            return p

        try:
            args = dict(coeffs=self.coeffs, pcm=pcm, dense_floor=dense)
            if memory == cabi.MEM_DEVICE:
                args = dict(coeffs=dev(self.coeffs), pcm=dev(pcm), dense_floor=None if dense is None else dev(dense))
            fk, fy = (dev(kinds), dev(ys)) if floor_memory == cabi.MEM_DEVICE else (kinds, ys)
            if batch == "plan":
                b = L.Batch(ctx, chains, cabi.ENTRY_RESIDUE, memory, args["coeffs"], args["pcm"], code, floor_kind=fk, floor1_y=fy,
                            dense_floor=args["dense_floor"], floor_memory=floor_memory)
                b.run()
                for c in chains:
                    c.pwr.reset()
                b.run()                                   # re-plans after the reset
                b.collect()
                b.close()
            elif batch == "ticket":
                t = ctx.submit_chains(chains, cabi.ENTRY_RESIDUE, memory, args["coeffs"], args["pcm"], code, floor_kind=fk, floor1_y=fy,
                                      dense_floor=args["dense_floor"], floor_memory=floor_memory)
                t.wait()
            else:
                L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, memory, args["coeffs"], args["pcm"], code, floor_kind=fk, floor1_y=fy,
                                dense_floor=args["dense_floor"], floor_memory=floor_memory)
            ctx.synchronize()
            if memory == cabi.MEM_DEVICE:
                ctx.d2h(pcm, args["pcm"])
        finally:
            for p in bufs:
                ctx.device_free(p)
        out = []
        for s, c in enumerate(chains):
            assert c.status == 0 and c.packets_done == len(self.streams[s][0])
            blk = pcm[s * self.C * self.stride:(s + 1) * self.C * self.stride]
            n = c.n_samples
            out.append(blk.reshape(self.C, self.stride)[:, :n] if planar else blk[: n * self.C].reshape(n, self.C).T)
        return out

    def check_oracle(self, oracle, got, fmt):
        for s, (g, w) in enumerate(zip(got, self.want)):
            assert g.shape == w.shape, (s, g.shape, w.shape)
            if fmt[1] == np.int16:
                assert np.array_equal(g, oracle.quantise_i16(w)), s
            else:
                assert bits_equal(g, w), (s, mismatch_report(g, w))


def floor0_case(oracle, seed, channels, bs0, bs1, **kw):
    """The first draw from seed, seed + 1000, ... whose packets have floor-0 rows (a setup's mappings may leave its
    type-0 floor unused)."""
    for k in range(20):
        case = Case(oracle, seed + 1000 * k, channels, bs0, bs1, **kw)
        if case.n_rec:
            return case
    raise AssertionError("no draw with floor-0 rows")


def forced_path_kernels(env, channels, bs1):
    """The kernels a forced path runs (LWB_FORCE_GENERIC=1: the four-kernel path; =2: the chain kernel where its shared
    memory holds the channels' blocks, else the four-kernel path)."""
    if env == "1" or channels > 8 or channels * (3 << bs1) * 2 > 200 * 1024:
        # (the four-kernel path's front stages are the two-kernel form up to 8 channels, k_prologue beyond)
        return {"k_imdct", "k_overlap", "k_save_state"} | ({"k_prologue"} if channels > 8 else {"k_prologue_fused", "k_floor1_segments"})
    return {"k_chain"}


SHAPES = [(8, 11), (10, 10), (6, 13)]


@pytest.mark.parametrize("bs0,bs1", SHAPES)
@pytest.mark.parametrize("channels", [1, 2, 6, 10])
def test_records_decode_like_dense_curves_on_every_path(ctx, oracle, monkeypatch, bs0, bs1, channels):
    case = floor0_case(oracle, 7000 + 10 * bs0 + bs1 + channels, channels, bs0, bs1)
    su = make_setup(ctx, case.spec)
    envs = [None, "2", "1"] if channels <= 8 else [None]
    for ei, env in enumerate(envs):
        if env is None:
            monkeypatch.delenv("LWB_FORCE_GENERIC", raising=False)
        else:
            monkeypatch.setenv("LWB_FORCE_GENERIC", env)
        for k, (memory, floor_memory) in enumerate([(cabi.MEM_HOST, cabi.MEM_HOST), (cabi.MEM_DEVICE, cabi.MEM_HOST),
                                                    (cabi.MEM_DEVICE, cabi.MEM_DEVICE), (cabi.MEM_HOST, cabi.MEM_DEVICE)]):
            fmt = FORMATS[(ei + k) % 4]
            with expect_kernels(ctx, not_ran=() if floor_memory == cabi.MEM_DEVICE else ("k_floor0_curves",)):
                dense = case.decode(ctx, su, False, fmt, memory, floor_memory)
            with expect_kernels(ctx, ran=("k_floor0_curves",)) as ran:
                rec = case.decode(ctx, su, True, fmt, memory, floor_memory)
            launched = {n for n, v in ran.items() if v}
            if env is None:
                assert launched & {"k_prologue_fused", "k_chain", "k_prologue"}, launched
            else:
                assert forced_path_kernels(env, channels, bs1) <= launched, (env, launched)
            for d, r in zip(dense, rec):
                assert d.tobytes() == r.tobytes(), (env, memory, floor_memory, fmt[0], mismatch_report(r, d))
            case.check_oracle(oracle, rec, fmt)


@pytest.mark.parametrize("batch", ["plan", "ticket"])
def test_records_through_plans_and_tickets(ctx, oracle, batch):
    case = floor0_case(oracle, 7100, 2, 8, 11, n_streams=4, n_packets=6)
    su = make_setup(ctx, case.spec)
    # (a host-memory submit takes page-locked arrays only: tickets run on device arenas)
    spaces = {"plan": [(cabi.MEM_HOST, cabi.MEM_HOST), (cabi.MEM_DEVICE, cabi.MEM_DEVICE)],
              "ticket": [(cabi.MEM_DEVICE, cabi.MEM_HOST), (cabi.MEM_DEVICE, cabi.MEM_DEVICE)]}[batch]
    for memory, floor_memory in spaces:
        fmt = FORMATS[0]
        with expect_kernels(ctx, ran=("k_floor0_curves", "k_prologue_fused")):
            rec = case.decode(ctx, su, True, fmt, memory, floor_memory, batch=batch)
        case.check_oracle(oracle, rec, fmt)


def test_single_packet_and_debug_taps(ctx, oracle):
    case = floor0_case(oracle, 7200, 2, 8, 11, n_streams=1, n_packets=4)
    su = make_setup(ctx, case.spec)
    modes, prevs, nexts = case.streams[0]
    pw_r, pw_d = L.PreviousWindowRight(su), L.PreviousWindowRight(su)
    coff = 0
    for k, mode in enumerate(modes):
        n2 = su.blocksize(mode) // 2
        res = case.coeffs[coff: coff + 2 * n2].reshape(2, n2)
        dn = case.dense[coff: coff + 2 * n2].reshape(2, n2)
        coff += 2 * n2
        fr, fd = [], []
        for c in range(2):
            kd, y = case.kinds[True][2 * k + c], case.ys[True][2 * k + c]
            if kd == cabi.FLOOR_ZERO:
                fr.append(case.records[(k, c)])
                fd.append(dn[c])
            elif kd == cabi.FLOOR_ONE:
                fr.append(list(y)); fd.append(list(y))
            else:
                fr.append(None); fd.append(None)
        pr = L.DecodedPacket(mode, res, fr, prevs[k], nexts[k])
        pd = L.DecodedPacket(mode, res, fd, prevs[k], nexts[k])
        with expect_kernels(ctx, ran=("k_floor0_curves",) if cabi.FLOOR_ZERO in case.kinds[True][2 * k: 2 * k + 2] else ()):
            _, pre_r, _ = L.debug_taps(su, pr, pw_r)
        _, pre_d, _ = L.debug_taps(su, pd, pw_d)
        assert bits_equal(pre_r, pre_d), k
        assert L.read_audio_packet_generic(su, pr, pw_r).tobytes() == L.read_audio_packet_generic(su, pd, pw_d).tobytes(), k


def test_refusals_and_setups_without_descriptions(ctx, oracle):
    case = floor0_case(oracle, 7300, 2, 8, 11)
    plain = make_setup(ctx, case.spec, describe=False)
    fmt = FORMATS[0]
    # kind 3 on a floor without a floor-0 description: refused, nothing decoded
    chains = case.chains(plain)
    pcm = np.full(len(chains) * 2 * case.stride, 7.0, np.float32)
    with pytest.raises(L.AudioReadError) as e:
        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_HOST, case.coeffs, pcm, fmt[0],
                        floor_kind=case.kinds[True], floor1_y=case.ys[True])
    assert e.value.code == cabi.ERR_INVALID and np.all(pcm == 7.0)
    assert all(c.pwr.is_empty() for c in chains)
    # a setup without descriptions launches what it launched before: no k_floor0_curves, device floor arrays included
    with expect_kernels(ctx, not_ran=("k_floor0_curves",)):
        case.decode(ctx, plain, False, fmt)
        case.decode(ctx, plain, False, fmt, cabi.MEM_DEVICE, cabi.MEM_DEVICE)
    # on the device a record the setup cannot serve acts as an unused floor
    got = case.decode(ctx, plain, True, fmt, cabi.MEM_DEVICE, cabi.MEM_DEVICE)
    assert all(np.isfinite(g).all() for g in got)
    # descriptions out of range, on a setup without streams
    fresh = make_setup(ctx, case.spec, describe=False)
    f0 = next(i for i, f in enumerate(case.spec.floors) if isinstance(f, vp.Floor0))
    for order, bits, rate, bms in ((64, 8, 44100, 64), (1, 8, 44100, 64), (8, 0, 44100, 64), (8, 65, 44100, 64), (8, 8, 0, 64),
                                   (8, 8, 44100, 0)):
        with pytest.raises(L.AudioReadError) as e:
            fresh.set_floor0(f0, order, rate, bms, bits, 10)
        assert e.value.code == cabi.ERR_INVALID
    fresh.set_floor0(f0, 8, 44100, 64, 8, 10)
    fresh.set_floor0(f0, 9, 22050, 32, 12, 3)             # described again before use: replaces the first description
    L.PreviousWindowRight(fresh)
    with pytest.raises(L.AudioReadError) as e:             # fixed once the setup has streams
        fresh.set_floor0(f0, 8, 44100, 64, 8, 10)
    assert e.value.code == cabi.ERR_INVALID
    f1 = [i for i, f in enumerate(case.spec.floors) if not isinstance(f, vp.Floor0)]
    other = make_setup(ctx, case.spec, describe=False)
    for idx in f1[:1] + [len(case.spec.floors)]:
        with pytest.raises(L.AudioReadError):
            other.set_floor0(idx, 8, 44100, 64, 8, 10)


def test_order_63_and_64_bit_amplitudes(ctx, monkeypatch):
    """The widest record: 63 coefficients (two lane passes of the coefficient load) and 64-bit amplitudes (the u64 ->
    f32 conversion, amplitude_bits == 64), decoded from records and from dense curves on every path."""
    from types import SimpleNamespace
    rng = np.random.default_rng(7400)
    fl = SimpleNamespace(order=63, rate=44100, bark_map_size=256, amplitude_bits=64, amplitude_offset=200)
    su = L.Setup(ctx, 2, 8, 11, [L.FloorTypeZero(fl.order, fl.rate, fl.bark_map_size, fl.amplitude_bits, fl.amplitude_offset)],
                 [L.Mapping(2, [0], [1])], [L.ModeInfo(False), L.ModeInfo(True)])
    modes = [1, 1, 0, 0, 1, 1]
    pk_rec, pk_dense = [], []
    for k, mode in enumerate(modes):
        n2 = 1024 if mode else 128
        res = (rng.standard_normal((2, n2)) * 0.3).astype(np.float32)
        fr, fd = [], []
        for c in range(2):
            amp = (1 << 64) - 1 if (k + c) % 2 else int(rng.integers(1, 1 << 53)) << 11
            rows = [list(rng.uniform(-0.5, 3.5, 7).astype(np.float32)) for _ in range(9)]
            fr.append(L.Floor0Record(amp, coeff_cosines(63, rows)))
            fd.append(floor0_expected(fl, amp, rows, mode, n2, 8, 11))
        prev = modes[k - 1] if k else 1
        nxt = modes[k + 1] if k + 1 < len(modes) else 1
        pk_rec.append(L.DecodedPacket(mode, res, fr, prev, nxt))
        pk_dense.append(L.DecodedPacket(mode, res, fd, prev, nxt))
    for env in (None, "2", "1"):
        if env is None:
            monkeypatch.delenv("LWB_FORCE_GENERIC", raising=False)
        else:
            monkeypatch.setenv("LWB_FORCE_GENERIC", env)
        pw_r, pw_d = L.PreviousWindowRight(su), L.PreviousWindowRight(su)
        for k in range(len(modes)):
            with expect_kernels(ctx, ran=("k_floor0_curves",)):
                got = L.read_audio_packet_generic(su, pk_rec[k], pw_r)
            want = L.read_audio_packet_generic(su, pk_dense[k], pw_d)
            assert got.tobytes() == want.tobytes(), (env, k, mismatch_report(got, want))


def vq_stream(seed):
    """A packer stream with a type-0 floor that qualifies for LWB_ENTRY_VQ, its headers and some audio packets."""
    for k in range(30):
        rng = np.random.default_rng(seed + 1000 * k)
        spec = vp.StreamSpec(rng, channels=2, floor0=True)
        hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        if not hdr.vq_capable():
            continue
        seqs = [consistent_modes(spec, rng, 6) for _ in range(4)]
        packets = [[spec.audio_packet(m, p, x, p_unused=0.1) for m, p, x in seq] for seq in seqs]
        if any(f is not None and f[0] == "zero" for st in packets for _, info in st for f in spec.expected(info)[0]):
            return spec, hdr, packets
    raise AssertionError("no VQ-capable floor-0 draw")


def test_vq_entry_records_through_the_batcher(ctx, oracle):
    """StreamBatcher(entry=VQ, floor0=True): the same PCM as the dense-curve batcher, equal to the oracle, and no dense
    floor arena crosses (the input shrinks by exactly the dense arena)."""
    spec, hdr, packets = vq_stream(7500)
    want = []
    for st in packets:
        pcm, _ = oracle_pcm(oracle, spec, [info for _, info in st])
        want.append(np.concatenate(pcm, axis=1))
    stride = (max(w.shape[1] for w in want) + 11) // 4 * 4
    out, nbytes = {}, {}
    for rec in (False, True):
        su = hdr.make_setup(ctx, floor0=rec)
        b = fe.StreamBatcher(ctx, hdr, threads=2, entry=cabi.ENTRY_VQ, floor0=rec)
        pcm = np.zeros(len(packets) * 2 * stride, np.float32)
        jobs = [(L.PreviousWindowRight(su), [p for p, _ in st]) for st in packets]
        with expect_kernels(ctx, ran=("k_floor0_curves", "k_prologue_fused") if rec else ("k_prologue_fused",),
                            not_ran=() if rec else ("k_floor0_curves",)):
            res = b.decode(jobs, pcm, stride)
        assert all(r[2] == 0 for r in res), res
        out[rec], nbytes[rec] = pcm, b.input_bytes
        for j, w in enumerate(want):
            got = pcm[j * 2 * stride:(j + 1) * 2 * stride].reshape(2, stride)[:, : w.shape[1]]
            assert bits_equal(got, w), (rec, j, mismatch_report(got, w))
        b.close()
    assert out[True].tobytes() == out[False].tobytes()
    coeff_elems = sum(2 * info["n"] // 2 for st in packets for _, info in st)
    assert nbytes[False] - nbytes[True] == coeff_elems * 4, (nbytes, coeff_elems)


@pytest.mark.parametrize("floor_memory", [cabi.MEM_HOST, cabi.MEM_DEVICE])
def test_vq_entry_records_through_decode_chains(ctx, oracle, floor_memory):
    """LWB_ENTRY_VQ batches built from lwf_packet_decode_vq_ex, records against dense curves, host and device floor / VQ
    arrays, against the oracle."""
    spec, hdr, packets = vq_stream(7600)
    want = []
    for st in packets:
        pcm, _ = oracle_pcm(oracle, spec, [info for _, info in st])
        want.append(np.concatenate(pcm, axis=1))
    stride = (max(w.shape[1] for w in want) + 11) // 4 * 4
    outs = {}
    for rec in (False, True):
        su = hdr.make_setup(ctx, floor0=rec)
        kinds, ys, dense, runs, ents, roff, eoff, chains = [], [], [], [], [], [0], [0], []
        coff, row = 0, 0
        for s, st in enumerate(packets):
            modes, prevs, nexts, step = [], [], [], 0
            for p, _ in st:
                d, r, e = hdr.decode_packet_vq(p, floor0_records=rec)
                n2 = d.n // 2
                k, y, dn = d.pack()
                kinds.append(k); ys.append(y)
                dense.append(dn.ravel() if dn is not None else np.zeros(2 * n2, np.float32))
                runs.append(r); ents.append(e)
                roff.append(roff[-1] + len(r)); eoff.append(eoff[-1] + len(e))
                modes.append(d.mode_number); prevs.append(d.prev_window_flag); nexts.append(d.next_window_flag)
                step += 2 * n2
            chains.append(L.ChainSpec(L.PreviousWindowRight(su), modes, prevs, nexts, coeff_offset=coff, packet_index=row,
                                      out_offset=s * 2 * stride, out_stride=stride))
            coff += step
            row += len(st)
        kinds, ys = np.concatenate(kinds), np.concatenate(ys)
        vq = [np.concatenate(runs), np.array(roff, np.uint64), np.concatenate(ents).astype(np.uint16), np.array(eoff, np.uint64)]
        dense = np.concatenate(dense)
        pcm = np.zeros(len(packets) * 2 * stride, np.float32)
        bufs = []

        def dev(a):
            p = ctx.device_alloc(max(a.nbytes, 16))
            ctx.h2d(p, a)
            bufs.append(p)
            return p

        try:
            if floor_memory == cabi.MEM_DEVICE:
                kinds, ys, vq = dev(kinds), dev(ys), [dev(np.ascontiguousarray(a)) for a in vq]
            with expect_kernels(ctx, ran=("k_floor0_curves", "k_prologue_fused") if rec else ("k_prologue_fused",)):
                L.decode_chains(ctx, chains, cabi.ENTRY_VQ, cabi.MEM_HOST, None, pcm, cabi.OUT_F32_PLANAR, floor_kind=kinds,
                                floor1_y=ys, dense_floor=None if rec else dense, floor_memory=floor_memory, vq=vq)
            ctx.synchronize()
        finally:
            for p in bufs:
                ctx.device_free(p)
        assert all(c.status == 0 for c in chains)
        for j, w in enumerate(want):
            got = pcm[j * 2 * stride:(j + 1) * 2 * stride].reshape(2, stride)[:, : w.shape[1]]
            assert bits_equal(got, w), (rec, j, mismatch_report(got, w))
        outs[rec] = pcm
    assert outs[True].tobytes() == outs[False].tobytes()


def test_plan_replay_renders_records_a_captured_step_did_not_have(ctx, oracle):
    """A prepared batch captured on steps without floor-0 rows replays later steps whose host floor arrays carry records:
    the floor-0 curves still run (compared with the same three steps through lwb_decode_chains, dense curves)."""
    case = floor0_case(oracle, 7700, 2, 8, 11)
    case.stride += 2048                                    # (steps after the first also emit their first packet's samples)
    su = make_setup(ctx, case.spec)
    fmt = FORMATS[0]
    quiet = case.kinds[True].copy()
    quiet[(quiet == cabi.FLOOR_ZERO)] = cabi.FLOOR_UNUSED
    # reference: three synchronous steps on fresh streams, the last one with dense curves
    chains = case.chains(su)
    want = np.zeros(len(chains) * 2 * case.stride, np.float32)
    for kinds, dense in ((quiet, None), (quiet, None), (case.kinds[False], case.dense)):
        want[:] = 0
        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_HOST, case.coeffs, want, fmt[0], floor_kind=kinds,
                        floor1_y=case.ys[True] if dense is None else case.ys[False], dense_floor=dense)
    # the plan: captured on the quiet steps (the second run leaves the stream states as the first did: the third replays)
    # (prepared batches are captured on device arenas; the floor arrays stay on the host and are uploaded each step)
    chains = case.chains(su)
    kinds = quiet.copy()
    pcm = np.zeros_like(want)
    d_coeffs, d_pcm = ctx.device_alloc(case.coeffs.nbytes), ctx.device_alloc(pcm.nbytes)
    try:
        ctx.h2d(d_coeffs, case.coeffs)
        ctx.h2d(d_pcm, pcm)
        b = L.Batch(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_DEVICE, d_coeffs, d_pcm, fmt[0], floor_kind=kinds, floor1_y=case.ys[True])
        b.run()
        b.run()
        ctx.synchronize()
        np.copyto(kinds, case.kinds[True])
        with expect_kernels(ctx, ran=("k_floor0_curves",)):
            b.run()
        ctx.synchronize()
        b.close()
        ctx.d2h(pcm, d_pcm)
    finally:
        ctx.device_free(d_coeffs)
        ctx.device_free(d_pcm)
    assert pcm.tobytes() == want.tobytes()

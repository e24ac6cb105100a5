"""Every kernel reads the blocksize tables the caller passed in lwb_setup_desc.tables[2] (caller_tables: f64, scrambled,
split) and the bark tables passed to lwb_setup_set_floor0, against the oracle fed the same tables: f32 PCM bit for bit
(up to +-0 and NaN), i16 exactly, end states bit for bit.  Each row names the kernels that must run, so a row cannot
pass on a path it was not written for."""
import numpy as np
import pytest
import torch

import boundary_cases as bc
import caller_tables as ct
import lewton_b200 as L
import test_batch_layouts as layouts
from helpers import (FUSED, GENERIC, RefStream, bits_equal, environ, expect_kernels, launches_are_attributed, make_setup,
                     mismatch_report)
from lewton_b200 import _cabi as cabi
from test_floor0_emu import _expected_from_table

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

MODES = [(0, 0), (1, 0)]             # mode 0 short, mode 1 long
FLOOR = layouts.FLOOR
FORMATS = {"f32": cabi.OUT_F32_PLANAR, "i16": cabi.OUT_I16_PLANAR, "f32i": cabi.OUT_F32_INTERLEAVED,
           "i16i": cabi.OUT_I16_INTERLEAVED}
DEV, HOST = cabi.MEM_DEVICE, cabi.MEM_HOST
CHAIN = {"LWB_FORCE_GENERIC": "2"}
FOUR = {"LWB_FORCE_GENERIC": "1"}
SETS = ("f64", "scrambled")
SPLITS = ("split_bs0", "split_bs1")


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Kind(layouts.Kind):
    """test_batch_layouts' setup (its floor, stereo coupling) created with table set `name` ("generated": none passed);
    otabs: the oracle's twin of its tables."""

    def __init__(self, ctx, oracle, C, bs0, bs1, name):
        super().__init__(ctx, C, bs0, bs1, tables=None if name == "generated" else ct.table_set(name, bs0, bs1))
        self.name = name
        self.otabs = None if self.tables is None else ct.oracle_pair(oracle, self.tables)


def streams_of(kind, texts):
    return [(kind, t) for t in texts]


def run(ctx, oracle, streams, fmt="f32", memory=DEV, env=None, residue=False, ran=(), not_ran=(), ran_any=(), seed=0):
    """Decodes the block sequences of `streams` ([(Kind, bc.stream text or its parse)]) from fresh streams, one
    test_batch_layouts.Batch (padded layout) per |-separated part, each held by Batch.check to the chains' oracle twins
    (fed the same tables), their end states and the write set.  The kernels launched over all batches must include `ran`
    (a dict: exact counts) and one of `ran_any`, and none of `not_ran`."""
    rng = np.random.default_rng(seed)
    sts, lens = [], []
    for k, seq in streams:
        batches = bc.stream(seq) if isinstance(seq, str) else seq
        st = layouts.Stream(oracle, k)
        st.bf, st.prev, st.nxt = (np.concatenate([bt[j] for bt in batches]) for j in range(3))
        sts.append(st)
        lens.append([len(bt[0]) for bt in batches])
    try:
        with expect_kernels(ctx, ran=ran, not_ran=not_ran) as launched:
            for b in range(len(lens[0])):
                items = [(st, layouts.Packets(rng, st, n[b], residue)) for st, n in zip(sts, lens)]
                batch = layouts.Batch(items, FORMATS[fmt], "padded", rng, residue)
                rc, pcm = batch.run(ctx, memory, env=env)
                assert rc == 0, (fmt, b, rc)
                batch.check(oracle, pcm, (fmt, memory, b, [st.kind.name for st in sts]))
    finally:
        for st in sts:
            st.pwr.close()
    if ran_any:
        assert any(launched[k] for k in ran_any), (sorted(ran_any), {k: v for k, v in launched.items() if v})
    return launched


# block sequences: S short, L long (flags from the neighbours), batches separated by |
LONG = ["L L L | L L L L | L L", "L L | L L L | L L L L", "L | L L L L L | L"]
MIXED = ["L S L L | S L L S | L L", "S L | L L S S L | S", "L L | S S | L S L", "S | L S L L L S | S L"]
MIXED_LONG = ["L L S L L L | L L S L L", "L L L S L | L L L L S L", "S L L L L | L S L L L"]     # long blocks in the majority


def both_formats(ctx, oracle, streams, **kw):
    """f32 from device memory and i16 from host memory, from fresh streams each."""
    run(ctx, oracle, streams, fmt="f32", memory=DEV, **kw)
    run(ctx, oracle, streams, fmt="i16", memory=HOST, seed=1, **kw)


def plan_launches(case, sm, env, memory):
    total = {}
    for p in bc.plans(case, sm, env, memory):
        for k, v in p.launches.items():
            total[k] = total.get(k, 0) + v
    return {k: v for k, v in total.items() if v}


# ---- the fused kernels ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tables", SETS)
def test_k_long(ctx, oracle, tables):
    k = Kind(ctx, oracle, 2, 8, 11, tables)
    both_formats(ctx, oracle, streams_of(k, LONG), ran={"k_long"}, not_ran={"k_chain"} | GENERIC)


@pytest.mark.parametrize("bs0", bc.RUNTIME_LS_BS0)
@pytest.mark.parametrize("tables", SETS)
def test_k_long_transitions(ctx, oracle, sm, tables, bs0):
    """k_long's runtime-ls transitions at every blocksize_0: the short slope is the caller's tab[0] window."""
    case = bc.CASES[f"runtime_ls_{bs0}"]
    env = bc.ROUNDS if bs0 == 8 else None
    k = Kind(ctx, oracle, case.C, bs0, 11, tables)
    for fmt, memory in (("f32", DEV), ("i16", HOST)):
        want = plan_launches(case, sm, env, "device" if memory == DEV else "host")
        assert want.get("k_long"), want
        run(ctx, oracle, [(k, s) for s in case.streams], fmt=fmt, memory=memory, env=env, ran=want, not_ran=GENERIC)


@pytest.mark.parametrize("case,env", [("precopy", None), ("cuts", None), ("precopy", bc.ROUNDS), ("cuts", bc.ROUNDS)])
@pytest.mark.parametrize("tables", SETS)
def test_one_pass_schedule(ctx, oracle, sm, tables, case, env):
    """k_long_s with k_short / k_short_g (and, with LWB_MIXED_ROUNDS=1, k_long and k_short in rounds)."""
    c = bc.CASES[case]
    k = Kind(ctx, oracle, c.C, c.bs0, 11, tables)
    want = plan_launches(c, sm, env, "device")
    assert want.get("k_long" if env else "k_long_s") and (want.get("k_short") or want.get("k_short_g")), want
    run(ctx, oracle, [(k, s) for s in c.streams], env=env, ran=want, not_ran=GENERIC)


@pytest.mark.parametrize("C,bs", [(2, 10), (1, 9)])
@pytest.mark.parametrize("tables", SETS + SPLITS)
def test_k_mid(ctx, oracle, tables, C, bs):
    """(10, 10) and (9, 9) with short packets and long blocks after short ones, which read tab[0]: k_mid takes equal
    tables; with two different ones (split) the batch goes to the chain kernel, which reads each packet's own."""
    k = Kind(ctx, oracle, C, bs, bs, tables)
    if tables in SPLITS:
        both_formats(ctx, oracle, streams_of(k, MIXED), ran={"k_chain"}, not_ran={"k_mid"} | GENERIC)
    else:
        both_formats(ctx, oracle, streams_of(k, MIXED), ran={"k_mid"}, not_ran={"k_chain"} | GENERIC)


@pytest.mark.parametrize("tables", SETS + SPLITS)
def test_k_short(ctx, oracle, tables):
    """Uniform (8, 8): k_short takes equal tables; split tables go to the chain kernel."""
    k = Kind(ctx, oracle, 2, 8, 8, tables)
    if tables in SPLITS:
        both_formats(ctx, oracle, streams_of(k, MIXED), ran={"k_chain"}, not_ran={"k_short", "k_short_g"} | GENERIC)
    else:
        both_formats(ctx, oracle, streams_of(k, MIXED), ran_any={"k_short", "k_short_g"}, not_ran={"k_chain"} | GENERIC)


@pytest.mark.parametrize("tables", SETS + SPLITS)
def test_k_long_equal_blocksizes(ctx, oracle, tables):
    """(11, 11) on the segmented path: a long block after a short one of the same size slopes its whole left half with
    tab[0]'s window.  Equal tables leave it on k_long / k_long_s; split ones send it to the chain kernel (which also
    takes the short blocks), while the long blocks between long ones stay on k_long."""
    k = Kind(ctx, oracle, 2, 11, 11, tables)
    both_formats(ctx, oracle, streams_of(k, MIXED_LONG), ran={"k_chain"}, ran_any={"k_long", "k_long_s"}, not_ran=GENERIC)


@pytest.mark.parametrize("bs1", range(6, 14))
@pytest.mark.parametrize("tables", SETS)
def test_k_chain(ctx, oracle, tables, bs1):
    """Every blocksize_1, planar and interleaved: one warp per chain up to n = 1024, several beyond."""
    bs0 = max(6, bs1 - 2)
    k = Kind(ctx, oracle, 2, bs0, bs1, tables)
    not_ran = FUSED | GENERIC
    run(ctx, oracle, streams_of(k, MIXED), fmt="f32", env=CHAIN, ran={"k_chain"}, not_ran=not_ran)
    run(ctx, oracle, streams_of(k, MIXED), fmt="f32i", memory=HOST, env=CHAIN, ran={"k_chain"}, not_ran=not_ran, seed=1)
    run(ctx, oracle, streams_of(k, MIXED[:2]), fmt="i16i", env=CHAIN, ran={"k_chain"}, not_ran=not_ran, seed=2)


@pytest.mark.parametrize("C,env", [(2, FOUR), (10, None)])
@pytest.mark.parametrize("tables", SETS + ("split_bs1",))
def test_four_kernel_path(ctx, oracle, tables, C, env):
    bs0 = 11 if tables == "split_bs1" else 8
    k = Kind(ctx, oracle, C, bs0, 11, tables)
    both_formats(ctx, oracle, streams_of(k, MIXED[:2]), env=env, ran={"k_imdct", "k_overlap"}, not_ran={"k_chain"} | FUSED)


@pytest.mark.parametrize("shape", ["k_long", "k_mid"])
@pytest.mark.parametrize("tables", SETS)
def test_residue_entry(ctx, oracle, tables, shape):
    """k_prologue_fused's spectrum into k_long / k_mid."""
    if shape == "k_long":
        k, texts = Kind(ctx, oracle, 2, 8, 11, tables), LONG
    else:
        k, texts = Kind(ctx, oracle, 2, 10, 10, tables), MIXED
    run(ctx, oracle, streams_of(k, texts), residue=True, ran={"k_prologue_fused", shape}, not_ran={"k_chain"} | GENERIC)
    run(ctx, oracle, streams_of(k, texts), fmt="i16", memory=HOST, residue=True, ran={"k_prologue_fused", shape},
        not_ran={"k_chain"} | GENERIC, seed=1)


# ---- batches of several setups, prepared batches -------------------------------------------------------------------
def test_batch_of_setups_with_different_tables(ctx, oracle):
    """Equal blocksizes, generated, f64 and scrambled tables: three twiddle packs, so no fused kernel takes the batch
    and every chain runs on the chain kernel with its own tables."""
    kinds = [Kind(ctx, oracle, 2, 8, 11, t) for t in ("generated", "f64", "scrambled")]
    streams = [(kinds[i % 3], t) for i, t in enumerate(MIXED + LONG)]
    run(ctx, oracle, streams, ran={"k_chain"}, not_ran=FUSED | GENERIC)
    run(ctx, oracle, streams, fmt="i16", memory=HOST, ran={"k_chain"}, not_ran=FUSED | GENERIC, seed=1)


def test_canonical_tables_passed_explicitly_share_the_generated_ones(ctx, oracle):
    """lwb_tables_generate's tables passed by the caller, bitrev included, are the context's cached ones: a batch of a
    setup with them and one without runs on k_long, which takes one twiddle pack per launch."""
    kinds = [Kind(ctx, oracle, 2, 8, 11, t) for t in ("generated", "canonical")]
    run(ctx, oracle, [(kinds[i % 2], t) for i, t in enumerate(LONG + LONG)], ran={"k_long"},
        not_ran={"k_chain"} | GENERIC)


def test_bitrev_other_than_compute_bitreverse_is_refused(ctx):
    for slot in (0, 1):
        for how in ("swap", "zero"):
            tabs = ct.table_set("f64", 8, 11)
            br = tabs[slot]["bitrev"]
            if how == "swap":
                br[[1, 2]] = br[[2, 1]]
            else:
                br[:] = 0
            with pytest.raises(L.AudioReadError) as e:
                make_setup(ctx, 2, 8, 11, modes=MODES, floors=[FLOOR], tables=tabs)
            assert e.value.code == cabi.ERR_INVALID, (slot, how)
            assert f"tables[{slot}].bitrev" in str(e.value), (slot, how, str(e.value))
    make_setup(ctx, 2, 8, 11, modes=MODES, floors=[FLOOR], tables=ct.table_set("f64", 8, 11)).close()     # still accepted


@pytest.mark.parametrize("tables", SETS)
def test_prepared_batch_replay(ctx, oracle, tables):
    """A prepared batch (lwb_plan_execute) executed four times on the same spectra: the plan, then replays of its steps."""
    k = Kind(ctx, oracle, 2, 8, 11, tables)
    rng = np.random.default_rng(5)
    S, P = 3, 4
    refs = [RefStream(oracle, 2, 8, 11, MODES, tables=k.otabs) for _ in range(S)]
    pwrs = [L.PreviousWindowRight(k.su) for _ in range(S)]
    spec = (rng.standard_normal((S, P, 2, 1024)) * 0.25).astype(np.float32)
    stride = P * 1024 + 4
    chains = [L.ChainSpec(pwrs[s], np.ones(P, np.uint8), coeff_offset=s * P * 2048, out_offset=s * 2 * stride, out_stride=stride)
              for s in range(S)]
    pcm = np.zeros(S * 2 * stride, np.float32)
    d_in, d_out = ctx.device_alloc(spec.nbytes), ctx.device_alloc(pcm.nbytes)
    try:
        ctx.h2d(d_in, spec.ravel())
        b = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, DEV, d_in, d_out, cabi.OUT_F32_PLANAR)
        with expect_kernels(ctx, ran={"k_long": 4}, not_ran={"k_chain"} | GENERIC):
            for r in range(4):
                b.run()
                ctx.synchronize()
                ctx.d2h(pcm, d_out)
                b.collect()
                for s in range(S):
                    w = np.concatenate([refs[s].spectrum(1, 1, 1, spec[s, p])[1] for p in range(P)], axis=1)
                    n = w.shape[1]
                    c = chains[s]
                    assert (c.status, c.n_samples) == (0, n), (r, s)
                    got = np.stack([pcm[c.out_offset + j * stride:][:n] for j in range(2)])
                    assert bits_equal(got, w), (r, s, mismatch_report(got, w))
                    assert bits_equal(pwrs[s].data(), refs[s].pwr.data()), (r, s, "end state")
        b.close()
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_out)
        for p in pwrs:
            p.close()


# ---- one packet at a time -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tables", SETS + ("split_bs1",))
def test_single_packet_calls(ctx, oracle, tables):
    """decode_spectrum and read_audio_packet_generic, packet by packet, on a (6, 13) setup (the chain kernel's)."""
    bs0 = 13 if tables == "split_bs1" else 6
    k = Kind(ctx, oracle, 2, bs0, 13, tables)
    rng = np.random.default_rng(9)
    seq = [(bf, pf, nf) for bf, pf, nf in zip(*bc.stream("L S L L S S L")[0])]
    for residue in (False, True):
        ref = RefStream(oracle, 2, bs0, 13, MODES, k.mappings, k.floors, tables=k.otabs)
        pwr = L.PreviousWindowRight(k.su)
        with expect_kernels(ctx, ran={"k_chain"}, not_ran=FUSED | GENERIC):
            for bf, pf, nf in seq:
                bf, pf, nf = int(bf), int(pf), int(nf)
                x = (rng.standard_normal((2, (1 << (13 if bf else bs0)) // 2)) * 0.25).astype(np.float32)
                if residue:
                    y = [[int(v) for v in rng.integers(0, 128, len(FLOOR[1]))] for _ in range(2)]
                    rc, w = ref.packet(bf, pf, nf, x, y)
                    got = L.read_audio_packet_generic(k.su, L.DecodedPacket(bf, x, y, pf, nf), pwr)
                else:
                    rc, w = ref.spectrum(bf, pf, nf, x)
                    got = L.decode_spectrum(k.su, bf, x, pwr, pf, nf)
                assert rc == 0 and bits_equal(got, w), (residue, bf, mismatch_report(got, w))
        e = pwr.data()
        assert bits_equal(e, ref.pwr.data()), (residue, "end state")
        pwr.close()


@pytest.mark.parametrize("bs0,bs1", [(8, 11), (6, 13)])
@pytest.mark.parametrize("tables", SETS + ("split_bs0",))
def test_post_imdct_tap(ctx, oracle, tables, bs0, bs1):
    """The debug taps' post-IMDCT samples against oracle.inverse_mdct of the pre-MDCT tap, with the same tables."""
    if tables == "split_bs0":
        bs0 = bs1
    k = Kind(ctx, oracle, 2, bs0, bs1, tables)
    rng = np.random.default_rng(3)
    pwr = L.PreviousWindowRight(k.su)
    for bf in (0, 1):
        n2 = (1 << (bs1 if bf else bs0)) // 2
        x = (rng.standard_normal((2, n2)) * 0.25).astype(np.float32)
        y = [[int(v) for v in rng.integers(0, 128, len(FLOOR[1]))] for _ in range(2)]
        with expect_kernels(ctx, ran={"k_imdct"}):
            _, pre, post = L.debug_taps(k.su, L.DecodedPacket(bf, x, y), pwr)
        t = None if k.otabs is None else k.otabs[bf]
        for c in range(2):
            w = oracle.inverse_mdct(pre[c], bs1 if bf else bs0, tables=t)
            assert bits_equal(post[c], w), (bf, c, mismatch_report(post[c], w))
    pwr.close()


# ---- floor 0 -------------------------------------------------------------------------------------------------------
def bark_table(rng, n2):
    """A caller's cached_bark_cos_omega: runs of equal values (1 to 12 bins), not monotone, some runs at +-1 and
    slightly beyond (what the generated table never holds)."""
    out = []
    while len(out) < n2:
        v = rng.uniform(-1, 1) if rng.random() < 0.8 else float(rng.choice([-1.05, -1.0, 1.0, 1.02]))
        out += [v] * int(rng.integers(1, 13))
    return np.array(out[:n2], np.float32)


@pytest.mark.parametrize("env", [None, CHAIN])
def test_floor0_bark_tables_of_the_caller(ctx, oracle, env):
    """Floor-0 records on a setup given one bark table per blockflag decode byte for byte like the dense curves
    _expected_from_table makes from the same tables, and like the oracle fed those curves; k_floor0_curves runs."""
    from types import SimpleNamespace
    rng = np.random.default_rng(21)
    C, bs0, bs1 = 2, 8, 11
    fl = SimpleNamespace(order=8, amplitude_bits=8, amplitude_offset=60, rate=44100, bark_map_size=256)
    su = L.Setup(ctx, C, bs0, bs1, [L.FloorTypeZero()], [L.Mapping(C)], [L.ModeInfo(0, 0), L.ModeInfo(1, 0)])
    bark = [bark_table(rng, 1 << (bs0 - 1)), bark_table(rng, 1 << (bs1 - 1))]
    su.set_floor0(0, fl.order, fl.rate, fl.bark_map_size, fl.amplitude_bits, fl.amplitude_offset, bark_cos_omega=bark)
    texts = ["L S L L | S S L", "S L L | L S L", "L L | S L S"]
    streams = [bc.stream(t) for t in texts]
    pwr_r = [L.PreviousWindowRight(su) for _ in texts]
    pwr_d = [L.PreviousWindowRight(su) for _ in texts]
    refs = [RefStream(oracle, C, bs0, bs1, MODES) for _ in texts]
    try:
        for b in range(2):
            coeffs, dense, ys, chains_r, chains_d, wants = [], [], [], [], [], []
            coff = ooff = pk = 0
            for s, batches in enumerate(streams):
                bf, pf, nf = batches[b]
                parts = []
                for i in range(len(bf)):
                    n2 = (1 << (bs1 if bf[i] else bs0)) // 2
                    res = (rng.standard_normal((C, n2)) * 0.5).astype(np.float32)
                    curves, words = [], []
                    for c in range(C):
                        while True:
                            amp = int(rng.integers(1, 256))
                            cosc = rng.uniform(-0.9, 0.9, fl.order).astype(np.float32)
                            curve = _expected_from_table(fl, amp, cosc, bark[int(bf[i])])
                            if np.all(np.isfinite(curve)):
                                break
                        curves.append(curve)
                        words.append(L.Floor0Record(amp, cosc).words())
                    rc, o = refs[s].packet(int(bf[i]), int(pf[i]), int(nf[i]), res, curves)
                    assert rc == 0
                    parts.append(o)
                    coeffs.append(res.ravel())
                    dense.append(np.stack(curves).ravel())
                    ys.append(np.stack(words))
                w = np.concatenate(parts, axis=1) if parts else np.zeros((C, 0), np.float32)
                stride = ((w.shape[1] + 3) & ~3) + 4
                for lst, pw in ((chains_r, pwr_r), (chains_d, pwr_d)):
                    lst.append(L.ChainSpec(pw[s], bf, pf, nf, coeff_offset=coff, packet_index=pk, out_offset=ooff, out_stride=stride))
                coff += sum(C * (1 << (bs1 if x else bs0)) // 2 for x in bf)
                ooff += C * stride
                pk += len(bf)
                wants.append(w)
            x = np.concatenate(coeffs)
            ys = np.stack(ys)
            out = {}
            for records, chains in ((True, chains_r), (False, chains_d)):
                pcm = np.zeros(ooff, np.float32)
                kinds = np.full((len(ys), C), cabi.FLOOR_ZERO if records else cabi.FLOOR_DENSE, np.uint8)
                with environ(env), expect_kernels(ctx, ran={"k_floor0_curves"} if records else (),
                                                  not_ran=() if records else {"k_floor0_curves"}) as launched:
                    L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, HOST, x, pcm, cabi.OUT_F32_PLANAR, floor_kind=kinds,
                                    floor1_y=ys, dense_floor=None if records else np.concatenate(dense))
                assert launched["k_chain" if env else "k_prologue_fused"], launched
                out[records] = pcm
                for s, c in enumerate(chains):
                    w = wants[s]
                    n = w.shape[1]
                    assert (c.status, c.n_samples) == (0, n), (records, b, s)
                    got = np.stack([pcm[c.out_offset + j * c.out_stride:][:n] for j in range(C)])
                    assert bits_equal(got, w), (records, b, s, mismatch_report(got, w))
            assert out[True].tobytes() == out[False].tobytes(), b
    finally:
        for p in pwr_r + pwr_d:
            p.close()

"""One stream batcher over several header sets (lwf_batcher_add_headers, StreamBatcher.add_headers) on the GPU: packets
from tests/vorbis_packer.py of streams with different channel counts, blocksizes and setups, in random order in one
call.  The batcher groups them by (channels, blocksize_0, blocksize_1) and synthesises one batch per group.

Every job is compared with the CPU oracle under the project's parity rule, and byte for byte (job results, PCM block,
end state) with the same jobs run through one single-header batcher per set on twin streams.  Arenas are sentinel-filled:
nothing outside a job's reported samples may change."""
import ctypes as C

import numpy as np
import pytest
import torch

import lewton_b200 as L
import vorbis_packer as vp
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from helpers import ALL_KERNELS, expect_kernels, launches_are_attributed
from test_batcher_submit_gpu import FORMATS, PLANAR, Arena, assert_contained, assert_oracle, assert_same_states, state
from test_f16_output_gpu import GUARDS, fill
from test_frontend_gpu import consistent_modes, oracle_pcm

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

HOST, DEVICE = cabi.MEM_HOST, cabi.MEM_DEVICE
RESIDUE, VQ = cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ
P, K = 3, 3                         # packets per stream and step, steps
STRIDE = P * 4096                   # room for P packets of the largest blocksize per channel plane
# name: (seed, channels, blocksize_0, blocksize_1 (log2), type-0 first floor, streams).  The first set's headers are the
# batcher's own (lwf_batcher_create), whose setup is never registered; the others are added.  Three modes each: two mode
# bits, so mode 3 does not exist.
SETS = {"mono": (901, 1, 8, 11, False, 2), "st_a": (902, 2, 8, 11, False, 3), "st_b": (903, 2, 8, 11, False, 2),
        "mid": (904, 2, 10, 10, False, 3), "six": (905, 6, 9, 12, False, 2), "floor0": (906, 2, 8, 11, True, 2),
        "ten": (907, 10, 8, 11, False, 1)}
LONG_SHORT = ("mono", "st_a", "st_b", "floor0")         # the 256/2048 sets


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


class Set:
    def __init__(self, oracle, name):
        seed, ch, bs0, bs1, floor0, n_streams = SETS[name]
        rng = np.random.default_rng(seed)
        self.name, self.channels = name, ch
        self.spec = spec = vp.StreamSpec(rng, channels=ch, bs0=bs0, bs1=bs1, floor0=floor0, n_modes=3)
        self.hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        assert ch > 8 or self.hdr.vq_capable()
        self.streams = []               # (packets, oracle PCM [C][n] of all of them)
        for _ in range(n_streams):
            pk, infos = [], []
            for mode, prev, nxt in consistent_modes(spec, rng, K * P):
                p, info = spec.audio_packet(mode, prev, nxt, p_unused=0.15)
                pk.append(p)
                infos.append(info)
            self.streams.append((pk, np.concatenate(oracle_pcm(oracle, spec, infos)[0], axis=1)))
        self.setups = {}

    def setup(self, ctx, records):
        if records not in self.setups:
            self.setups[records] = self.hdr.make_setup(ctx, floor0=records)
        return self.setups[records]


_sets = {}


def sets(oracle, entry):
    if not _sets:
        for name in SETS:
            _sets[name] = Set(oracle, name)
    return [s for s in _sets.values() if entry != VQ or s.channels <= 8]


def multi_batcher(ctx, sts, entry, records):
    bt = fe.StreamBatcher(ctx, sts[0].hdr, threads=3, entry=entry, floor0=records)
    for s in sts[1:]:
        bt.add_headers(s.hdr, s.setup(ctx, records))
    return bt


def block(buf, off, ch, n, fmt):
    """A job's n samples per channel as [ch][n], its PCM at element `off`."""
    blk = buf[off:off + ch * STRIDE]
    return blk.reshape(ch, STRIDE)[:, :n] if fmt in PLANAR else blk[:n * ch].reshape(n, ch).T


def spans(res, offs, chans, fmt):
    out = []
    for (n, _, _), off, ch in zip(res, offs, chans):
        out += [(off + c * STRIDE, n) for c in range(ch)] if fmt in PLANAR else [(off, n * ch)]
    return [s for s in out if s[1]]


def run_singles(ctx, sts, entry, records, twins, step_jobs, fmt):
    """Each set's jobs of one step (in the step's order) through a single-header batcher of that set: {(set, stream):
    (result, PCM block of C * STRIDE elements)}."""
    out = {}
    for s in sts:
        keys = [key for key in step_jobs if key[0] == s.name]
        if not keys:
            continue
        buf = fill(np.empty(sum(s.channels for _ in keys) * STRIDE, FORMATS[fmt]))
        res = s.single.decode([(twins[key], step_jobs[key]) for key in keys], buf, STRIDE, fmt)
        for j, key in enumerate(keys):
            out[key] = (res[j], buf[j * s.channels * STRIDE:(j + 1) * s.channels * STRIDE])
    return out


def run_steps(ctx, oracle, entry, records, fmt, how, packets_of=None, seed=0):
    """K steps of random jobs over every set (each stream once per step, in a random order per step) through one
    multi-header batcher: `how` "decode", or "host" / "device" two-deep submits.  Checks each job against the
    single-header batchers and (with the packer's packets) the oracle, the arenas' sentinels and the end states.
    packets_of(set, stream, step) -> packets replaces the packer's packets (no oracle check then)."""
    sts = sets(oracle, entry)
    by_name = {s.name: s for s in sts}
    rng = np.random.default_rng(seed)
    dt = FORMATS[fmt]
    bt = multi_batcher(ctx, sts, entry, records)
    for s in sts:
        s.single = fe.StreamBatcher(ctx, s.hdr, threads=3, entry=entry, floor0=records)
    keys = [(s.name, i) for s in sts for i in range(len(s.streams))]
    pwrs = {key: L.PreviousWindowRight(by_name[key[0]].setup(ctx, records)) for key in keys}
    twins = {key: L.PreviousWindowRight(by_name[key[0]].setup(ctx, records)) for key in keys}
    steps = []
    for k in range(K):
        order = [keys[i] for i in rng.permutation(len(keys))]
        step_jobs = {key: (packets_of(key[0], key[1], k) if packets_of else by_name[key[0]].streams[key[1]][0][k * P:(k + 1) * P])
                     for key in order}
        chans = [by_name[key[0]].channels for key in order]
        offs = list(np.cumsum([0] + [c * STRIDE for c in chans])[:-1])
        n_out = sum(chans) * STRIDE
        jobs = [(pwrs[key], step_jobs[key]) for key in order]
        if how == "decode":
            buf = fill(np.empty(n_out, dt))
            res = bt.decode(jobs, buf, STRIDE, fmt)
            steps.append((order, offs, chans, res, lambda buf=buf: buf))
        else:
            arena = Arena(ctx, HOST if how == "host" else DEVICE, n_out, dt)
            t = bt.submit(jobs, arena.pcm, STRIDE, fmt)
            steps.append((order, offs, chans, t, arena.read))
        assert bt.input_bytes > 0
        steps[-1] += (run_singles(ctx, sts, entry, records, twins, step_jobs, fmt),)
    pcm = {key: [] for key in keys}
    for k, (order, offs, chans, res, read, singles) in enumerate(steps):
        if how != "decode":
            res = res.wait()
        got = read()
        what = (entry, records, fmt, how, k)
        assert_contained(got, spans(res, offs, chans, fmt), what)
        for j, key in enumerate(order):
            want_res, want_blk = singles[key]
            assert res[j] == want_res, (what, key)
            blk = got[offs[j]:offs[j] + chans[j] * STRIDE]
            assert np.array_equal(blk.view(np.uint8), want_blk.view(np.uint8)), (what, key, "multi and single batchers differ")
            if packets_of is None:
                assert res[j][1:] == (P, 0), (what, key, res[j])
            pcm[key].append(block(got, offs[j], chans[j], res[j][0], fmt))
    if packets_of is None:
        for key in keys:
            got = np.concatenate(pcm[key], axis=1)
            want = by_name[key[0]].streams[key[1]][1]
            assert got.shape == want.shape, key
            assert_oracle(oracle, got, want, fmt, (entry, records, fmt, how, key))
    assert_same_states([pwrs[key] for key in keys], [twins[key] for key in keys], (entry, records, fmt, how))
    for p in list(pwrs.values()) + list(twins.values()):
        p.close()
    bt.close()
    for s in sts:
        s.single.close()


@pytest.mark.parametrize("how", ["decode", "host", "device"])
@pytest.mark.parametrize("records", [False, True], ids=["dense", "records"])
@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
def test_mixed_header_sets_match_single_batchers_and_oracle(ctx, oracle, entry, records, how):
    """Every format: three steps of random jobs over all header sets equal the single-header batchers byte for byte and
    the oracle under the parity rule, write nothing outside the jobs' samples and leave the twins' end states."""
    for i, fmt in enumerate(FORMATS):
        run_steps(ctx, oracle, entry, records, fmt, how, seed=100 * i + 10 * entry + records)


@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
def test_groups_run_on_their_fused_kernels(ctx, oracle, entry):
    """Planar output: the 1024/1024 group runs on k_mid and the 256/2048 groups on k_long or k_long_s (with k_short /
    k_short_g), none on k_chain, alone and in one call together."""
    sts = sets(oracle, entry)
    by_name = {s.name: s for s in sts}
    bt = multi_batcher(ctx, sts, entry, False)
    pwrs = {(s.name, i): L.PreviousWindowRight(s.setup(ctx, False)) for s in sts for i in range(len(s.streams))}
    longs = {"k_long", "k_long_s"}
    for k, names in enumerate([("mid",), LONG_SHORT, ("mid",) + LONG_SHORT]):
        keys = [key for key in pwrs if key[0] in names]
        buf = fill(np.empty(sum(by_name[n].channels for n, _ in keys) * STRIDE, np.float32))
        with expect_kernels(ctx, not_ran={"k_chain"}) as delta:
            res = bt.decode([(pwrs[key], by_name[key[0]].streams[key[1]][0][k * P:(k + 1) * P]) for key in keys], buf, STRIDE)
        ran = {name for name, v in delta.items() if v}
        assert all(r[1:] == (P, 0) for r in res), (names, res)
        assert ("k_mid" in ran) == ("mid" in names), (names, ran)
        assert bool(longs & ran) == (names != ("mid",)), (names, ran)
    for p in pwrs.values():
        p.close()
    bt.close()


@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
def test_bad_packets_report_single_batcher_status(ctx, oracle, entry):
    """Jobs with a truncated packet or a mode number the headers do not have, in every set, report the status the
    single-header batchers report for them (run_steps compares results, PCM and end states)."""
    def packets_of(name, i, k):
        pk = list(_sets[name].streams[i][0][k * P:(k + 1) * P])
        if k == 1 and i == 0:
            pk[1] = pk[1][:max(2, len(pk[1]) // 3)]
        if k == 1 and i == 1:
            pk[2] = bytes([(pk[2][0] & ~0x06) | 0x06]) + pk[2][1:]
        return pk

    for how in ("decode", "host"):
        run_steps(ctx, oracle, entry, False, cabi.OUT_F32_PLANAR, how, packets_of=packets_of, seed=7)
    # the statuses themselves: stream 1 of every set with two streams stopped at its mode-3 packet in step 1
    sts = sets(oracle, entry)
    bt = multi_batcher(ctx, sts, entry, False)
    keys = [(s.name, i) for s in sts for i in range(min(2, len(s.streams)))]
    pwrs = {key: L.PreviousWindowRight(_sets[key[0]].setup(ctx, False)) for key in keys}
    buf = fill(np.empty(sum(_sets[n].channels for n, _ in keys) * STRIDE, np.float32))
    res = bt.decode([(pwrs[key], packets_of(key[0], key[1], 1)) for key in keys], buf, STRIDE)
    for key, r in zip(keys, res):
        if key[1] == 1:
            assert r[1:] == (2, cabi.ERR_BAD_FORMAT), (key, r)
    for p in pwrs.values():
        p.close()
    bt.close()


@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
def test_refusals_change_nothing(ctx, oracle, entry):
    """A setup registered twice, a setup that does not match its headers, 10-channel headers on a VQ batcher, a submit
    whose only page-locked problem lies in a later group's PCM and one whose only repeated stream lies in a later group
    are refused; the refused submits issue no ticket, launch no kernel and change no job result, stream state or PCM
    element, and the next submit carries on as if they had not happened."""
    sts = sets(oracle, entry)
    by_name = {s.name: s for s in sts}
    lib = fe.lib()
    bt = multi_batcher(ctx, sts, entry, False)
    st_a, mid = by_name["st_a"], by_name["mid"]
    assert lib.lwf_batcher_add_headers(bt._h, st_a.hdr._h, st_a.setup(ctx, False)._h) == cabi.ERR_INVALID       # twice
    # setups no set has registered, so that only the comparison with the headers (or the context) can refuse them
    fresh_mid, fresh_six = mid.hdr.make_setup(ctx), by_name["six"].hdr.make_setup(ctx)
    assert lib.lwf_batcher_add_headers(bt._h, st_a.hdr._h, fresh_mid._h) == cabi.ERR_INVALID                  # blocksizes
    assert lib.lwf_batcher_add_headers(bt._h, mid.hdr._h, fresh_six._h) == cabi.ERR_INVALID                   # channels too
    assert lib.lwf_batcher_add_headers(bt._h, by_name["six"].hdr._h, fresh_mid._h) == cabi.ERR_INVALID
    other = L.Context(0)
    try:
        assert lib.lwf_batcher_add_headers(bt._h, st_a.hdr._h, st_a.hdr.make_setup(other)._h) == cabi.ERR_INVALID
    finally:
        other.close()
    # the same fresh setup with its own headers is taken (and its streams, of which this test has none, join mid's group)
    assert lib.lwf_batcher_add_headers(bt._h, mid.hdr._h, fresh_mid._h) == 0
    ten = _sets["ten"]
    if entry == VQ:
        assert lib.lwf_batcher_add_headers(bt._h, ten.hdr._h, ten.setup(ctx, False)._h) == cabi.ERR_INVALID
    # group 0 (mono, the batcher's own headers) first in the PCM, then a page boundary, then st_a's group
    mono = by_name["mono"]
    keys = [("mono", i) for i in range(len(mono.streams))] + [("st_a", i) for i in range(len(st_a.streams))]
    pwrs = {key: L.PreviousWindowRight(by_name[key[0]].setup(ctx, False)) for key in keys}
    page = 4096 // 4
    split = -(-len(mono.streams) * STRIDE // page) * page
    offs = [i * STRIDE for i in range(len(mono.streams))] + [split + i * 2 * STRIDE for i in range(len(st_a.streams))]
    n_out = split + len(st_a.streams) * 2 * STRIDE
    first = Arena(ctx, HOST, n_out, np.float32)
    step0 = [(pwrs[key], by_name[key[0]].streams[key[1]][0][:P]) for key in keys]

    def c_jobs(jobs):
        arr, keep, n = bt._jobs(jobs, STRIDE)
        for j in range(n):
            arr[j].out_offset = offs[j]
        return arr, keep, n

    arr0, keep0, n = c_jobs(step0)
    t0 = C.c_uint64()
    ctx.check(lib.lwf_batcher_submit(bt._h, arr0, n, cabi.OUT_F32_PLANAR, first.host.ctypes.data, HOST, C.byref(t0)))
    ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, t0.value))
    before = [state(pwrs[key]) for key in keys]
    nxt = [(pwrs[key], by_name[key[0]].streams[key[1]][0][P:2 * P]) for key in keys]
    raw = fill(np.empty(n_out + 2 * page, np.float32))
    lo = (-(raw.ctypes.data // 4)) % page
    pageable = raw[lo:lo + n_out]
    cudart = torch.cuda.cudart()
    torch.cuda.check_error(cudart.cudaHostRegister(pageable.ctypes.data, split * 4, 0))
    try:
        arena = Arena(ctx, HOST, n_out, np.float32)
        dup = nxt[:-1] + [(pwrs[("st_a", 0)], st_a.streams[0][0][P:2 * P])]
        for what, jobs, pcm in [("later group's pcm pageable", nxt, pageable), ("stream twice in a later group", dup, arena.host)]:
            arr, _, n = c_jobs(jobs)
            for j in range(n):
                arr[j].n_samples, arr[j].packets_done, arr[j].status = 1234, 56, -7
            t = C.c_uint64(999)
            with expect_kernels(ctx, not_ran=ALL_KERNELS):
                rc = lib.lwf_batcher_submit(bt._h, arr, n, cabi.OUT_F32_PLANAR, pcm.ctypes.data, HOST, C.byref(t))
            assert rc == cabi.ERR_INVALID, what
            assert t.value == 999, what
            assert all((arr[j].n_samples, arr[j].packets_done, arr[j].status) == (1234, 56, -7) for j in range(n)), what
            for key, b in zip(keys, before):
                a = state(pwrs[key])
                assert (a is None) == (b is None) and (a is None or np.array_equal(a.view(np.uint32), b.view(np.uint32))), what
            ctx.synchronize()
            for buf in (pageable, arena.read()):
                assert not np.any(buf.view(np.uint32) != GUARDS[np.dtype(np.float32)][1]), what
    finally:
        torch.cuda.check_error(cudart.cudaHostUnregister(pageable.ctypes.data))
    arr, keep1, n = c_jobs(nxt)
    t1 = C.c_uint64()
    ctx.check(lib.lwf_batcher_submit(bt._h, arr, n, cabi.OUT_F32_PLANAR, arena.host.ctypes.data, HOST, C.byref(t1)))
    assert t1.value == t0.value + 2, "a refused submit issued a ticket"         # two groups: two tickets
    ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, t1.value))
    got = arena.read()
    for j, key in enumerate(keys):
        s = by_name[key[0]]
        assert (arr[j].packets_done, arr[j].status) == (P, 0), key
        pcm = np.concatenate([block(first.host, offs[j], s.channels, arr0[j].n_samples, cabi.OUT_F32_PLANAR),
                              block(got, offs[j], s.channels, arr[j].n_samples, cabi.OUT_F32_PLANAR)], axis=1)
        want = s.streams[key[1]][1][:, :pcm.shape[1]]
        assert_oracle(oracle, pcm, want, cabi.OUT_F32_PLANAR, key)
    for p in pwrs.values():
        p.close()
    bt.close()

"""Refusals of a batch.  Every batch is walked once, before a batch path is chosen, and that walk makes every refusal a
batch can get from its arguments and arrays.  For a batch shaped for each of the five batch paths and each refusal,
called through lwb_decode_chains, lwb_submit_chains and lwb_plan_execute: the call returns the refusal's code and
message, launches no kernel, issues no ticket and changes no PCM element, chain result or stream state.  The same batch,
unbroken, then decodes on its path as the oracle does.  A stream-batcher submit of two groups whose later group has too
small an out_stride is refused before the first group is queued.  A chain whose PCM write set, coefficient range or
packet-row range would wrap past 2^64 is refused the same way, with the batch in host or in device memory: a wrapped sum
would otherwise give an extent that ends before it starts, and kernels queued against the wrapped address.

Do not run the wrap cases against a library without the wrap check: it queues kernels at the wrapped addresses."""
import ctypes as C

import numpy as np
import pytest

import lewton_b200 as L
import test_batcher_multi_gpu as multi
from helpers import ALL_KERNELS, FRONT, GENERIC, bits_equal, expect_kernels, launches_are_attributed
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from test_async_batches import AsyncCall, seq, setups, twins
from test_f16_output_gpu import GUARDS
from test_queued_batches import MIXED_EXTRA

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, RESIDUE, VQ, HOST, DEVICE = cabi.OUT_F32_PLANAR, cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ, cabi.MEM_HOST, cabi.MEM_DEVICE
MIXED = {"k_long_s", "k_short_g"}
# shape: (setup kind, sequence kind, packets per chain, kernels the unbroken residue batch runs, kernels it may add)
SHAPES = {
    "long": ("mixed", "long", 8, FRONT | {"k_long"}, set()),
    "mid": ("mid", "uniform", 8, FRONT | {"k_mid"}, set()),
    "mixed": ("mixed", "mixed", 16, FRONT | {"k_long_s"}, MIXED | MIXED_EXTRA),
    "chain": ("mixed", "mixed", 12, {"k_chain"}, set()),          # out_offset off the fused kernels' alignment
    "generic": ("wide", "mixed", 6, GENERIC, set()),
}
OUT_STRIDE = "chain: out_stride smaller than the samples produced"
WRAP = "chain: a PCM, coefficient or packet-row range does not fit in 64 bits"
U64 = 1 << 64
# case: (entry points, code, message).  lwb_decode_chains and lwb_plan_execute take pageable host memory.
CASES = {
    "out_stride": (("decode", "submit", "plan"), cabi.ERR_BUFFER, OUT_STRIDE),
    "stream_twice": (("decode", "submit", "plan"), cabi.ERR_INVALID, "a stream appears in two chains of one batch"),
    "dense_floor_missing": (("decode", "submit", "plan"), cabi.ERR_INVALID, "dense_floor missing"),
    "floor1_y_missing": (("decode", "submit", "plan"), cabi.ERR_INVALID, "floor1_y missing"),
    "floor_kind_range": (("decode", "submit", "plan"), cabi.ERR_INVALID, "floor_kind out of range"),
    "vq_offsets": (("decode", "submit", "plan"), cabi.ERR_INVALID, "vq offsets must be non-decreasing"),
    "wrap_out_offset": (("decode", "submit", "plan"), cabi.ERR_BUFFER, WRAP),
    "wrap_out_stride": (("decode", "submit", "plan"), cabi.ERR_BUFFER, WRAP),
    "wrap_coeff_offset": (("decode", "submit", "plan"), cabi.ERR_BUFFER, WRAP),
    "wrap_packet_index": (("decode", "submit", "plan"), cabi.ERR_BUFFER, WRAP),
    "wrap_out_bytes": (("decode", "submit", "plan"), cabi.ERR_BUFFER, WRAP),
    "wrap_coeff_bytes": (("decode", "submit", "plan"), cabi.ERR_BUFFER, WRAP),
    "wrap_packet_bytes": (("decode", "submit", "plan"), cabi.ERR_BUFFER, WRAP),
    "pageable": (("submit",), cabi.ERR_INVALID,
                 "host-memory submit: coeffs is not page-locked (lwb_host_alloc, cudaHostAlloc or cudaHostRegister)"),
}


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sus(ctx):
    return setups(ctx)


def break_batch(ctx, call, case, arr, io):
    """Breaks the marshalled batch (arr, io) of `call` as `case` says; returns the arrays io now points to."""
    kinds = call.kinds.copy()                     # [packet row][channel]
    last = arr[len(call.chains) - 1]
    if case == "out_stride":
        last.out_stride = 4
    elif case == "wrap_out_offset":               # out_offset + out_stride + n_samples passes 2^64
        last.out_offset = U64 - last.out_stride - 8
    elif case == "wrap_out_stride":               # (C - 1) * out_stride (+ n_samples) passes 2^64
        last.out_stride = U64 - 4
    elif case == "wrap_coeff_offset":             # the coefficient end passes 2^64
        last.coeff_offset = U64 - 16
    elif case == "wrap_packet_index":             # packet_index + packets passes 2^64
        last.packet_index = U64 - 2
    elif case == "wrap_out_bytes":                # the PCM end fits in elements, not in bytes (f32: * 4)
        last.out_offset = 1 << 62
    elif case == "wrap_coeff_bytes":              # the coefficient end fits in elements, not in bytes
        last.coeff_offset = 1 << 62
    elif case == "wrap_packet_bytes":             # the packet-row end fits, its floor1_y bytes (* C * LWB_MAX_POSTS * 4) do not
        last.packet_index = 1 << 60
    elif case == "stream_twice":
        arr[1].stream = arr[0].stream
    elif case == "dense_floor_missing":
        kinds[0] = cabi.FLOOR_DENSE
        io.floor_kind, io.dense_floor = kinds.ctypes.data, None
    elif case == "floor1_y_missing":
        kinds[0] = cabi.FLOOR_ONE
        io.floor_kind, io.floor1_y = kinds.ctypes.data, None
    elif case == "floor_kind_range":
        kinds[-1] = 7                             # the last channel of the last packet: the walk reads every row
        io.floor_kind = kinds.ctypes.data
    elif case == "vq_offsets":
        rows = sum(len(c.modes) for c in call.chains)
        offs = ctx.host_alloc(rows + 1, np.uint64)  # page-locked, so that only the order of the offsets is at fault
        offs[...] = 0
        offs[0] = 1
        runs, entries = ctx.host_alloc(4, np.uint64), ctx.host_alloc(4, np.uint16)
        io.entry = VQ
        io.vq_runs, io.vq_run_offsets, io.vq_entries, io.vq_entry_offsets = (runs.ctypes.data, offs.ctypes.data,
                                                                             entries.ctypes.data, offs.ctypes.data)
        return kinds, offs, runs, entries
    elif case == "pageable":
        plain = call.coeffs.copy()                # ordinary, pageable numpy memory
        io.coeffs = plain.ctypes.data
        return kinds, plain
    return (kinds,)


def sequence(rng, seq_kind, P):
    """seq's packets; a 'mixed' chain holds a short block, without which the batch is one k_long would take."""
    while True:
        s = seq(rng, seq_kind, P)
        if seq_kind != "mixed" or not s[0].all():
            return s


def empty_submit(ctx, io):
    """The ticket of a submit of no chains: the newest ticket issued."""
    t = C.c_uint64()
    ctx.check(cabi.lib().lwb_submit_chains(ctx._h, None, 0, C.byref(io), C.byref(t)))
    return t.value


@pytest.mark.parametrize("case,way", [(case, way) for case, (ways, _, _) in CASES.items() for way in ways])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_refused_batch_changes_nothing(ctx, oracle, sus, shape, case, way):
    refused_batch_changes_nothing(ctx, oracle, sus, shape, case, way, HOST)


@pytest.mark.parametrize("way", ["decode", "submit", "plan"])
@pytest.mark.parametrize("case", [case for case in CASES if case.startswith("wrap_")])
@pytest.mark.parametrize("shape", ["long", "chain", "generic"])
def test_wrapping_range_refused_in_device_memory(ctx, oracle, sus, shape, case, way):
    """The wrap refusals with coefficients, dense floors and PCM in device memory, where a wrapped address would be
    written in place."""
    refused_batch_changes_nothing(ctx, oracle, sus, shape, case, way, DEVICE)


def refused_batch_changes_nothing(ctx, oracle, sus, shape, case, way, memory):
    _, code, message = CASES[case]
    kind, seq_kind, P, ran, extra = SHAPES[shape]
    rng = np.random.default_rng([list(SHAPES).index(shape), list(CASES).index(case), ["decode", "submit", "plan"].index(way), memory])
    tws = twins(oracle, sus, kind, 2)
    call = AsyncCall(ctx, rng, [(tw, sequence(rng, seq_kind, P)) for tw in tws], RESIDUE, F32P, memory,
                     (ran, ALL_KERNELS - ran - extra))
    if shape == "chain":
        for c in call.chains:
            c.out_offset += 1
    coeffs, pcm = call.arenas()
    dense = call.kw["dense_floor"] if memory == DEVICE else call.dense
    arr, io = L.api._marshal(call.chains, RESIDUE, memory, coeffs, pcm, F32P, call.kinds, call.ys, dense, HOST, None)
    t0 = empty_submit(ctx, io)
    keep = break_batch(ctx, call, case, arr, io)
    n = len(call.chains)
    for i in range(n):
        arr[i].n_samples, arr[i].packets_done, arr[i].status = 7, 7, 7
    states = [tw.pwr.data() for tw in tws]
    t = C.c_uint64(999)
    with expect_kernels(ctx, not_ran=ALL_KERNELS):
        if way == "decode":
            rc = cabi.lib().lwb_decode_chains(ctx._h, arr, n, C.byref(io))
        elif way == "submit":
            rc = cabi.lib().lwb_submit_chains(ctx._h, arr, n, C.byref(io), C.byref(t))
        else:
            plan = C.c_void_p()
            ctx.check(cabi.lib().lwb_plan_create(ctx._h, arr, n, C.byref(io), C.byref(plan)))
            rc = cabi.lib().lwb_plan_execute(plan)
            cabi.lib().lwb_plan_destroy(plan)
    assert rc == code, (rc, cabi.lib().lwb_last_error(ctx._h).decode())
    assert cabi.lib().lwb_last_error(ctx._h).decode() == message
    assert t.value == 999
    assert all((arr[i].n_samples, arr[i].packets_done, arr[i].status) == (7, 7, 7) for i in range(n))
    ctx.synchronize()
    assert call.untouched()
    for tw, s in zip(tws, states):
        a = tw.pwr.data()
        assert (a is None) == (s is None) and (a is None or bits_equal(a, s))
    del keep                                      # (the arrays the broken io pointed to)
    call.submit(ctx)
    assert call.ticket.id == t0 + 1, "the refused call issued a ticket"
    call.ticket.wait()
    call.check(oracle, (shape, case, way))
    for tw in tws:
        tw.check_state((shape, case, way))


def test_batcher_refuses_a_later_group_before_queuing_the_first(ctx, oracle):
    """Two groups (mono and stereo 256/2048 headers): a job of the later group with too small an out_stride refuses the
    whole submit before the first group is queued -- no kernel, no ticket, no job result, stream state or PCM element
    changes -- and the unbroken submit then decodes as the oracle does."""
    sts = [multi.Set(oracle, name) for name in ("mono", "st_a")]       # (not the shared sets: their setups live on ctx)
    by_name = {s.name: s for s in sts}
    lib = fe.lib()
    bt = multi.multi_batcher(ctx, sts, RESIDUE, False)
    keys = [("mono", i) for i in range(len(by_name["mono"].streams))] + [("st_a", i) for i in range(len(by_name["st_a"].streams))]
    pwrs = {key: L.PreviousWindowRight(by_name[key[0]].setup(ctx, False)) for key in keys}
    jobs = [(pwrs[key], by_name[key[0]].streams[key[1]][0][:multi.P]) for key in keys]
    n_out = sum(by_name[key[0]].channels for key in keys) * multi.STRIDE
    arena = multi.Arena(ctx, HOST, n_out, np.float32)
    arr, keep, n = bt._jobs(jobs, multi.STRIDE)
    assert keys[-1][0] == "st_a"
    arr[n - 1].out_stride = 4
    for j in range(n):
        arr[j].n_samples, arr[j].packets_done, arr[j].status = 1234, 56, -7
    t = C.c_uint64(999)
    with expect_kernels(ctx, not_ran=ALL_KERNELS):
        rc = lib.lwf_batcher_submit(bt._h, arr, n, F32P, arena.host.ctypes.data, HOST, C.byref(t))
    assert rc == cabi.ERR_BUFFER
    assert cabi.lib().lwb_last_error(ctx._h).decode() == OUT_STRIDE
    assert t.value == 999
    assert all((arr[j].n_samples, arr[j].packets_done, arr[j].status) == (1234, 56, -7) for j in range(n))
    assert all(multi.state(p) is None for p in pwrs.values())
    ctx.synchronize()
    assert not np.any(arena.read().view(np.uint32) != GUARDS[np.dtype(np.float32)][1])
    arr[n - 1].out_stride = multi.STRIDE
    ctx.check(lib.lwf_batcher_submit(bt._h, arr, n, F32P, arena.host.ctypes.data, HOST, C.byref(t)))
    ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, t.value))
    got = arena.read()
    off = 0
    for j, key in enumerate(keys):
        s = by_name[key[0]]
        assert (arr[j].packets_done, arr[j].status) == (multi.P, 0), key
        pcm = multi.block(got, off, s.channels, arr[j].n_samples, F32P)
        multi.assert_oracle(oracle, pcm, s.streams[key[1]][1][:, :pcm.shape[1]], F32P, key)
        off += s.channels * multi.STRIDE
    for p in pwrs.values():
        p.close()
    bt.close()

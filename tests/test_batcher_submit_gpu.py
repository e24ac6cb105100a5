"""lwf_batcher_submit (StreamBatcher.submit) on the GPU: packets from tests/vorbis_packer.py, entropy-decoded by the
batcher's host threads, synthesised by asynchronous batches whose PCM lands in page-locked host memory or in device
memory.

Every submit is compared with lwf_batcher_decode on twin streams fed the same packets (PCM arenas byte for byte, job
results, end states) and with the CPU oracle under the project's parity rule (f32 bit for bit, i16 exactly, f16 as the
round-to-nearest-even binary16 of the oracle's f32).  Arenas are sentinel-filled: nothing outside a job's reported
samples may change."""
import ctypes as C

import numpy as np
import pytest
import torch

import lewton_b200 as L
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from helpers import ALL_KERNELS, bits_equal, expect_kernels, launches_are_attributed, mismatch_report
from test_f16_output_cpu import to_f16
from test_f16_output_gpu import GUARDS, fill, same_f16
from test_frontend_gpu import build_stream, oracle_pcm
from test_queued_batches import Gate

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

HOST, DEVICE = cabi.MEM_HOST, cabi.MEM_DEVICE
RESIDUE, VQ = cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ
FORMATS = {cabi.OUT_F32_PLANAR: np.float32, cabi.OUT_I16_PLANAR: np.int16, cabi.OUT_F16_PLANAR: np.float16,
           cabi.OUT_F32_INTERLEAVED: np.float32, cabi.OUT_I16_INTERLEAVED: np.int16, cabi.OUT_F16_INTERLEAVED: np.float16}
PLANAR = (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR, cabi.OUT_F16_PLANAR)
CH, S, P, K = 2, 6, 4, 3           # channels, streams, packets per stream and submit, submits


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


_streams = {}


def streams(oracle, floor0):
    """(spec, headers, [(packets, oracle PCM [C][n] of those packets)] per stream): stream s takes K * P consecutive
    packets of one packer sequence (seed 811; floor0: its first floor is of type 0)."""
    if floor0 not in _streams:
        spec, packets, infos = build_stream(811, CH, floor0, S * K * P)
        out = []
        for s in range(S):
            sl = slice(s * K * P, (s + 1) * K * P)
            out.append((packets[sl], np.concatenate(oracle_pcm(oracle, spec, infos[sl])[0], axis=1)))
        hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        _streams[floor0] = (spec, hdr, out)
    return _streams[floor0]


def make_batcher(ctx, hdr, entry, records):
    """A batcher, and the setup its streams need (records: type-0 floors travel as floor-0 records)."""
    su = hdr.make_setup(ctx, floor0=records)
    return su, fe.StreamBatcher(ctx, hdr, threads=3, entry=entry, floor0=records)


def stride_of(spec, packets):
    """Room for `packets` packets per channel plane: a long packet between a long and a short one yields 3/4 of its
    blocksize, less a quarter of the short one, so a blocksize each is enough."""
    return packets * (1 << spec.bs1)


class Arena:
    """A sentinel-filled PCM arena of n elements: page-locked host memory, or a torch CUDA tensor (passed to submit as the
    tensor, or as its integer address when as_int)."""

    def __init__(self, ctx, memory, n, dtype, as_int=False):
        self.host = fill(ctx.host_alloc(n, dtype))
        self.memory = memory
        if memory == DEVICE:
            self.dev = torch.from_numpy(self.host.copy()).cuda()
            torch.cuda.synchronize()
        self.pcm = self.host if memory == HOST else (self.dev.data_ptr() if as_int else self.dev)

    def read(self):
        return self.host.copy() if self.memory == HOST else self.dev.cpu().numpy()


def spans(res, stride, fmt):
    """Element intervals job j wrote (out_offset = j * CH * stride): [(start, length)]."""
    out = []
    for j, (n, _, _) in enumerate(res):
        off = j * CH * stride
        out += [(off + c * stride, n) for c in range(CH)] if fmt in PLANAR else [(off, n * CH)]
    return [s for s in out if s[1]]


def assert_contained(buf, sp, what):
    u, g = GUARDS[buf.dtype]
    outside = np.ones(buf.size, bool)
    for s, n in sp:
        outside[s:s + n] = False
    bad = np.nonzero(outside & (buf.view(u) != g))[0]
    assert not bad.size, f"{what}: {bad.size} elements outside the jobs' samples were written, first at {bad[:4]}"


def job_pcm(buf, j, n, stride, fmt):
    """Job j's n samples per channel as [CH][n]."""
    blk = buf[j * CH * stride:(j + 1) * CH * stride]
    return blk.reshape(CH, stride)[:, :n] if fmt in PLANAR else blk[:n * CH].reshape(n, CH).T


def assert_oracle(oracle, got, want, fmt, what):
    if FORMATS[fmt] == np.float32:
        assert bits_equal(got, want), (what, mismatch_report(got, want))
    elif FORMATS[fmt] == np.int16:
        assert np.array_equal(got, oracle.quantise_i16(want)), what
    else:
        assert same_f16(got, to_f16(want)), what


def state(pwr):
    d = pwr.data()
    return None if d is None else np.array(d, np.float32)


def assert_same_states(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        x, y = state(x), state(y)
        assert (x is None) == (y is None) and (x is None or bits_equal(x, y)), (what, i)


@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("floor0", ["none", "dense", "records"])
@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
def test_queued_submits_match_decode_and_oracle(ctx, oracle, entry, floor0, memory):
    """Three submits queued back to back over the same streams, no wait between them, every format.  After the waits:
    each arena equals lwf_batcher_decode's on twin streams byte for byte, and holds nothing outside the jobs' reported
    samples; the job results and end states are the twins'; every stream is the oracle's decode of its packets."""
    spec, hdr, sts = streams(oracle, floor0 != "none")
    if entry == VQ:
        assert hdr.vq_capable()
    records = floor0 == "records"
    stride = stride_of(spec, P)
    n_out = S * CH * stride
    for fmt, dt in FORMATS.items():
        what = (entry, floor0, memory, fmt)
        su, bt = make_batcher(ctx, hdr, entry, records)
        su2, twin = make_batcher(ctx, hdr, entry, records)
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        twins = [L.PreviousWindowRight(su2) for _ in range(S)]
        arenas, tickets = [], []
        for k in range(K):
            jobs = [(pwrs[s], sts[s][0][k * P:(k + 1) * P]) for s in range(S)]
            arenas.append(Arena(ctx, memory, n_out, dt, as_int=k == 1))
            tickets.append(bt.submit(jobs, arenas[-1].pcm, stride, fmt))
            assert bt.input_bytes > 0
        results = [t.wait() for t in tickets]
        assert all(t.done() for t in tickets)
        got = [a.read() for a in arenas]
        for k in range(K):
            want = fill(np.empty(n_out, dt))
            res = twin.decode([(twins[s], sts[s][0][k * P:(k + 1) * P]) for s in range(S)], want, stride, fmt)
            assert results[k] == res, (what, k)
            assert all(r[1:] == (P, 0) for r in res), (what, k, res)
            assert np.array_equal(got[k].view(np.uint8), want.view(np.uint8)), (what, k, "submit and decode differ")
            assert_contained(got[k], spans(results[k], stride, fmt), (what, k))
        for s in range(S):
            pcm = np.concatenate([job_pcm(got[k], s, results[k][s][0], stride, fmt) for k in range(K)], axis=1)
            assert pcm.shape == sts[s][1].shape, (what, s)
            assert_oracle(oracle, pcm, sts[s][1], fmt, (what, s))
        assert_same_states(pwrs, twins, what)
        for p in pwrs + twins:
            p.close()
        bt.close()
        twin.close()


def c_jobs(pwrs, bufs, stride):
    """An lwf_stream_job array over packets held in numpy buffers (which the caller may overwrite)."""
    arr = (fe._StreamJob * len(pwrs))()
    keep = []
    for j, (pwr, pk) in enumerate(zip(pwrs, bufs)):
        ptrs = (C.c_char_p * len(pk))(*[b.ctypes.data for b in pk])
        lens = (C.c_size_t * len(pk))(*[b.size for b in pk])
        keep.append((ptrs, lens))
        arr[j].stream, arr[j].n_packets, arr[j].packets, arr[j].lengths = pwr._h, len(pk), ptrs, lens
        arr[j].out_offset, arr[j].out_stride = j * CH * stride, stride
    return arr, keep


def c_submit(ctx, bt, arr, pcm, memory, fmt=cabi.OUT_F32_PLANAR):
    t = C.c_uint64()
    ctx.check(fe.lib().lwf_batcher_submit(bt._h, arr, len(arr), fmt, pcm, memory, C.byref(t)))
    return t.value


@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
def test_submits_overlap_the_gpu_and_reuse_arena_sets(ctx, oracle, memory):
    """Behind a closed gate on the context's stream, the second submit returns while the gate is still closed; four more
    reuse the two arena sets (each waits for the submit two back).  Every packet buffer is overwritten as soon as its
    submit returns.  A decode right after the submits, on other streams, waits for them.  The PCM of the gated run is
    the oracle's and the ungated run's."""
    spec, hdr, sts = streams(oracle, False)
    n_sub, per = 6, K * P // 6
    stride = stride_of(spec, per)
    n_out = S * CH * stride
    su, bt = make_batcher(ctx, hdr, RESIDUE, False)
    gate = Gate(ctx)
    runs = {}
    for gated in (False, True):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        arenas = [Arena(ctx, memory, n_out, np.float32) for _ in range(n_sub)]
        others = [L.PreviousWindowRight(su) for _ in range(S)]
        torch.cuda.synchronize()
        if gated:
            gate.close()
        tickets, arrs = [], []
        for k in range(n_sub):
            bufs = [[np.frombuffer(p, np.uint8).copy() for p in sts[s][0][k * per:(k + 1) * per]] for s in range(S)]
            arr, keep = c_jobs(pwrs, bufs, stride)
            tickets.append(c_submit(ctx, bt, arr, arenas[k].host.ctypes.data if memory == HOST else arenas[k].dev.data_ptr(), memory))
            for pk in bufs:
                for b in pk:
                    b[:] = 0xa5
            arrs.append((arr, keep, bufs))
            if gated and k == 1:
                gate.assert_closed("second lwf_batcher_submit")
        assert tickets == list(range(tickets[0], tickets[0] + n_sub))
        plain = fill(np.empty(S * CH * stride_of(spec, P), np.float32))
        res = bt.decode([(others[s], sts[s][0][:P]) for s in range(S)], plain, stride_of(spec, P))
        for s in range(S):
            n = res[s][0]
            assert res[s] == (n, P, 0)
            assert bits_equal(job_pcm(plain, s, n, stride_of(spec, P), cabi.OUT_F32_PLANAR), sts[s][1][:, :n]), s
        for t in tickets:
            ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, t))
        got = [a.read() for a in arenas]
        for s in range(S):
            parts = []
            for k, (arr, _, _) in enumerate(arrs):
                assert (arr[s].packets_done, arr[s].status) == (per, 0), (gated, k, s)
                parts.append(job_pcm(got[k], s, arr[s].n_samples, stride, cabi.OUT_F32_PLANAR))
            pcm = np.concatenate(parts, axis=1)
            assert bits_equal(pcm, sts[s][1]), (gated, s, mismatch_report(pcm, sts[s][1]))
        runs[gated] = got
        for p in pwrs + others:
            p.close()
    for a, b in zip(runs[False], runs[True]):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    bt.close()


@pytest.mark.parametrize("memory", [HOST, DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("entry", [RESIDUE, VQ], ids=["residue", "vq"])
def test_job_errors_and_refused_submits(ctx, oracle, entry, memory):
    """Jobs whose packet is cut short, whose packet header cannot be read (an empty packet, a header packet) or whose
    mode number is out of range get lwf_batcher_decode's results.  Refused submits (unknown out_format, unknown memory
    space, pageable host PCM, a stream in two jobs) leave job results, stream states and the PCM arena as they were,
    issue no ticket and launch no kernel; the next submit carries on as if they had not happened."""
    spec, hdr, sts = streams(oracle, False)
    assert len(spec.modes) == 3                       # two mode bits: mode 3 does not exist
    stride = stride_of(spec, P)
    n_out = S * CH * stride
    su, bt = make_batcher(ctx, hdr, entry, False)
    su2, twin = make_batcher(ctx, hdr, entry, False)
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    twins = [L.PreviousWindowRight(su2) for _ in range(S)]
    pk = [list(sts[s][0][:P]) for s in range(S)]
    pk[1][2] = pk[1][2][:max(2, len(pk[1][2]) // 3)]
    pk[2][1] = b""
    pk[3][3] = b"\x01bad"
    pk[4][2] = bytes([(pk[4][2][0] & ~0x06) | 0x06]) + pk[4][2][1:]
    arena = Arena(ctx, memory, n_out, np.float32)
    res = bt.submit([(pwrs[s], pk[s]) for s in range(S)], arena.pcm, stride).wait()
    want = fill(np.empty(n_out, np.float32))
    assert res == twin.decode([(twins[s], pk[s]) for s in range(S)], want, stride)
    assert np.array_equal(arena.read().view(np.uint8), want.view(np.uint8))
    assert_same_states(pwrs, twins, "errors")
    assert res[2][1:] == (1, fe.ERR_END_OF_PACKET) and res[3][1:] == (3, fe.ERR_AUDIO_IS_HEADER)
    assert res[4][1:] == (2, cabi.ERR_BAD_FORMAT)
    for s in (0, 5):
        assert res[s][1:] == (P, 0)
        assert bits_equal(job_pcm(want, s, res[s][0], stride, cabi.OUT_F32_PLANAR), sts[s][1][:, :res[s][0]])

    # refusals, on fresh streams that have decoded one submit
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    first = Arena(ctx, memory, n_out, np.float32)
    t0 = bt.submit([(p, sts[s][0][:P]) for s, p in enumerate(pwrs)], first.pcm, stride)
    t0.wait()
    before = [state(p) for p in pwrs]
    nxt = [(p, sts[s][0][P:2 * P]) for s, p in enumerate(pwrs)]
    arena = Arena(ctx, memory, n_out, np.float32)
    pageable = fill(np.empty(n_out, np.float32))
    cases = [("bad out_format", nxt, arena.pcm, 6, memory), ("bad memory space", nxt, arena.pcm, 0, 2),
             ("two jobs of one stream", nxt[:-1] + [(pwrs[0], sts[5][0][P:2 * P])], arena.pcm, 0, memory)]
    if memory == HOST:
        cases.append(("pageable host pcm", nxt, pageable, 0, HOST))
    for what, jobs, pcm, fmt, mem in cases:
        arr, _, n = bt._jobs(jobs, stride)
        for j in range(n):
            arr[j].n_samples, arr[j].packets_done, arr[j].status = 1234, 56, -7
        t = C.c_uint64(999)
        addr = pcm.ctypes.data if isinstance(pcm, np.ndarray) else (pcm if isinstance(pcm, int) else pcm.data_ptr())
        with expect_kernels(ctx, not_ran=ALL_KERNELS):
            rc = fe.lib().lwf_batcher_submit(bt._h, arr, n, fmt, addr, mem, C.byref(t))
        assert rc == cabi.ERR_INVALID, what
        assert t.value == 999, what
        assert all((arr[j].n_samples, arr[j].packets_done, arr[j].status) == (1234, 56, -7) for j in range(n)), what
        for p, b in zip(pwrs, before):
            a = state(p)
            assert (a is None) == (b is None) and (a is None or bits_equal(a, b)), what
        ctx.synchronize()
        assert not np.any(arena.read().view(np.uint32) != GUARDS[np.dtype(np.float32)][1]), what
        assert not np.any(pageable.view(np.uint32) != GUARDS[np.dtype(np.float32)][1]), what
    t1 = bt.submit(nxt, arena.pcm, stride)
    assert t1.id == t0.id + 1, "a refused submit issued a ticket"
    res = t1.wait()
    got = arena.read()
    for s in range(S):
        pcm = np.concatenate([job_pcm(first.read(), s, t0.wait()[s][0], stride, cabi.OUT_F32_PLANAR),
                              job_pcm(got, s, res[s][0], stride, cabi.OUT_F32_PLANAR)], axis=1)
        w = sts[s][1][:, :pcm.shape[1]]
        assert res[s][1:] == (P, 0) and bits_equal(pcm, w), (s, mismatch_report(pcm, w))
    for p in pwrs + twins:
        p.close()
    bt.close()
    twin.close()


@pytest.mark.parametrize("fmt", [cabi.OUT_F32_PLANAR, cabi.OUT_F16_INTERLEAVED], ids=["f32_planar", "f16_interleaved"])
def test_torch_tensor_pcm_equals_pinned_host_pcm(ctx, oracle, fmt):
    """A torch CUDA tensor as the PCM arena, read after wait(), equals the pinned-host arena of twin streams.  The
    batcher is closed before the wait: it waits for its submits before it frees its arenas, and the ticket stays valid."""
    spec, hdr, sts = streams(oracle, True)
    stride = stride_of(spec, K * P)
    dt = FORMATS[fmt]
    outs = {}
    for memory in (HOST, DEVICE):
        su, bt = make_batcher(ctx, hdr, VQ, True)
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        arena = Arena(ctx, memory, S * CH * stride, dt)
        if memory == DEVICE:
            assert isinstance(arena.pcm, torch.Tensor) and arena.pcm.is_cuda
        t = bt.submit([(pwrs[s], sts[s][0]) for s in range(S)], arena.pcm, stride, fmt)
        bt.close()
        res = t.wait()
        outs[memory] = (arena.read(), res, [state(p) for p in pwrs])
        for s in range(S):
            assert res[s][1:] == (K * P, 0)
            assert_oracle(oracle, job_pcm(outs[memory][0], s, res[s][0], stride, fmt), sts[s][1], fmt, (memory, s))
        for p in pwrs:
            p.close()
    assert np.array_equal(outs[HOST][0].view(np.uint8), outs[DEVICE][0].view(np.uint8))
    assert outs[HOST][1] == outs[DEVICE][1]
    for a, b in zip(outs[HOST][2], outs[DEVICE][2]):
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b))

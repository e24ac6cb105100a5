"""OggStreamReaders' seek_absgp_pg and skip_samples_linear (lwf_readers_seek_absgp_pg, lwf_readers_skip_samples_linear)
on the GPU.  Every file of the readers' nine-file corpus (tests/test_ogg_readers_gpu.py: chained, foreign, errors,
spanning pages, floor 0, ten channels, granule positions above and below the decoded count) runs one script of reads,
seeks and skips on a single OggStreamReader and, in batched calls, on one OggStreamReaders -- reads and skips left
queued while the next call is issued, in every sample format and layout, into host and device PCM.  After every
operation each reader must agree with its single reader: PCM (f32 bit for bit, i16/f16 exactly), got_packet,
left_to_skip, status, absgp, headers and channel count, and the next read's packets; nothing outside the written samples
may change.  A skip batch of a uniform stereo corpus must run on the fused kernels."""
import ctypes as C

import numpy as np
import pytest

from helpers import FUSED, GENERIC, assert_contained, expect_kernels, launches_are_attributed
from lewton_b200 import frontend as fe
from lewton_b200.api import sample_format
from test_frontend_gpu import consistent_modes, oracle_pcm
from test_ogg_readers_gpu import (ALL, FORMATS, _buffer, _host, audio_pages, corpus, ctx, granules, header_pages,  # noqa: F401
                                  same_samples, single_trace, stream)

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

# (op, argument): "read" max_packets, "seek" absgp ("last": the last page's granule position), "skip" to_skip (one
# count for every file, or a list with one per file)
SCRIPT = [("read", 1), ("skip", 3), ("read", 3), ("seek", 3000), ("skip", 2500), ("read", ALL), ("seek", 0),
          ("read", ALL), ("skip", 10 ** 5), ("seek", "last"), ("skip", 40), ("read", 3), ("seek", 10 ** 9), ("read", 1),
          ("seek", 0), ("skip", 3), ("read", ALL), ("skip", 10 ** 7), ("read", 1)]


def last_granule(data):
    """The granule position of the file's last page that has one."""
    at, g = 0, 0
    while at + 27 <= len(data):
        v = int.from_bytes(data[at + 6: at + 14], "little")
        if v != (1 << 64) - 1:
            g = v
        at += 27 + data[at + 26] + sum(data[at + 27: at + 27 + data[at + 26]])
    return g


def planar(pcm, ch, interleaved):
    """[ch][n] from a single reader's packet or a batched job's slice"""
    if interleaved:
        return pcm.reshape(-1, ch).T
    return np.stack(pcm) if len(pcm) else np.zeros((ch, 0))


def same_error(got_status, want, ctx, what):
    e = fe.read_error(ctx, got_status)
    assert type(e) is type(want) and str(e) == str(want), (what, got_status, want)


class Single:
    """The single reader's side of the script"""

    def __init__(self, ctx, data, sample, interleaved):
        self.ctx, self.rd, self.sample, self.itl = ctx, fe.OggStreamReader(ctx, data), sample, interleaved

    def _call(self, skip=None):
        """One lwf_reader_read_dec_packet (skip None) or lwf_reader_skip_samples_linear call through the C ABI, laid
        out with the channel count of the reader's headers after the call (as single_trace does)"""
        lib = fe.lib()
        fmt, dt = sample_format(self.sample, self.itl and skip is None)
        cap = 16 * 8192
        buf = np.zeros(cap, dt)
        n, left, got = C.c_size_t(), C.c_size_t(), C.c_int(1)
        if skip is None:
            rc = lib.lwf_reader_read_dec_packet(self.rd._h, fmt, buf.ctypes.data, cap, C.byref(n))
        else:
            rc = lib.lwf_reader_skip_samples_linear(self.rd._h, skip, fmt, buf.ctypes.data, cap, C.byref(n), C.byref(left),
                                                    C.byref(got))
        if rc == fe.ERR_NO_MORE_PACKETS or (rc == 0 and not got.value):
            return None if skip is None else (None, left.value)
        if rc:
            return fe.read_error(self.ctx, rc)
        ch, n = self.channels, n.value
        if self.itl and skip is None:
            return buf[: n * ch].copy()
        pk = [buf[c * (cap // ch): c * (cap // ch) + n].copy() for c in range(ch)]
        return pk if skip is None else (pk, left.value)

    def read(self):
        return self._call()

    def skip(self, n):
        return self._call(skip=n)

    def seek(self, g):
        try:
            self.rd.seek_absgp_pg(g)
        except Exception as e:      # noqa: BLE001
            return e
        return None

    @property
    def headers(self):
        """the reader's headers now (also after a call that raised, which OggStreamReader.headers may not show yet)"""
        return fe.Headers(None, None, None, _handle=fe.lib().lwf_reader_headers(self.rd._h))

    @property
    def channels(self):
        return self.headers.audio_channels


def run_script(ctx, files, sample, interleaved, memory, script=SCRIPT, threads=4):
    """Runs `script` on a single reader and on one OggStreamReaders per file and compares them after every operation.
    Returns the readers and, per step, the batched call's results (None for a seek)."""
    _, dt = sample_format(sample, interleaved)
    log = []
    singles = [Single(ctx, d, sample, interleaved) for d in files]
    rs = fe.OggStreamReaders(ctx, threads=threads)
    idx = [rs.add(d) for d in files]
    chained_after = [False] * len(files)          # the last batched read stopped at a chained stream
    pending = []

    def check(item):
        t, buf, want, what = item
        t.wait()
        host = _host(buf, dt)
        spans = []
        for i, (off, stride, ch, n, pkts) in enumerate(want):
            s0 = 0
            for k, w in enumerate(pkts):
                m = w.shape[1]
                if interleaved:
                    got = host[off + s0 * ch: off + (s0 + m) * ch].reshape(m, ch).T
                else:
                    got = np.stack([host[off + c * stride + s0: off + c * stride + s0 + m] for c in range(ch)])
                assert same_samples(got, w, sample), (what, i, k)
                s0 += m
            assert s0 == n, (what, i, s0, n)
            if interleaved:
                spans.append((i, [(off, n * ch)] if n else []))
            else:
                spans.append((i, [(off + c * stride, n) for c in range(ch)] if n else []))
        assert_contained(host, spans, what)

    for step, (op, arg) in enumerate(script):
        what = "step %d %s %r" % (step, op, arg)
        if op == "seek":
            goals = [last_granule(d) if arg == "last" else arg for d in files]
            got = rs.seek_absgp_pg(idx, goals)
            for i, s in enumerate(singles):
                want = s.seek(goals[i])
                if want is None:
                    assert got[i] is None, (what, i, got[i])
                else:
                    assert type(got[i]) is type(want) and str(got[i]) == str(want), (what, i, got[i], want)
                chained_after[i] = False
            log.append(None)
        elif op == "read":
            stride = max(1, max(rs.stride(j, arg) for j in idx))
            chs = [rs.headers(j).audio_channels for j in idx]
            buf = _buffer(ctx, memory, sum(chs) * stride + 64, dt)
            t = rs.read([(j, arg) for j in idx], buf, stride, sample, interleaved)
            want = []
            for i, (r, s) in enumerate(zip(t.results, singles)):
                w = "%s file %d %r" % (what, i, r)
                pkts = []
                for k in range(r.n_packets):
                    p = s.read()
                    assert p is not None and not isinstance(p, Exception), (w, k, p)
                    pk = planar(p, r.channels, interleaved)
                    assert pk.shape[1] == r.packet_samples[k], (w, k)
                    pkts.append(pk)
                if r.status:
                    same_error(r.status, s.read(), ctx, w)
                elif r.ended:
                    assert s.read() is None, w
                elif not r.next_chained:
                    assert r.n_packets == arg, w
                assert r.channels == s.channels or (r.next_chained and not r.n_packets), w
                chained_after[i] = r.next_chained
                want.append((r.out_offset, stride, r.channels, r.n_samples, pkts))
            pending.append((t, buf, want, what))
            log.append(t.results)
        else:
            counts = arg if isinstance(arg, list) else [arg] * len(files)
            rooms = [rs.skip_room(j) for j in idx]
            stride = max(st for _, st in rooms)
            buf = _buffer(ctx, memory, sum(c for c, _ in rooms) * stride + 64, dt)
            t = rs.skip_samples_linear(list(zip(idx, counts)), buf, stride, sample, interleaved)
            want = []
            for i, (r, s) in enumerate(zip(t.results, singles)):
                w = "%s file %d %r" % (what, i, r)
                single = s.skip(counts[i])
                pkts = []
                if isinstance(single, Exception):
                    assert not r.got_packet, w
                    same_error(r.status, single, ctx, w)
                else:
                    assert not r.status, (w, single)
                    pk, left = single
                    assert r.left_to_skip == left, (w, left)
                    assert r.got_packet == (pk is not None), w
                    if pk is not None:
                        # the single reader's skip is planar; the batched job is laid out as asked
                        pkts.append(np.stack(pk))
                        assert pkts[0].shape == (r.channels, r.n_samples), (w, pkts[0].shape)
                assert r.channels == s.channels, w
                chained_after[i] = False
                want.append((r.out_offset, stride, r.channels, r.n_samples if r.got_packet else 0, pkts))
            pending.append((t, buf, want, what))
            log.append(t.results)
        # absgp, headers and channels after every operation (a read that stopped at a chained stream stands at the new
        # stream's headers, which the single reader reaches with its next call)
        for i, s in enumerate(singles):
            assert rs.get_last_absgp(idx[i]) == s.rd.get_last_absgp(), (what, i)
            if not chained_after[i]:
                h, g = rs.headers(idx[i]), s.headers
                assert (h.audio_channels, h.blocksize_0, h.blocksize_1, h.audio_sample_rate, h.vendor, h.comment_list) == \
                    (g.audio_channels, g.blocksize_0, g.blocksize_1, g.audio_sample_rate, g.vendor, g.comment_list), (what, i)
        if len(pending) == 2:
            check(pending.pop(0))                  # the older of two queued calls
    while pending:
        check(pending.pop(0))
    # the next read's packets agree to the end
    for i, s in enumerate(singles):
        for _ in range(40):
            got = rs.read_dec_packets([idx[i]], 1, sample, interleaved)[0]
            if not got:
                continue                           # stopped at a chained stream: the single reader crosses next
            want = s.read()
            g = got[0]
            if want is None or isinstance(want, Exception):
                assert (g is None and want is None) or (type(g) is type(want) and str(g) == str(want)), (i, g, want)
                if want is None or isinstance(want, fe.OggReadError):
                    break
                continue
            assert same_samples(planar(g, s.channels, interleaved), planar(want, s.channels, interleaved), sample), i
        s.rd.close()
    return rs, log


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("sample,interleaved", FORMATS)
def test_seek_and_skip_return_what_the_single_reader_returns(ctx, corpus, sample, interleaved, memory):
    files = [d for d, _ in corpus.values()]
    run_script(ctx, files, sample, interleaved, memory)[0].close()


def test_seek_after_next_chained_goes_back_to_the_stream_before(ctx, corpus):
    """A read that stops at the chained file's second stream has read its headers; a seek then seeks in the first
    stream, as the single reader (which has not read them) does, and the readers read on from there."""
    data = corpus["chained"][0]
    script = [("read", ALL), ("seek", 2000), ("read", 2), ("read", ALL), ("seek", 0), ("skip", 3), ("read", ALL),
              ("read", ALL), ("skip", 10 ** 4), ("read", ALL)]
    run_script(ctx, [data], "f32", False, "host", script=script)[0].close()


def returned(ctx, data):
    """Samples per channel of every packet the single reader returns reading `data` from its start"""
    return [e[1].shape[1] for e in single_trace(ctx, data, "f32", False) if e[0] == "pkt"]


# files whose first stream's last packet is cut by its granule position and whose granule position is known after 4
# packets: (name, index of that packet among the packets the single reader returns)
TRUNCATED = [("stereo_256_2048_cut", 13), ("stereo_floor0_mid_page", 7), ("chained", 6)]
FOREIGN_LAST = 8


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("sample,interleaved", FORMATS)
def test_skip_into_the_truncated_last_packet(ctx, corpus, sample, interleaved, memory):
    """After 4 packets, a skip that lands 2 samples into the last packet of each file's (first) stream.  The granule
    position is known and the state is not fresh, so the single reader decodes that packet alone on the state it stands
    in (inside_ogg.rs:258-262) and cuts it to its page's granule position: the batched job's target is cut by the
    stream's output window, and it returns what the single reader returns."""
    names = list(corpus)
    files = [corpus[n][0] for n in names]
    last = dict(TRUNCATED + [("foreign", FOREIGN_LAST)])
    counts = []
    for n, d in zip(names, files):
        got = returned(ctx, d)
        k = last.get(n, len(got) - 1 if n not in ("errors", "headers_only") else None)
        counts.append(sum(got[4:k]) + 2 if k is not None and k > 4 else 3)
    rs, log = run_script(ctx, files, sample, interleaved, memory, script=[("read", 4), ("skip", counts), ("read", 3)])
    # the foreign file's last packet lands on the state of its fourth, whose block size differs: the overlap guard
    # refuses it (LWB_ERR_BAD_FORMAT) in the single reader and in the batch, which clears the stream state
    r = log[1][names.index("foreign")]
    assert not r.got_packet and r.status == 1 and r.left_to_skip == counts[names.index("foreign")], r
    for n, k in TRUNCATED:
        i = names.index(n)
        r = log[1][i]
        full = (corpus[n][1][0] if n == "chained" else corpus[n][1])[k].shape[1]
        assert r.got_packet and r.left_to_skip == 2 and r.n_samples == returned(ctx, files[i])[k] < full, (n, r, full)
    rs.close()


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("sample,interleaved", FORMATS)
def test_skip_into_a_chained_stream(ctx, corpus, sample, interleaved, memory):
    """Skips whose target lies in the chained file's second stream (mono 512/4096 after stereo 256/2048), against the
    single reader: from the middle of the first stream to the middle of the second ([packet before, target] on a reset
    state) and to its first returned packet (the packet before is the first stream's last); and from a read that stopped
    at the second stream (the drop pending) to its first returned packet ([dropped packet, target] on the fresh state)
    and its third."""
    data = corpus["chained"][0]
    n = returned(ctx, data)                         # stream 1: n[0:7]; stream 2 after its dropped packet: n[7:11]
    cases = [([("read", 2), ("skip", sum(n[2:9]) + 5)], 9, 5),
             ([("read", 2), ("skip", sum(n[2:7]) + 5)], 7, 5),
             ([("read", ALL), ("skip", 3)], 7, 3),
             ([("read", ALL), ("skip", sum(n[7:9]) + 3)], 9, 3)]
    for script, k, left in cases:
        rs, log = run_script(ctx, [data], sample, interleaved, memory, script=script + [("read", 3), ("seek", 0), ("read", 2)])
        r = log[1][0]
        if r.got_packet:
            assert r.channels == 1 and r.left_to_skip == left and r.n_samples == n[k], (script, r)
        else:
            assert k == 7 and r.status, (script, r)      # the first stream's last packet decoded with the second's headers
        rs.close()


def test_skip_samples_linear_dec_lays_out_a_chained_target(ctx, corpus):
    """skip_samples_linear_dec returns a target in the second stream with that stream's channel count, planar and
    interleaved, as the single reader returns it."""
    data = corpus["chained"][0]
    n = returned(ctx, data)
    for sample, interleaved in (("f32", False), ("i16", True), ("f16", False)):
        single = Single(ctx, data, sample, False)
        rs = fe.OggStreamReaders(ctx)
        rs.add(data)
        rs.read_dec_packets([0], 2)
        for _ in range(2):
            single.read()
        (pk, left), = rs.skip_samples_linear_dec([0], sum(n[2:9]) + 5, sample, interleaved)
        want, wleft = single.skip(sum(n[2:9]) + 5)
        assert left == wleft == 5
        got = planar(pk, 1, interleaved)
        assert got.shape == (1, n[9]) and same_samples(got, np.stack(want), sample)
        rs.close()
        single.rd.close()


def test_skip_batches_of_a_uniform_corpus_run_on_the_fused_kernels(ctx, oracle):
    """Skips of sixteen stereo 256/2048 files of one encoder setting -- chains of the packet before the target and the
    target on a reset state -- go to the fused kernels, not to k_chain or the four-kernel path."""
    spec, _, _ = stream(811, 2)
    files = []
    rng = np.random.default_rng(812)
    for k in range(16):
        spec.rng = rng
        packets, infos = [], []
        for mode, prev, nxt in consistent_modes(spec, rng, 12, p_short=0.2 if k % 2 else 0.0):
            pk, info = spec.audio_packet(mode, prev, nxt)
            packets.append(pk)
            infos.append(info)
        want, _ = oracle_pcm(oracle, spec, infos)
        files.append(header_pages(200 + k, spec) + b"".join(audio_pages(200 + k, packets, granules(want, 7), per_page=4)))
    rs = fe.OggStreamReaders(ctx, threads=4)
    idx = [rs.add(d) for d in files]
    rooms = [rs.skip_room(j) for j in idx]
    stride = max(s for _, s in rooms)
    buf = _buffer(ctx, "device", sum(c for c, _ in rooms) * stride + 64, np.float32)
    singles = [Single(ctx, d, "f32", False) for d in files]
    with expect_kernels(ctx, not_ran=GENERIC | {"k_chain"}) as ran:
        for to_skip in (5000, 3):
            t = rs.skip_samples_linear([(j, to_skip + 97 * j) for j in idx], buf, stride)
            t.wait()
            host = _host(buf, np.float32)
            for i, r in enumerate(t.results):
                pk, left = singles[i].skip(to_skip + 97 * i)
                assert r.got_packet and r.left_to_skip == left and not r.status, (i, r)
                got = np.stack([host[r.out_offset + c * stride: r.out_offset + c * stride + r.n_samples] for c in range(2)])
                assert same_samples(got, np.stack(pk), "f32"), i
    assert ran["k_long"] + ran["k_long_s"] + ran["k_mid"] > 0, ran
    assert set(k for k, v in ran.items() if v) <= FUSED | {"k_row_copy", "k_floor1_segments", "k_prologue_fused"}, ran
    rs.close()
    for s in singles:
        s.rd.close()

"""Output windows (lwb_stream_set_window) with the host front half, on the GPU.

* LWB_ENTRY_VQ batches of packer-made streams (VQ records from the front half's entropy decode) on k_long and on the
  one-pass mixed schedule, in host and device memory: the windowed decode writes exactly the window of the unwindowed
  one, which equals the oracle's decode; every other element keeps its sentinel; the stream states are the unwindowed
  ones; the batch runs the unwindowed batch's kernels plus one k_row_copy.
* The stream batcher against OggStreamReader: packer-made Ogg streams decoded packet by packet through
  StreamBatcher.submit, with the last packet of each stream given the window (0, final granule position - samples
  written) -- what the reader does on the host, inside_ogg.rs:219-222 -- equal the reader's output packet for packet,
  n_samples included.  And seek_absgp_pg followed by a skip window (a reset, then set_window(target - page start))
  equals the matching slice of a full decode and of the reader's own output after the same seek."""
import numpy as np
import pytest
import torch

import lewton_b200 as L
import vorbis_packer as vp
from helpers import bits_equal, expect_kernels, launches_are_attributed, mismatch_report
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from test_frontend_gpu import consistent_modes, oracle_pcm, page_granules
from test_stream_windows_gpu import F32P, Arena, check_batch, deinterleave

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


class _Stream:
    """A windowed stream and its unwindowed twin over one packer-made packet sequence."""

    def __init__(self, su, pkts, infos, want, window):
        self.win, self.full = L.PreviousWindowRight(su), L.PreviousWindowRight(su)
        self.pkts, self.infos, self.want, self.window = pkts, infos, want, window
        self.at = self.pos = 0
        if window:
            self.win.set_window(*window)

    def expect(self, n):
        if not self.window:
            return 0, n
        skip, limit = self.window
        end = np.inf if limit is None else skip + limit
        a = int(min(max(skip - self.pos, 0), n))
        return a, int(max(a, min(end - self.pos, n)))


class _VqBatch:
    """The next k packets of every stream as one LWB_ENTRY_VQ batch (the attributes check_batch reads)."""

    def __init__(self, hdr, su, streams, k):
        self.fmt, self.streams, self.parts, self.K = F32P, streams, [], [su.output_channels] * len(streams)
        kinds, ys, runs, ents, roffs, eoffs = [], [], [], [], [0], [0]
        self.specs, self.coeff_offs, coeff = [], [], 0
        for st in streams:
            pk = st.pkts[st.at:st.at + k]
            st.at += k
            modes, prevs, nexts, n, has = [], [], [], 0, not st.full.is_empty()
            self.coeff_offs.append(coeff)
            for p in pk:
                dense = hdr.decode_packet(p)
                dp, rr, ee = hdr.decode_packet_vq(p)
                kd, y, _ = dense.pack()
                coeff += dense.residue.size           # (the device-only coefficient arena is laid out by coeff_offset)
                kinds.append(kd)
                ys.append(y)
                runs.append(rr)
                ents.append(ee)
                roffs.append(roffs[-1] + len(rr))
                eoffs.append(eoffs[-1] + len(ee))
                modes.append(dp.mode_number)
                prevs.append(dp.prev_window_flag)
                nexts.append(dp.next_window_flag)
                if has:
                    n += L.get_decoded_sample_count(su, dp.mode_number, dp.prev_window_flag, dp.next_window_flag)
                has = True
            self.specs.append((np.array(modes, np.uint8), np.array(prevs, np.uint8), np.array(nexts, np.uint8)))
            self.parts.append((None,) * 7 + (n,))
        self.kinds, self.ys = np.concatenate(kinds), np.concatenate(ys)
        self.vq = (np.concatenate(runs) if roffs[-1] else np.zeros(1, fe.VQ_RUN_DTYPE), np.array(roffs, np.uint64),
                   np.concatenate(ents) if eoffs[-1] else np.zeros(1, np.uint16), np.array(eoffs, np.uint64))
        C = self.K[0]
        self.full_lay, self.win_lay, fo, wo = [], [], 0, 0
        for i, p in enumerate(self.parts):
            n = p[7]
            self.full_lay.append((fo, n))
            fo += C * n
            self.win_lay.append((wo, n + 8))
            wo += C * (n + 8) + 4
        self.full_elems, self.win_elems = max(fo, 1), wo + 8

    def chains(self, which, lay, k):
        return [L.ChainSpec(getattr(st, which), *self.specs[i], coeff_offset=self.coeff_offs[i], packet_index=i * k, out_offset=lay[i][0], out_stride=lay[i][1])
                for i, st in enumerate(self.streams)]


@pytest.mark.parametrize("memory", [cabi.MEM_DEVICE, cabi.MEM_HOST], ids=["device", "host"])
@pytest.mark.parametrize("p_short,kernel", [(0.0, "k_long"), (0.3, "k_long_s")], ids=["k_long", "one_pass"])
def test_vq_entry_windows(ctx, oracle, p_short, kernel, memory):
    rng = np.random.default_rng(611)
    spec = vp.StreamSpec(rng, channels=2, bs0=8, bs1=11)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    assert hdr.vq_capable()
    su = hdr.make_setup(ctx)
    windows = [(100, None), None, (0, 1500), (3000, 40), (1700, 2600), (5000, None), (0, 10), (700, 0)]
    k, n_batches, streams = 4, 3, []
    for s in range(8):
        pkts, infos = [], []
        for mode, prev, nxt in consistent_modes(spec, rng, k * n_batches, p_short=p_short):
            pk, info = spec.audio_packet(mode, prev, nxt, p_unused=0.1)
            pkts.append(pk)
            infos.append(info)
        want = oracle_pcm(oracle, spec, infos)[0]
        streams.append(_Stream(su, pkts, infos, np.concatenate(want, axis=1), windows[s]))
    full_pcm = [[] for _ in streams]
    for _ in range(n_batches):
        b = _VqBatch(hdr, su, streams, k)
        fa, wa = Arena(ctx, b.full_elems, F32P, memory), Arena(ctx, b.win_elems, F32P, memory)
        fch, wch = b.chains("full", b.full_lay, k), b.chains("win", b.win_lay, k)
        kw = dict(floor_kind=b.kinds, floor1_y=b.ys, vq=b.vq)
        deltas = []
        for ch, ar in ((fch, fa), (wch, wa)):
            with expect_kernels(ctx) as d:
                L.decode_chains(ctx, ch, cabi.ENTRY_VQ, memory, None, ar.ptr, F32P, **kw)
                if memory == cabi.MEM_DEVICE:
                    ctx.synchronize()
            deltas.append(d)
        fbuf, wbuf = fa.read(), wa.read()
        moved = any(st.expect(p[7]) != (0, p[7]) and st.expect(p[7])[1] > st.expect(p[7])[0] for st, p in zip(streams, b.parts))
        for i, p in enumerate(b.parts):
            full_pcm[i].append(deinterleave(fbuf.view(np.float32)[b.full_lay[i][0]:], F32P, b.K[i], p[7]))
        check_batch(b, fch, wch, fbuf, wbuf)
        assert deltas[0][kernel] > 0, deltas[0]
        want = dict(deltas[0])
        want["k_row_copy"] += 1 if moved else 0
        assert deltas[1] == want, deltas
    for st, parts in zip(streams, full_pcm):
        got = np.concatenate(parts, axis=1)
        assert bits_equal(got, st.want), mismatch_report(got, st.want)
        assert st.win.is_empty() == st.full.is_empty() and bits_equal(st.win.data(), st.full.data())


def _ogg_streams(oracle, rng, spec, n, P, per_page):
    """n packer-made Ogg streams of P audio packets: (bytes, packets, oracle PCM per packet, page granules, cut)."""
    out = []
    for s in range(n):
        pkts, infos = [], []
        for mode, prev, nxt in consistent_modes(spec, rng, P, p_short=0.3):
            pk, info = spec.audio_packet(mode, prev, nxt, p_unused=0.1)
            pkts.append(pk)
            infos.append(info)
        want = oracle_pcm(oracle, spec, infos)[0]
        last, prev_last = want[-1].shape[1], want[-2].shape[1]
        # truncated inside the last packet, not at all, behind the samples before it (lewton gives 0), to half
        cut = [37, 0, last + prev_last // 2, last // 2][s % 4]
        gran = page_granules(want, per_page, cut)
        data = vp.ogg_stream(0x100 + s, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], pkts, gran, packets_per_page=per_page)
        out.append((data, pkts, want, gran, cut))
    return out


def _pcm_buffer(ctx, memory, n):
    if memory == cabi.MEM_HOST:
        buf = ctx.host_alloc(n, np.float32)
        buf[...] = np.nan
        return buf, lambda: np.array(buf)
    t = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    return t, lambda: (torch.cuda.synchronize(), t.cpu().numpy())[1]


@pytest.mark.parametrize("entry", [cabi.ENTRY_RESIDUE, cabi.ENTRY_VQ], ids=["residue", "vq"])
@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE], ids=["host", "device"])
def test_batcher_end_of_stream_windows_equal_the_reader(ctx, oracle, memory, entry):
    rng = np.random.default_rng(621)
    spec = vp.StreamSpec(rng, channels=2, bs0=8, bs1=11)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    su = hdr.make_setup(ctx)
    S, P, per_page, C = 8, 11, 3, 2
    streams = _ogg_streams(oracle, rng, spec, S, P, per_page)
    reader = []
    for data, _, _, _, _ in streams:
        rd = fe.OggStreamReader(ctx, data)
        reader.append([np.array(rd.read_dec_packet_f32(), np.float32).reshape(C, -1) for _ in range(P)])
        assert rd.read_dec_packet_f32() is None
        rd.close()
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    written = [0] * S
    stride = 1 << spec.bs1                  # (a long packet between short neighbours produces up to 3/4 of it)
    bt = fe.StreamBatcher(ctx, hdr, threads=2, entry=entry)
    for j in range(P):                      # one packet of every stream per submit: packet for packet
        if j == P - 1:
            for s in range(S):
                final = streams[s][3][-1]
                pwrs[s].set_window(0, max(final - written[s], 0))     # inside_ogg.rs:219-222
        buf, read = _pcm_buffer(ctx, memory, S * C * stride)
        res = bt.submit([(pwrs[s], [streams[s][1][j]]) for s in range(S)], buf, stride).wait()
        pcm = read()
        for s in range(S):
            want = reader[s][j]
            n_samples, done, status = res[s]
            assert (done, status) == (1, 0) and n_samples == want.shape[1], (j, s, res[s], want.shape)
            got = pcm[s * C * stride:(s + 1) * C * stride].reshape(C, stride)
            assert bits_equal(got[:, :n_samples], want), (j, s, mismatch_report(got[:, :n_samples], want))
            assert np.isnan(got[:, n_samples:]).all(), (j, s)
            written[s] += n_samples
    for s in range(S):
        assert written[s] == sum(r.shape[1] for r in reader[s])
        if s % 4 != 2:                      # (s % 4 == 2: a final granule position behind the samples before the last packet)
            assert written[s] == streams[s][3][-1]
        assert pwrs[s].window == (0, 0)
    bt.close()


@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE], ids=["host", "device"])
def test_seek_then_skip_window_equals_a_slice_of_the_full_decode(ctx, oracle, memory):
    rng = np.random.default_rng(631)
    spec = vp.StreamSpec(rng, channels=2, bs0=8, bs1=11)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    su = hdr.make_setup(ctx)
    P, per_page, C = 17, 3, 2
    data, pkts, want, gran, cut = _ogg_streams(oracle, rng, spec, 1, P, per_page)[0]
    full = np.concatenate(want, axis=1)
    lens = [w.shape[1] for w in want]
    bt = fe.StreamBatcher(ctx, hdr, threads=2)
    pwr = L.PreviousWindowRight(su)
    stride = P * (1 << spec.bs1) // 2
    buf, read = _pcm_buffer(ctx, memory, C * stride)
    bt.submit([(pwr, pkts[:5])], buf, stride).wait()       # the stream is somewhere else when the seek comes
    for goal in (gran[2] + 5, gran[4] + 50, gran[1]):
        rd = fe.OggStreamReader(ctx, data)
        rd.seek_absgp_pg(goal)
        after = []
        while (p := rd.read_dec_packet_f32()) is not None:
            after.append(np.array(p, np.float32).reshape(C, -1))
        rd.close()
        q = P - len(after)                                  # the packet the seek landed on: it decodes to nothing
        start = sum(lens[:q + 1])                           # the full decode's sample the next packet starts at
        assert after[0].shape[1] == 0 and start <= goal
        pwr.reset()
        pwr.set_window(goal - start)
        buf, read = _pcm_buffer(ctx, memory, C * stride)
        (n_samples, done, status), = bt.submit([(pwr, pkts[q:])], buf, stride).wait()
        assert (done, status) == (P - q, 0) and n_samples == full.shape[1] - goal
        got = read().reshape(C, stride)[:, :n_samples]
        assert bits_equal(got, full[:, goal:]), (goal, mismatch_report(got, full[:, goal:]))
        rd_pcm = np.concatenate(after, axis=1)[:, goal - start:]       # the reader's last packet is truncated by `cut`
        assert bits_equal(got[:, :rd_pcm.shape[1]], rd_pcm) and rd_pcm.shape[1] == n_samples - cut
        assert pwr.window == (0, None)
    bt.close()

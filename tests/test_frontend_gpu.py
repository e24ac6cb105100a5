"""End to end on the GPU: synthetic Ogg/Vorbis bytes (tests/vorbis_packer.py) -> host front half
(Ogg paging, headers, entropy decode) -> CUDA synthesis, against the CPU oracle fed with what the
packer knows it encoded.  Covers the OggStreamReader loop (per packet, inside_ogg.rs:60-227: sample
counts, end-of-stream truncation, absgp accounting) and the batched residue entry driven by real
bitstreams (SURVEY.md configs 1 and 3 shapes)."""
import numpy as np
import pytest

import lewton_b200 as L
import vorbis_packer as vp
from helpers import (ALL_KERNELS, FRONT, RefStream, bits_equal, expect_kernels, launches_are_attributed,
                     mismatch_report)
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from test_frontend_cpu import floor0_expected

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def consistent_modes(spec, rng, n_packets, p_short=0.3):
    """A legal block sequence: (mode, prev_flag, next_flag) per packet, flags describing the neighbours."""
    short_modes = [i for i, (bf, _) in enumerate(spec.modes) if not bf]
    long_modes = [i for i, (bf, _) in enumerate(spec.modes) if bf]
    bf = [(rng.random() >= p_short) for _ in range(n_packets)]
    out = []
    for i in range(n_packets):
        mode = int(rng.choice(long_modes if bf[i] else short_modes))
        prev = int(bf[i - 1]) if i else 1
        nxt = int(bf[i + 1]) if i + 1 < n_packets else 1
        out.append((mode, prev, nxt))
    return out


def build_stream(seed, channels, floor0, n_packets, serial=1, cut_last=0):
    rng = np.random.default_rng(seed)
    spec = vp.StreamSpec(rng, channels=channels, floor0=floor0)
    seq = consistent_modes(spec, rng, n_packets)
    packets, infos = [], []
    for mode, prev, nxt in seq:
        pk, info = spec.audio_packet(mode, prev, nxt, p_unused=0.15)
        packets.append(pk)
        infos.append(info)
    return spec, packets, infos


def oracle_pcm(oracle, spec, infos):
    """Decode the packer's own record of every packet with the CPU oracle: list of [channels][n] f32."""
    floors = [(f.multiplier, f.x_list) if isinstance(f, vp.Floor1) else (1, [0, 128]) for f in spec.floors]
    mappings = []
    for m in spec.mappings:
        mappings.append({"coupling": m["coupling"], "floor_of_channel": [m["floors"][m["mux"][c]] for c in range(spec.channels)]})
    ref = RefStream(oracle, spec.channels, spec.bs0, spec.bs1, spec.modes, mappings, floors)
    out = []
    for info in infos:
        fl_exp, res = spec.expected(info)
        n2 = info["n"] // 2
        fl = []
        for f in fl_exp:
            if f is None:
                fl.append(None)
            elif f[0] == "one":
                fl.append(list(f[1]))
            else:
                fl.append(floor0_expected(f[3], f[1], f[2], info["blockflag"], n2, spec.bs0, spec.bs1))
        rc, pcm = ref.packet(info["mode"], info["prev"], info["next"], res, fl)
        assert rc == 0
        out.append(pcm)
    return out, ref


def page_granules(pcm_list, per_page, cut_last):
    """absgp of each audio page = samples decoded up to its last packet; the last page claims
    `cut_last` samples fewer (end-of-stream truncation, inside_ogg.rs:219-222)."""
    tot, out = 0, []
    for i in range(0, len(pcm_list), per_page):
        tot += sum(p.shape[1] for p in pcm_list[i: i + per_page])
        out.append(tot)
    out[-1] -= cut_last
    return out


@pytest.mark.parametrize("seed,channels,floor0", [(101, 2, False), (102, 1, True), (103, 6, False), (104, 2, True)])
def test_ogg_stream_reader_end_to_end(ctx, oracle, seed, channels, floor0):
    spec, packets, infos = build_stream(seed, channels, floor0, 14)
    want, ref = oracle_pcm(oracle, spec, infos)
    cut = 37
    assert want[-1].shape[1] > cut
    data = vp.ogg_stream(0x1234, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets,
                         page_granules(want, 3, cut), packets_per_page=3)
    for api in ("f32", "i16", "itl"):
        rd = fe.OggStreamReader(ctx, data)
        assert rd.headers.audio_channels == channels and rd.headers.vendor == spec.vendor
        assert rd.get_last_absgp() is None
        total = 0
        for i, w in enumerate(want):
            n = w.shape[1] - (cut if i == len(want) - 1 else 0)
            if api == "f32":
                got = rd.read_dec_packet_f32()
                assert len(got) == channels and all(len(g) == n for g in got), (i, n, [len(g) for g in got])
                assert bits_equal(np.array(got).reshape(channels, n), w[:, :n]), (i, mismatch_report(np.array(got), w[:, :n]))
            elif api == "i16":
                got = rd.read_dec_packet()
                assert np.array_equal(np.array(got).reshape(channels, n), oracle.quantise_i16(w[:, :n])), i
            else:
                got = rd.read_dec_packet_itl()
                assert np.array_equal(got.reshape(n, channels), oracle.quantise_i16(w[:, :n]).T), i
            total += n
            if (i + 1) % 3 == 0 or i == len(want) - 1:
                assert rd.get_last_absgp() == sum(x.shape[1] for x in want[: i + 1]) - (cut if i == len(want) - 1 else 0)
        assert rd.read_dec_packet() is None
        rd.close()


def _split_pages(data):
    pages, at = [], 0
    while at < len(data):
        assert data[at:at + 4] == b"OggS"
        nseg = data[at + 26]
        ln = 27 + nseg + sum(data[at + 27: at + 27 + nseg])
        pages.append(data[at: at + ln])
        at += ln
    return pages


def test_chained_stream_headers_take_the_next_two_packets(ctx, oracle):
    """inside_ogg.rs:124-137: in front of a chained stream the reference reads the comment and the setup header with
    read_packet_expected, i.e. the next two packets whatever their serial -- unlike read_headers at the start of the
    data (:30-47), which skips other streams' packets.  A foreign packet between the ident and the comment header of the
    second stream is therefore a bad header, not something to skip."""
    a = build_stream(211, 2, False, 4)
    b = build_stream(212, 1, False, 4)
    want_a, _ = oracle_pcm(oracle, a[0], a[2])
    want_b, _ = oracle_pcm(oracle, b[0], b[2])
    sa = vp.ogg_stream(11, [a[0].ident_packet(), a[0].comment_packet(), a[0].setup_packet()], a[1], page_granules(want_a, 2, 0), 2)
    pb = _split_pages(vp.ogg_stream(22, [b[0].ident_packet(), b[0].comment_packet(), b[0].setup_packet()], b[1],
                                    page_granules(want_b, 2, 0), 2))
    foreign = vp.ogg_page(33, 0, 0, [(b"not a vorbis header", True)], bos=True)
    # the same foreign page in front of the FIRST stream's comment header is skipped (read_headers)
    pa = _split_pages(sa)
    rd = fe.OggStreamReader(ctx, pa[0] + foreign + b"".join(pa[1:]))
    for w in want_a:
        assert bits_equal(np.array(rd.read_dec_packet_f32()).reshape(2, -1), w)
    rd.close()
    # ... but not in front of the chained stream's
    rd = fe.OggStreamReader(ctx, sa + pb[0] + foreign + b"".join(pb[1:]))
    for w in want_a:
        assert bits_equal(np.array(rd.read_dec_packet_f32()).reshape(2, -1), w)
    with pytest.raises(fe.HeaderReadError):
        rd.read_dec_packet_f32()
    rd.close()


def test_chained_streams_reset_the_decoder(ctx, oracle):
    """inside_ogg.rs:118-141: a new logical stream (other serial, bos page) brings new headers and a fresh
    PreviousWindowRight; its first audio packet is decoded and dropped, reading continues with the second."""
    a = build_stream(201, 2, False, 6)
    b = build_stream(202, 1, False, 7)
    want_a, _ = oracle_pcm(oracle, a[0], a[2])
    want_b, _ = oracle_pcm(oracle, b[0], b[2])
    data = (vp.ogg_stream(11, [a[0].ident_packet(), a[0].comment_packet(), a[0].setup_packet()], a[1], page_granules(want_a, 2, 0), 2) +
            vp.ogg_stream(22, [b[0].ident_packet(), b[0].comment_packet(), b[0].setup_packet()], b[1], page_granules(want_b, 2, 0), 2))
    rd = fe.OggStreamReader(ctx, data)
    for w in want_a:
        got = rd.read_dec_packet_f32()
        assert bits_equal(np.array(got).reshape(2, -1), w)
    got = rd.read_dec_packet_f32()                       # first packet handed out from the second stream: its packet 1
    assert rd.headers.audio_channels == 1
    assert bits_equal(np.array(got).reshape(1, -1), want_b[1])
    for w in want_b[2:]:
        got = rd.read_dec_packet_f32()
        assert bits_equal(np.array(got).reshape(1, -1), w)
    assert rd.read_dec_packet_f32() is None
    rd.close()


@pytest.mark.parametrize("memory", [cabi.MEM_HOST, cabi.MEM_DEVICE])
def test_batched_residue_entry_from_real_bitstreams(ctx, oracle, memory):
    """Many streams sharing one setup: the host front half decodes every packet's floors and residue,
    one lwb_decode_chains call (residue entry) synthesises all of them; bit-identical to the oracle and
    to the per-packet reader."""
    rng = np.random.default_rng(301)
    channels, S, P = 2, 9, 10
    spec = vp.StreamSpec(rng, channels=channels)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    su = hdr.make_setup(ctx)
    streams, wants = [], []
    for s in range(S):
        seq = consistent_modes(spec, rng, P, p_short=0.25)
        infos, pkts = [], []
        for mode, prev, nxt in seq:
            pk, info = spec.audio_packet(mode, prev, nxt)
            pkts.append(pk)
            infos.append(info)
        w, _ = oracle_pcm(oracle, spec, infos)
        streams.append((pkts, infos))
        wants.append(np.concatenate(w, axis=1))
    coeffs, kinds, ys, chains = [], [], [], []
    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    coeff_off = out_off = 0
    for s, (pkts, infos) in enumerate(streams):
        dps = [hdr.decode_packet(pk) for pk in pkts]
        for dp in dps:
            k, y, d = dp.pack()
            assert d is None
            kinds.append(k)
            ys.append(y)
            coeffs.append(dp.residue.ravel())
        n = wants[s].shape[1]
        chains.append(L.ChainSpec(pwrs[s], np.array([dp.mode_number for dp in dps], np.uint8),
                                  np.array([dp.prev_window_flag for dp in dps], np.uint8),
                                  np.array([dp.next_window_flag for dp in dps], np.uint8),
                                  coeff_offset=coeff_off, packet_index=s * P, out_offset=out_off, out_stride=n))
        coeff_off += sum(dp.residue.size for dp in dps)
        out_off += n * channels
    coeffs, kinds, ys = np.concatenate(coeffs), np.concatenate(kinds), np.concatenate(ys)
    pcm = np.zeros(out_off, np.float32)
    if memory == cabi.MEM_HOST:
        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, memory, coeffs, pcm, cabi.OUT_F32_PLANAR, floor_kind=kinds, floor1_y=ys)
    else:
        d_in, d_out = ctx.device_alloc(coeffs.nbytes), ctx.device_alloc(pcm.nbytes)
        ctx.h2d(d_in, coeffs)
        L.decode_chains(ctx, chains, cabi.ENTRY_RESIDUE, memory, d_in, d_out, cabi.OUT_F32_PLANAR, floor_kind=kinds, floor1_y=ys)
        ctx.synchronize()
        ctx.d2h(pcm, d_out)
        ctx.device_free(d_in)
        ctx.device_free(d_out)
    pos = 0
    for s in range(S):
        n = wants[s].shape[1]
        assert chains[s].status == 0 and chains[s].n_samples == n, s
        got = pcm[pos: pos + n * channels].reshape(channels, n)
        assert bits_equal(got, wants[s]), (s, mismatch_report(got, wants[s]))
        pos += n * channels


def test_stream_batcher_parallel_entropy_decode_one_synthesis_call(ctx, oracle):
    """lwf_batcher: 24 streams (6 distinct bitstreams x 4) decoded by 4 host threads + one batched
    synthesis call; every stream bit-identical to the oracle; a corrupt packet ends only its own stream."""
    rng = np.random.default_rng(401)
    channels, P = 2, 9
    spec = vp.StreamSpec(rng, channels=channels, floor0=True)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    su = hdr.make_setup(ctx)
    distinct = []
    for d in range(6):
        seq = consistent_modes(spec, rng, P, p_short=0.3)
        pkts, infos = [], []
        for mode, prev, nxt in seq:
            pk, info = spec.audio_packet(mode, prev, nxt)
            pkts.append(pk)
            infos.append(info)
        w, _ = oracle_pcm(oracle, spec, infos)
        distinct.append((pkts, w))
    S = 24
    jobs, pwrs = [], []
    for s in range(S):
        pw = L.PreviousWindowRight(su)
        pwrs.append(pw)
        jobs.append((pw, list(distinct[s % 6][0])))
    # stream 5: its 4th packet claims to be a header packet
    jobs[5] = (jobs[5][0], jobs[5][1][:3] + [b"\x01bad"] + jobs[5][1][4:])
    stride = P * 1024
    pcm = np.full(S * channels * stride, np.nan, np.float32)
    bt = fe.StreamBatcher(ctx, hdr, threads=4)
    res = bt.decode(jobs, pcm, stride)
    for s in range(S):
        n_samples, done, status = res[s]
        w = distinct[s % 6][1]
        if s == 5:
            assert done == 3 and status == fe.ERR_AUDIO_IS_HEADER
            w = w[:3]
        else:
            assert done == P and status == 0
        want = np.concatenate(w, axis=1)
        assert n_samples == want.shape[1]
        got = pcm[s * channels * stride:(s + 1) * channels * stride].reshape(channels, stride)[:, :n_samples]
        assert bits_equal(got, want), (s, mismatch_report(got, want))
    assert bt.entropy_seconds > 0 and bt.synthesis_seconds > 0
    bt.close()


def test_hostile_but_parseable_streams_do_not_break_the_gpu_path(ctx, oracle):
    """Mutated setup headers / audio packets that still parse (re-paged with valid CRCs) go through the
    whole reader: every call must end in PCM or a reference-style error, and the context must stay usable
    (checked with a bit-exact decode afterwards; run under compute-sanitizer in profiles/)."""
    rng = np.random.default_rng(501)
    spec, packets, infos = build_stream(77, 2, True, 8)
    want, _ = oracle_pcm(oracle, spec, infos)
    hdrs = [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()]

    def mutate(b):
        b = bytearray(b)
        for _ in range(int(rng.integers(1, 6))):
            b[int(rng.integers(8, len(b)))] ^= 1 << int(rng.integers(0, 8))
        return bytes(b)

    outcomes = {"ok": 0, "header": 0, "audio": 0, "ogg": 0}
    for it in range(60):
        h = list(hdrs)
        pk = list(packets)
        if it % 3 == 0:
            h[2] = mutate(h[2])
        else:
            pk = [mutate(p) if len(p) > 9 and rng.random() < 0.7 else p for p in pk]
        data = vp.ogg_stream(5, h, pk, page_granules(want, 3, 0), packets_per_page=3)
        try:
            rd = fe.OggStreamReader(ctx, data)
        except fe.HeaderReadError:
            outcomes["header"] += 1
            continue
        except L.AudioReadError:
            outcomes["header"] += 1          # the device-side setup refused the (parseable) header
            continue
        try:
            while True:
                got = rd.read_dec_packet_f32()
                if got is None:
                    break
            outcomes["ok"] += 1
        except L.AudioReadError:
            outcomes["audio"] += 1
        except fe.OggReadError:
            outcomes["ogg"] += 1
        finally:
            rd.close()
        ctx.synchronize()
    assert outcomes["ok"] > 10, outcomes
    # the context still decodes bit-exactly
    data = vp.ogg_stream(5, hdrs, packets, page_granules(want, 3, 0), packets_per_page=3)
    rd = fe.OggStreamReader(ctx, data)
    for w in want:
        got = rd.read_dec_packet_f32()
        assert bits_equal(np.array(got).reshape(2, -1), w)
    rd.close()


def _oracle_stream(oracle, spec):
    floors = [(f.multiplier, f.x_list) if isinstance(f, vp.Floor1) else (1, [0, 128]) for f in spec.floors]
    mappings = [{"coupling": m["coupling"], "floor_of_channel": [m["floors"][m["mux"][c]] for c in range(spec.channels)]}
                for m in spec.mappings]
    return RefStream(oracle, spec.channels, spec.bs0, spec.bs1, spec.modes, mappings, floors)


def _oracle_packet(ref, spec, info):
    fl_exp, res = spec.expected(info)
    n2 = info["n"] // 2
    fl = []
    for f in fl_exp:
        if f is None:
            fl.append(None)
        elif f[0] == "one":
            fl.append(list(f[1]))
        else:
            fl.append(floor0_expected(f[3], f[1], f[2], info["blockflag"], n2, spec.bs0, spec.bs1))
    rc, pcm = ref.packet(info["mode"], info["prev"], info["next"], res, fl)
    assert rc == 0
    return pcm


def _sample_count(spec, info):
    """audio::get_decoded_sample_count (audio.rs:874-909): right_win_start - left_win_start, whatever the state."""
    n, n0 = info["n"], 1 << spec.bs0
    lng = bool(info["blockflag"])
    ls = 0 if (not lng or info["prev"]) else (n - n0) // 4
    rs = n // 2 if (not lng or info["next"]) else (3 * n - n0) // 4
    return rs - ls


class _ReaderModel:
    """The reference's OggStreamReader state machine (inside_ogg.rs:107-313) over the packer's record of a stream,
    with the oracle as the decoder: what read_dec_packet_generic / skip_samples_linear / seek_absgp_pg must return."""

    def __init__(self, oracle, spec, infos, granules, per_page):
        self.spec, self.infos, self.gran, self.pp = spec, infos, granules, per_page
        self.ref = _oracle_stream(oracle, spec)
        self.idx, self.absgp = 0, None

    def _page(self, i):
        return i // self.pp

    def _dec(self, i):
        pcm = _oracle_packet(self.ref, self.spec, self.infos[i])
        last_in_stream = i == len(self.infos) - 1
        last_in_page = (i + 1) % self.pp == 0 or last_in_stream
        n = pcm.shape[1]
        if self.absgp is not None and last_in_stream:
            n = min(n, max(self.gran[self._page(i)] - self.absgp, 0))
        if last_in_page:
            self.absgp = self.gran[self._page(i)]
        elif self.absgp is not None:
            self.absgp += n
        return pcm[:, :n]

    def read(self):
        if self.idx >= len(self.infos):
            return None
        self.idx += 1
        return self._dec(self.idx - 1)

    def skip(self, to_skip):
        last = None
        while True:
            if self.idx >= len(self.infos):
                return None, to_skip
            i = self.idx
            self.idx += 1
            cnt = _sample_count(self.spec, self.infos[i])
            if self.absgp is not None and i == len(self.infos) - 1:
                last = None
                cnt = min(cnt, max(self.gran[self._page(i)] - self.absgp, 0))
            if to_skip < cnt:
                if last is not None:
                    self.ref.pwr.reset()
                    _oracle_packet(self.ref, self.spec, self.infos[last])
                return self._dec(i), to_skip
            to_skip -= cnt
            if self.absgp is not None:
                self.absgp += cnt
            last = i

    def seek(self, goal):
        pages = [j for j in range(len(self.gran)) if self.gran[j] <= goal]
        self.idx = (pages[-1] if pages else 0) * self.pp
        self.absgp = None
        self.ref.pwr.reset()


@pytest.mark.parametrize("seed,channels", [(401, 2), (402, 1), (403, 6)])
def test_skip_samples_linear_and_seek_absgp_pg(ctx, oracle, seed, channels):
    """inside_ogg.rs:244-283 and :307-313 through the GPU reader: packets are skipped by their sample counts, the
    packet before the target is decoded on a fresh PreviousWindowRight and dropped, the target packet comes back
    with the leftover count; a page-granular seek lands at or before the goal, clears the granule position and the
    overlap state.  Every returned packet, leftover count and get_last_absgp() value is compared with a model of the
    reference's state machine that decodes with the oracle."""
    n_packets, per_page = 23, 3
    spec, packets, infos = build_stream(seed, channels, False, n_packets)
    want, _ = oracle_pcm(oracle, spec, infos)
    gran = page_granules(want, per_page, 11)
    data = vp.ogg_stream(0x77, [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()], packets, gran, packets_per_page=per_page)
    rd = fe.OggStreamReader(ctx, data)
    model = _ReaderModel(oracle, spec, infos, gran, per_page)

    def same(got, w, what):
        if w is None:
            assert got is None, what
            return
        assert got is not None and len(got) == channels and all(len(g) == w.shape[1] for g in got), (what, w.shape)
        assert bits_equal(np.array(got).reshape(channels, -1), w), (what, mismatch_report(np.array(got).reshape(channels, -1), w))

    for i in range(2):
        same(rd.read_dec_packet_f32(), model.read(), ("read", i))
    # a skip that stays inside the next packet, one that crosses several packets and a page, one that lands in the
    # truncated last packet, one that runs off the end of the stream
    for to_skip in (3, 2500, 40, 10 ** 7):
        got, left = rd.skip_samples_linear(to_skip)
        w, wleft = model.skip(to_skip)
        same(got, w, ("skip", to_skip))
        assert left == wleft and rd.get_last_absgp() == model.absgp, (to_skip, left, wleft, rd.get_last_absgp(), model.absgp)
        if w is not None and model.idx < n_packets:
            same(rd.read_dec_packet_f32(), model.read(), ("after skip", to_skip))
    assert rd.read_dec_packet_f32() is None
    # seeks: into the middle, before the first page's end, beyond the end, and back to the middle
    for goal in (gran[3] + 5, 0, gran[-1] + 1000, gran[2]):
        rd.seek_absgp_pg(goal)
        model.seek(goal)
        assert rd.get_last_absgp() is None
        for k in range(5):
            w = model.read()
            same(rd.read_dec_packet_f32(), w, ("after seek", goal, k))
            assert rd.get_last_absgp() == model.absgp, (goal, k)
            if w is None:
                break
    rd.close()


@pytest.mark.parametrize("channels,rtype,memory,floor_mem,fmt,seed", [
    (2, 1, cabi.MEM_HOST, cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 501),
    (2, 0, cabi.MEM_DEVICE, cabi.MEM_DEVICE, cabi.OUT_F32_PLANAR, 502),
    (2, 2, cabi.MEM_HOST, cabi.MEM_HOST, cabi.OUT_I16_PLANAR, 503),
    (6, None, cabi.MEM_DEVICE, cabi.MEM_HOST, cabi.OUT_F32_PLANAR, 504),
    (1, None, cabi.MEM_HOST, cabi.MEM_HOST, cabi.OUT_I16_INTERLEAVED, 505),
    (3, 2, cabi.MEM_DEVICE, cabi.MEM_DEVICE, cabi.OUT_I16_PLANAR, 506)])
def test_vq_entry_accumulates_the_residue_on_the_device(ctx, oracle, channels, rtype, memory, floor_mem, fmt, seed):
    """LWB_ENTRY_VQ (SURVEY.md 8f rank 2; audio.rs:587-717): no dense coefficients cross the boundary -- the front half
    hands over VQ records, the device accumulates the residue vectors pass by pass in shared memory and runs the rest
    of the path.  Every stream is bit-identical to the oracle's decode of what the packer encoded, and the whole PCM
    arena is identical to the dense residue entry on the same packets -- including streams whose packets were cut at
    arbitrary bytes (the residue decode keeps what it had, audio.rs:640-716)."""
    rng = np.random.default_rng(seed)
    S, P = 7, 9
    spec = vp.StreamSpec(rng, channels=channels, residue_types=[rtype] if rtype is not None else None)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    assert hdr.vq_capable()
    su = hdr.make_setup(ctx)
    streams, wants = [], []
    for s in range(S):
        seq = consistent_modes(spec, rng, P, p_short=0.3 if s % 2 else 0.0)
        infos, pkts = [], []
        for mode, prev, nxt in seq:
            pk, info = spec.audio_packet(mode, prev, nxt, p_unused=0.1)
            if s >= S - 2:                               # the last two streams carry truncated packets
                lo = min((info["header_bits"] + 7) // 8 + 1, len(pk))
                pk = pk[:int(rng.integers(lo, len(pk) + 1))]
            pkts.append(pk)
            infos.append(info)
        streams.append((pkts, infos))
        wants.append(np.concatenate(oracle_pcm(oracle, spec, infos)[0], axis=1) if s < S - 2 else None)
    f32 = fmt == cabi.OUT_F32_PLANAR
    dt = np.float32 if f32 else np.int16
    planar = fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR)
    outs = {}
    for entry in (cabi.ENTRY_VQ, cabi.ENTRY_RESIDUE):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        coeffs, kinds, ys, runs, ents, roffs, eoffs, chains = [], [], [], [], [], [0], [0], []
        coeff_off = out_off = 0
        for s, (pkts, infos) in enumerate(streams):
            modes, prevs, nexts, n_out, size = [], [], [], 0, 0
            for pk in pkts:
                dense = hdr.decode_packet(pk)
                dp, rr, ee = hdr.decode_packet_vq(pk)
                k, y, d = dense.pack()
                assert d is None
                kinds.append(k)
                ys.append(y)
                coeffs.append(dense.residue.ravel())
                runs.append(rr)
                ents.append(ee)
                roffs.append(roffs[-1] + len(rr))
                eoffs.append(eoffs[-1] + len(ee))
                modes.append(dp.mode_number); prevs.append(dp.prev_window_flag); nexts.append(dp.next_window_flag)
                size += dense.residue.size
            stride = P * (1 << spec.bs1) // 2
            chains.append(L.ChainSpec(pwrs[s], np.array(modes, np.uint8), np.array(prevs, np.uint8), np.array(nexts, np.uint8),
                                      coeff_offset=coeff_off, packet_index=s * P, out_offset=out_off, out_stride=stride if planar else 0))
            coeff_off += size
            out_off += stride * channels
        coeffs, kinds, ys = np.concatenate(coeffs), np.concatenate(kinds), np.concatenate(ys)
        runs = np.concatenate(runs) if roffs[-1] else np.zeros(1, fe.VQ_RUN_DTYPE)
        ents = np.concatenate(ents) if eoffs[-1] else np.zeros(1, np.uint16)
        roffs, eoffs = np.array(roffs, np.uint64), np.array(eoffs, np.uint64)
        pcm = np.zeros(out_off, dt)
        kw = dict(floor_kind=kinds, floor1_y=ys)
        frees = []
        if floor_mem == cabi.MEM_DEVICE:
            def dev(arr):
                d = ctx.device_alloc(max(arr.nbytes, 16))
                ctx.h2d(d, arr)
                frees.append(d)
                return d
            kw = dict(floor_kind=dev(kinds), floor1_y=dev(ys), floor_memory=cabi.MEM_DEVICE)
            if entry == cabi.ENTRY_VQ:
                kw["vq"] = (dev(runs), dev(roffs), dev(ents), dev(eoffs))
        elif entry == cabi.ENTRY_VQ:
            kw["vq"] = (runs, roffs, ents, eoffs)
        if memory == cabi.MEM_HOST:
            L.decode_chains(ctx, chains, entry, memory, None if entry == cabi.ENTRY_VQ else coeffs, pcm, fmt, **kw)
        else:
            d_out = ctx.device_alloc(pcm.nbytes)
            ctx.h2d(d_out, pcm)
            d_in = None
            if entry == cabi.ENTRY_RESIDUE:
                d_in = ctx.device_alloc(coeffs.nbytes)
                ctx.h2d(d_in, coeffs)
            L.decode_chains(ctx, chains, entry, memory, d_in, d_out, fmt, **kw)
            ctx.synchronize()
            ctx.d2h(pcm, d_out)
            ctx.device_free(d_out)
            if d_in:
                ctx.device_free(d_in)
        for d in frees:
            ctx.device_free(d)
        outs[entry] = (pcm, [(c.status, c.n_samples) for c in chains], [p.data() for p in pwrs])
        for p in pwrs:
            p.close()
    pcm, res, states = outs[cabi.ENTRY_VQ]
    stride = P * (1 << spec.bs1) // 2
    for s in range(S - 2):
        n = wants[s].shape[1]
        assert res[s] == (0, n), (s, res[s], n)
        blk = pcm[s * stride * channels:(s + 1) * stride * channels]
        got = blk.reshape(channels, stride)[:, :n] if planar else blk[: n * channels].reshape(n, channels).T
        if f32:
            assert bits_equal(got, wants[s]), (s, mismatch_report(got, wants[s]))
        else:
            assert np.array_equal(got, oracle.quantise_i16(wants[s])), s
    assert res == outs[cabi.ENTRY_RESIDUE][1]
    assert np.array_equal(pcm.view(np.uint8), outs[cabi.ENTRY_RESIDUE][0].view(np.uint8)), "VQ entry and dense residue entry differ"
    for a, b in zip(states, outs[cabi.ENTRY_RESIDUE][2]):
        assert (a is None) == (b is None) and (a is None or bits_equal(a, b))


@pytest.mark.filterwarnings("ignore:overflow encountered:RuntimeWarning")      # (the packer's own f32 sums)
def test_vq_entry_sums_that_overflow_to_inf(ctx, oracle):
    """VQ books whose values are finite but within a factor of two of FLT_MAX (minimum +-2^127, delta 2^120): two passes
    over a bin overflow the f32 sum to +-inf (and +inf + -inf to NaN) in d_vq_accumulate, as the reference's `+=` does
    (audio.rs:595, :611).  Uniform long stereo packets, so k_floor1_segments + k_prologue_fused<VQ> form the spectrum
    and k_long transforms it; bit-identical to the oracle and to the dense residue entry of the same packets."""
    rng = np.random.default_rng(531)
    S, P, channels = 4, 6, 2
    spec = vp.StreamSpec(rng, channels=channels, residue_types=[1], cascade_p=1.0)
    for i in spec.vq_ids:
        spec.books[i].set_values(2.0 ** 127 * (1 if i % 2 else -1), 2.0 ** 120, False)
    assert all(np.all(np.isfinite(spec.books[i].vq)) for i in spec.vq_ids)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    assert hdr.vq_capable()
    su = hdr.make_setup(ctx)
    streams, wants, overflowed = [], [], False
    for s in range(S):
        pkts, infos = [], []
        for mode, prev, nxt in consistent_modes(spec, rng, P, p_short=0.0):
            pk, info = spec.audio_packet(mode, prev, nxt, p_unused=0.1)
            pkts.append(pk)
            infos.append(info)
            overflowed |= bool(np.any(np.isinf(spec.expected(info)[1])))
        streams.append(pkts)
        wants.append(np.concatenate(oracle_pcm(oracle, spec, infos)[0], axis=1))
    assert overflowed, "test should overflow a residue sum to inf"
    assert all(not np.all(np.isfinite(w)) for w in wants[:2]), "test should carry inf / NaN to the output"
    stride = P * (1 << spec.bs1) // 2
    outs = {}
    for entry in (cabi.ENTRY_VQ, cabi.ENTRY_RESIDUE):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        coeffs, kinds, ys, runs, ents, roffs, eoffs, chains = [], [], [], [], [], [0], [0], []
        for s, pkts in enumerate(streams):
            modes, prevs, nexts = [], [], []
            for pk in pkts:
                dense = hdr.decode_packet(pk)
                dp, rr, ee = hdr.decode_packet_vq(pk)
                k, y, _ = dense.pack()
                kinds.append(k)
                ys.append(y)
                coeffs.append(dense.residue.ravel())
                runs.append(rr)
                ents.append(ee)
                roffs.append(roffs[-1] + len(rr))
                eoffs.append(eoffs[-1] + len(ee))
                modes.append(dp.mode_number); prevs.append(dp.prev_window_flag); nexts.append(dp.next_window_flag)
            chains.append(L.ChainSpec(pwrs[s], np.array(modes, np.uint8), np.array(prevs, np.uint8), np.array(nexts, np.uint8),
                                      coeff_offset=s * channels * stride, packet_index=s * P,
                                      out_offset=s * channels * stride, out_stride=stride))
        kw = dict(floor_kind=np.concatenate(kinds), floor1_y=np.concatenate(ys))
        if entry == cabi.ENTRY_VQ:
            kw["vq"] = (np.concatenate(runs), np.array(roffs, np.uint64), np.concatenate(ents), np.array(eoffs, np.uint64))
        pcm = np.zeros(S * channels * stride, np.float32)
        with expect_kernels(ctx, ran={"k_floor1_segments": 1, "k_prologue_fused": 1, "k_long": 1},
                            not_ran=ALL_KERNELS - FRONT - {"k_long"}):
            L.decode_chains(ctx, chains, entry, cabi.MEM_HOST, None if entry == cabi.ENTRY_VQ else np.concatenate(coeffs), pcm,
                            cabi.OUT_F32_PLANAR, **kw)
        outs[entry] = (pcm, [p.data() for p in pwrs])
        for s in range(S):
            n = wants[s].shape[1]
            assert chains[s].status == 0 and chains[s].n_samples == n, (entry, s)
            got = pcm[s * channels * stride:(s + 1) * channels * stride].reshape(channels, stride)[:, :n]
            assert bits_equal(got, wants[s]), (entry, s, mismatch_report(got, wants[s]))
        for p in pwrs:
            p.close()
    assert np.array_equal(outs[cabi.ENTRY_VQ][0].view(np.uint8), outs[cabi.ENTRY_RESIDUE][0].view(np.uint8))
    for a, b in zip(outs[cabi.ENTRY_VQ][1], outs[cabi.ENTRY_RESIDUE][1]):
        assert bits_equal(a, b)


def test_stream_batcher_vq_entry(ctx, oracle):
    """lwf_batcher with LWB_ENTRY_VQ: the host threads entropy-decode to VQ records, one batched call accumulates and
    synthesises; bit-identical to the oracle and to the dense batcher."""
    rng = np.random.default_rng(521)
    channels, P, S = 2, 10, 16
    spec = vp.StreamSpec(rng, channels=channels)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    su = hdr.make_setup(ctx)
    distinct = []
    for d in range(4):
        seq = consistent_modes(spec, rng, P, p_short=0.2)
        pkts, infos = [], []
        for mode, prev, nxt in seq:
            pk, info = spec.audio_packet(mode, prev, nxt)
            pkts.append(pk)
            infos.append(info)
        distinct.append((pkts, np.concatenate(oracle_pcm(oracle, spec, infos)[0], axis=1)))
    stride = P * (1 << spec.bs1) // 2
    results = {}
    for entry in (cabi.ENTRY_VQ, cabi.ENTRY_RESIDUE):
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        jobs = [(pwrs[s], list(distinct[s % 4][0])) for s in range(S)]
        pcm = np.zeros(S * channels * stride, np.float32)
        bt = fe.StreamBatcher(ctx, hdr, threads=3, entry=entry)
        res = bt.decode(jobs, pcm, stride)
        bt.close()
        results[entry] = pcm
        for s in range(S):
            w = distinct[s % 4][1]
            assert res[s] == (w.shape[1], P, 0), (entry, s, res[s])
            got = pcm[s * channels * stride:(s + 1) * channels * stride].reshape(channels, stride)[:, : w.shape[1]]
            assert bits_equal(got, w), (entry, s, mismatch_report(got, w))
        for p in pwrs:
            p.close()

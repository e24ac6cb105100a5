"""OggStreamReaders (lwf_readers) on the GPU: many Ogg Vorbis files of the packer (tests/vorbis_packer.py) read in batched
calls of varied max_packets (1, 3, all), two calls queued before the first is waited for, in every sample format and
layout, into host and device PCM.  Every job must return exactly what a single OggStreamReader returns reading the same
bytes packet by packet -- PCM, packet sample counts, status, end, chained-stream stops, absgp and headers -- and write
nothing outside its samples; the single reader is in turn held to the CPU oracle fed with the packer's record."""
import ctypes as C

import numpy as np
import pytest

import lewton_b200 as L
import vorbis_packer as vp
from helpers import FUSED, GENERIC, assert_contained, bits_equal, expect_kernels, fill_guard, launches_are_attributed
from lewton_b200 import frontend as fe
from lewton_b200.api import sample_format
from test_frontend_gpu import consistent_modes, oracle_pcm

launches_are_attributed  # (autouse)

pytestmark = pytest.mark.gpu

FORMATS = [(s, itl) for s in ("f32", "i16", "f16") for itl in (False, True)]
ALL = 20                                   # more packets than any stream of these files has
SCHEDULE = (1, 3, ALL)


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ---- files ---------------------------------------------------------------------------------------
def stream(seed, channels, bs0=8, bs1=11, floor0=False, n_packets=10, n_modes=None):
    rng = np.random.default_rng(seed)
    spec = vp.StreamSpec(rng, channels=channels, bs0=bs0, bs1=bs1, floor0=floor0, n_modes=n_modes)
    packets, infos = [], []
    for mode, prev, nxt in consistent_modes(spec, rng, n_packets):
        pk, info = spec.audio_packet(mode, prev, nxt)
        packets.append(pk)
        infos.append(info)
    return spec, packets, infos


def headers_of(spec):
    return [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()]


def header_pages(serial, spec):
    return vp.ogg_stream(serial, headers_of(spec), [], [])


def audio_pages(serial, packets, granule_after, seq0=2, per_page=3, segs_per_page=None):
    """Pages of the audio packets: per_page packets per page, or (segs_per_page) at most that many lacing values per
    page with packets continued across pages.  A page's granule position is granule_after[k] of the last packet k that
    ends on it (-1 if none does); the last page ends the stream."""
    pages, seq = [], seq0
    if segs_per_page is None:
        for i in range(0, len(packets), per_page):
            grp = packets[i: i + per_page]
            pages.append(vp.ogg_page(serial, seq, granule_after[i + len(grp) - 1], [(p, True) for p in grp],
                                     eos=i + per_page >= len(packets)))
            seq += 1
        return pages
    # lacing values of every packet, then cut into pages
    segs = []
    for k, p in enumerate(packets):
        full, rem = divmod(len(p), 255)
        for s in range(full):
            segs.append((k, p[s * 255:(s + 1) * 255], False))
        segs.append((k, p[full * 255:], True))
    continued = False
    for i in range(0, len(segs), segs_per_page):
        grp = segs[i: i + segs_per_page]
        ends = [k for k, _, last in grp if last]
        gran = granule_after[ends[-1]] if ends else (1 << 64) - 1
        pieces = []
        for k, data, last in grp:
            if pieces and pieces[-1][2] == k and not pieces[-1][1]:
                pieces[-1] = (pieces[-1][0] + data, last, k)
            else:
                pieces.append((data, last, k))
        pages.append(vp.ogg_page(serial, seq, gran, [(d, last) for d, last, _ in pieces], continued=continued,
                                 eos=i + segs_per_page >= len(segs)))
        continued = not grp[-1][2]
        seq += 1
    return pages


def granules(want, cut=0):
    """absgp after each packet: the samples decoded up to it; the last one claims `cut` fewer (cut < 0: more)."""
    out = list(np.cumsum([w.shape[1] for w in want]))
    out[-1] -= cut
    return [int(g) for g in out]


def clean_file(oracle, seed, channels, bs0=8, bs1=11, floor0=False, n_packets=10, cut=0, per_page=3, segs_per_page=None,
               serial=0x51):
    spec, packets, infos = stream(seed, channels, bs0, bs1, floor0, n_packets)
    want, _ = oracle_pcm(oracle, spec, infos)
    pages = audio_pages(serial, packets, granules(want, cut), per_page=per_page, segs_per_page=segs_per_page)
    return header_pages(serial, spec) + b"".join(pages), want


def foreign_file(oracle):
    """A stereo stream with a foreign logical stream multiplexed in: its first page between the ident and the comment
    header (skipped by read_headers), and one of its pages behind every audio page (skipped by read_next_audio_packet)."""
    spec, packets, infos = stream(401, 2, n_packets=9)
    want, _ = oracle_pcm(oracle, spec, infos)
    hp = _split_pages(header_pages(7, spec))
    data = hp[0] + vp.ogg_page(99, 0, 0, [(b"foreign header", True)], bos=True) + b"".join(hp[1:])
    for k, p in enumerate(audio_pages(7, packets, granules(want, 5), per_page=2)):
        data += p + vp.ogg_page(99, k + 1, 1000 * k, [(b"foreign %d" % k, True), (bytes(300), True)])
    return data, want


def chained_file(oracle):
    """Three logical streams one after the other: stereo 256/2048, mono 512/4096, six channels 1024/1024."""
    data, want = b"", []
    for serial, (seed, ch, bs0, bs1, n, cut) in zip((11, 22, 33), [(501, 2, 8, 11, 7, 20), (502, 1, 9, 12, 5, 0),
                                                                    (503, 6, 10, 10, 6, 9)]):
        spec, packets, infos = stream(seed, ch, bs0, bs1, False, n)
        w, _ = oracle_pcm(oracle, spec, infos)
        data += header_pages(serial, spec) + b"".join(audio_pages(serial, packets, granules(w, cut), per_page=2))
        want.append(w)
    return data, want


def error_file():
    """Stereo, three modes (so mode number 3 is out of range), with a packet of no bytes, a bad mode number, a header
    packet among the audio packets and a packet cut after its first byte between good ones."""
    spec, packets, _ = stream(601, 2, n_packets=9, n_modes=3)
    bad_mode = bytes([0b110]) + bytes(40)
    packets = (packets[:2] + [b""] + packets[2:4] + [bad_mode] + packets[4:6] + [b"\x01vorbis"] + [packets[6][:1]] +
               packets[6:])
    gran = [1 << 40] * len(packets)
    return header_pages(5, spec) + b"".join(audio_pages(5, packets, gran, per_page=3)), None


def headers_only_file():
    spec, _, _ = stream(701, 2, n_packets=1)
    return header_pages(3, spec), None


def _split_pages(data):
    pages, at = [], 0
    while at < len(data):
        nseg = data[at + 26]
        ln = 27 + nseg + sum(data[at + 27: at + 27 + nseg])
        pages.append(data[at: at + ln])
        at += ln
    return pages


@pytest.fixture(scope="module")
def corpus(oracle):
    files = {
        "stereo_256_2048_cut": clean_file(oracle, 301, 2, cut=37, n_packets=14),
        "mono_1024_1024_floor0_above": clean_file(oracle, 302, 1, 10, 10, True, n_packets=11, cut=-300, per_page=4),
        "six_512_4096_spanning": clean_file(oracle, 303, 6, 9, 12, n_packets=9, cut=11, segs_per_page=5),
        "ten_256_2048": clean_file(oracle, 304, 10, n_packets=7, per_page=2),
        "stereo_floor0_mid_page": clean_file(oracle, 305, 2, floor0=True, n_packets=8, cut=23, per_page=3),
        "foreign": foreign_file(oracle),
        "chained": chained_file(oracle),
        "errors": error_file(),
        "headers_only": headers_only_file(),
    }
    return files


# ---- the single reader, packet by packet ---------------------------------------------------------
def single_trace(ctx, data, sample, interleaved):
    """Every call of lwf_reader_read_dec_packet until the end: ("pkt", [channels][n] PCM, absgp after, channels) |
    ("err", code, absgp after, channels) | ("end", None, absgp after, channels).  An Ogg error repeats: it ends the
    trace."""
    fmt, dt = sample_format(sample, interleaved)
    lib = fe.lib()
    rd = fe.OggStreamReader(ctx, data)
    cap = 16 * 8192
    buf = np.zeros(cap, dt)
    out = []
    for _ in range(200):
        n = C.c_size_t()
        rc = lib.lwf_reader_read_dec_packet(rd._h, fmt, buf.ctypes.data, cap, C.byref(n))
        ch = fe.Headers(None, None, None, _handle=lib.lwf_reader_headers(rd._h)).audio_channels
        absgp = rd.get_last_absgp()
        if rc == fe.ERR_NO_MORE_PACKETS:
            out.append(("end", None, absgp, ch))
            break
        if rc:
            out.append(("err", rc, absgp, ch))
            if rc == fe.ERR_OGG:
                break
            continue
        n = n.value
        if interleaved:
            pcm = buf[: n * ch].reshape(n, ch).T.copy()
        else:
            per = cap // ch
            pcm = np.stack([buf[c * per: c * per + n] for c in range(ch)]) if n else np.zeros((ch, 0), dt)
        out.append(("pkt", pcm, absgp, ch))
    rd.close()
    return out


def same_samples(a, b, sample):
    if a.shape != b.shape:
        return False
    return bits_equal(a, b) if sample == "f32" else bool(np.array_equal(a.view(np.uint16), b.view(np.uint16)))


def test_single_reader_matches_the_oracle(ctx, corpus):
    """The specification the batched readers are held to: the single reader's f32 packets are the oracle's, the first
    packet of the file empty, the first of a chained stream dropped, the last of a stream cut to its granule position."""
    for name, (data, want) in corpus.items():
        if want is None:
            continue
        streams = want if name == "chained" else [want]
        expect = []
        for s, w in enumerate(streams):
            expect += w[1:] if s else w          # a chained stream's first packet is decoded and dropped
        ev = single_trace(ctx, data, "f32", False)
        pk = [e for e in ev if e[0] == "pkt"]
        assert ev[-1][0] == "end" and len(pk) == len(expect), name
        for k, (e, w) in enumerate(zip(pk, expect)):
            n = e[1].shape[1]
            assert n == w.shape[1] or (n < w.shape[1] and (k == len(pk) - 1 or name == "chained")), (name, k, n, w.shape)
            assert bits_equal(e[1], w[:, :n]), (name, k)


# ---- the batched readers -------------------------------------------------------------------------
def _buffer(ctx, memory, n, dt):
    guard = fill_guard(np.empty(n, dt))
    if memory == "host":
        buf = ctx.host_alloc(n, dt)
        buf[...] = guard
        return buf
    import torch
    t = torch.from_numpy(guard.view(np.int16 if dt != np.float32 else np.float32).copy()).cuda()
    return t


def _host(buf, dt):
    if isinstance(buf, np.ndarray):
        return buf
    return buf.cpu().numpy().view(dt)


def read_all(ctx, files, traces, sample, interleaved, memory, schedule=SCHEDULE, threads=4):
    """Reads every file to its end through one OggStreamReaders, two calls in flight, and checks each job against the
    single reader's trace.  Returns the readers object."""
    _, dt = sample_format(sample, interleaved)
    rs = fe.OggStreamReaders(ctx, threads=threads)
    idx = [rs.add(d) for d in files]
    pos = [0] * len(files)
    done = [False] * len(files)
    pending = []

    def check(item):
        t, buf, stride, meta = item
        results = t.wait()
        host = _host(buf, dt)
        spans = []
        for r, (i, maxp, ch_before, absgp, ch_after) in zip(results, meta):
            ev, p = traces[i], pos[i]
            what = "file %d call job %r" % (i, r)
            assert r.reader == idx[i] and r.channels == ch_before, what
            if done[i]:                                # a reader that ended in the call before stays at its end
                assert r.ended and not r.n_packets and not r.status and ev[p][0] == "end", what
                assert absgp == (ev[p - 1][2] if p else None), what
                continue
            s0 = 0
            for k in range(r.n_packets):
                e = ev[p]
                n = int(r.packet_samples[k])
                assert e[0] == "pkt" and e[1].shape == (ch_before, n), (what, k, e[0], e[1] if e[0] != "pkt" else e[1].shape)
                if interleaved:
                    got = host[r.out_offset + s0 * ch_before: r.out_offset + (s0 + n) * ch_before].reshape(n, ch_before).T
                else:
                    got = np.stack([host[r.out_offset + c * stride + s0: r.out_offset + c * stride + s0 + n]
                                    for c in range(ch_before)])
                assert same_samples(got, e[1], sample), (what, k)
                s0 += n
                p += 1
            assert r.n_samples == s0, what
            if r.status:
                assert ev[p][0] == "err" and ev[p][1] == r.status, (what, ev[p][:2])
                p += 1
                if r.status == fe.ERR_OGG:
                    done[i] = True
                assert not r.ended and not r.next_chained, what
            elif r.ended:
                assert ev[p][0] == "end", what
                assert not r.next_chained, what
                done[i] = True
            elif r.next_chained:
                assert ev[p][3] == ch_after, what          # the single reader's next call is in the new stream
            else:
                assert r.n_packets == maxp, what
            assert absgp == (ev[p - 1][2] if p else None), (what, absgp, ev[p - 1][2] if p else None)
            pos[i] = p
            if interleaved:
                spans.append((i, [(r.out_offset, r.n_samples * ch_before)] if r.n_samples else []))
            else:
                spans.append((i, [(r.out_offset + c * stride, r.n_samples) for c in range(ch_before) if r.n_samples]))
        assert_contained(host, spans, "readers call")

    call = 0
    while True:
        # every reader that has not been seen to end joins the call, also while its previous call is still in flight
        jobs = [(i, schedule[(call + i) % len(schedule)]) for i in range(len(files)) if not done[i]]
        if jobs:
            stride = max(1, max(rs.stride(idx[i], m) for i, m in jobs))
            ch = [rs.headers(idx[i]).audio_channels for i, _ in jobs]
            buf = _buffer(ctx, memory, sum(ch) * stride + 64, dt)
            try:
                t = rs.read([(idx[i], m) for i, m in jobs], buf, stride, sample, interleaved)
            except L.AudioReadError as e:
                raise AssertionError("call %d refused: stride %d, jobs (file, max_packets, blocksize_1, trace position) %r" % (
                    call, stride, [(i, m, rs.headers(idx[i]).blocksize_1, pos[i]) for i, m in jobs])) from e
            meta = [(i, m, c, rs.get_last_absgp(idx[i]), rs.headers(idx[i]).audio_channels) for (i, m), c in zip(jobs, ch)]
            pending.append((t, buf, stride, meta))
            call += 1
            assert call < 100, "the readers do not reach the end"
        if len(pending) == 2 or (pending and not jobs):
            check(pending.pop(0))                  # the older of two queued calls
        if not jobs and not pending:
            break
    for i in range(len(files)):
        assert pos[i] == len(traces[i]) - (traces[i][-1][0] == "end"), (i, pos[i], len(traces[i]))
    return rs


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("sample,interleaved", FORMATS)
def test_readers_return_what_the_single_reader_returns(ctx, corpus, sample, interleaved, memory):
    files = [d for d, _ in corpus.values()]
    traces = [single_trace(ctx, d, sample, interleaved) for d in files]
    rs = read_all(ctx, files, traces, sample, interleaved, memory)
    # the chained file's three streams, the others' one, and the repeated headers of no two files are byte-equal
    assert rs.setup_count == len(files) + 2
    rs.close()


def test_max_packets_one_and_all_alone(ctx, corpus):
    """Every reader one packet per call, and every reader to its end (or its next stop) in each call."""
    files = [d for d, _ in corpus.values()]
    traces = [single_trace(ctx, d, "f32", False) for d in files]
    for schedule in ((1,), (ALL,)):
        read_all(ctx, files, traces, "f32", False, "host", schedule=schedule).close()


def test_pageable_host_pcm_is_refused_and_changes_nothing(ctx, corpus):
    """Pageable host PCM is refused (as lwf_batcher_submit refuses it) before any reader moves: the reads after it
    return the files from their first packet."""
    files = [d for d, _ in corpus.values()]
    traces = [single_trace(ctx, d, "f32", False) for d in files]
    rs = fe.OggStreamReaders(ctx, threads=2)
    for d in files:
        rs.add(d)
    stride = max(rs.stride(i, 3) for i in range(len(files)))
    pageable = np.zeros(len(files) * 10 * stride, np.float32)
    with pytest.raises(L.AudioReadError):
        rs.read([(i, 3) for i in range(len(files))], pageable, stride)
    assert not pageable.any()
    got = rs.read_dec_packets(list(range(len(files))), ALL)
    for i, pk in enumerate(got):
        arrays = [g for g in pk if isinstance(g, list)]
        assert arrays or traces[i][0][0] != "pkt", i
        for k, g in enumerate(arrays):                     # from the first packet on
            e = traces[i][k]
            assert e[0] == "pkt" and bits_equal(np.array(g).reshape(e[1].shape), e[1]), (i, k)
    rs.close()


def test_read_dec_packets_has_the_single_readers_form(ctx, corpus):
    """read_dec_packets gives per reader what read_dec_packet_generic gives call by call: planar lists of channel arrays
    or interleaved arrays, None at the end, and the single reader's exception where it raised one."""
    data = corpus["errors"][0]
    for sample, interleaved in (("f32", False), ("i16", True)):
        single = fe.OggStreamReader(ctx, data)
        rs = fe.OggStreamReaders(ctx)
        rs.add(data)
        for _ in range(20):
            got = rs.read_dec_packets([0], 4, sample, interleaved)[0]
            for g in got:
                try:
                    want = single.read_dec_packet_generic(sample, interleaved)
                except Exception as e:          # noqa: BLE001
                    assert type(g) is type(e) and str(g) == str(e)
                    continue
                if want is None:
                    assert g is None
                elif interleaved:
                    assert np.array_equal(g, want)
                else:
                    assert len(g) == len(want) and all(np.array_equal(a, b) for a, b in zip(g, want))
            if got and got[-1] is None:
                break
        else:
            raise AssertionError("the reader did not reach the end")
        single.close()
        rs.close()


def test_uniform_corpus_runs_on_the_fused_kernels(ctx, oracle):
    """Sixteen stereo 256/2048 files of one encoder setting share one setup and go to the fused kernels (the one-pass
    mixed schedule or k_long), not to the per-packet path of lwb_decode_packet (the four-kernel path)."""
    spec, _, _ = stream(801, 2)
    files = []
    rng = np.random.default_rng(802)
    for k in range(16):
        spec.rng = rng
        packets, infos = [], []
        for mode, prev, nxt in consistent_modes(spec, rng, 12, p_short=0.2 if k % 2 else 0.0):
            pk, info = spec.audio_packet(mode, prev, nxt)
            packets.append(pk)
            infos.append(info)
        want, _ = oracle_pcm(oracle, spec, infos)
        files.append(header_pages(100 + k, spec) + b"".join(audio_pages(100 + k, packets, granules(want, 7), per_page=4)))
    traces = [single_trace(ctx, d, "f32", False) for d in files]
    with expect_kernels(ctx, not_ran=GENERIC | {"k_chain"}) as ran:
        rs = read_all(ctx, files, traces, "f32", False, "device", schedule=(ALL,))
    assert ran["k_long"] + ran["k_long_s"] > 0, ran
    assert set(k for k, v in ran.items() if v) <= FUSED | {"k_row_copy", "k_floor1_segments", "k_prologue_fused"}, ran
    assert rs.setup_count == 1
    rs.close()

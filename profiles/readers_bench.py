"""Many Ogg Vorbis files read packet for packet, three ways: N single OggStreamReaders, the stream batcher fed by
hand-written de-paging (the glue INTEGRATION.md section 4 used to show), and OggStreamReaders (lwf_readers).

Corpora (packets of tests/vorbis_packer.py, long blocks, exact granule positions so that nothing is truncated;
the files of a corpus are a few distinct files repeated):
  uniform   2048 stereo 256/2048 files of one encoder setting (one setup).
  mixed     2048 files: mono, stereo and six-channel 256/2048 files, and one file in eight chained (a stereo stream
            followed by a mono one, crossed during the run).
A step reads 16 packets of every file.  Steps are submitted two deep (step k waits for the ticket of step k - 2 before
it reuses that PCM buffer), with f32 planar PCM in page-locked host memory or in device memory:
  single      lwf_reader_read_dec_packet 16 times per file, on --single-files files only (one lwb_decode_packet and a
              synchronise per packet); its ms_per_step is scaled to the corpus size, its Gsamples/s is as measured.
  batcher     lwf_batcher_submit with one header set per distinct setup (lwf_batcher_add_headers).  The glue's
              de-paging, stream switching at a chained stream and job arrays are made before the timed steps: this is
              the hand glue's best case, its host paging cost not counted.
  readers     lwf_readers_read on the same files; de-paging is part of every step.
Prints one JSON line: per corpus and way, ms per step and Gsamples/s (PCM samples of all channels), the host seconds per
step of the de-paging pass (readers; lwf_readers_last_timing) and of the entropy decode (both ways), with the GPU's
name and power limit read in the same run.  The last step's PCM of readers and batcher is compared bit for bit.
Run from the repository root: python profiles/readers_bench.py"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import lewton_b200 as L  # noqa: E402
import vorbis_packer as vp  # noqa: E402
from lewton_b200 import _cabi as cabi  # noqa: E402
from lewton_b200 import frontend as fe  # noqa: E402

P = 16                        # packets per file per step


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def kind_spec(seed, channels):
    rng = np.random.default_rng(seed)
    spec = vp.StreamSpec(rng, channels=channels)
    long_mode = [m for m, (b, _) in enumerate(spec.modes) if b][0]
    distinct = [spec.audio_packet(long_mode, 1, 1, p_unused=0.02)[0] for _ in range(32)]
    return spec, distinct


def ogg_file(serial, spec, packets):
    """Four packets per page; each page's granule position is the samples decoded up to its last packet (the long
    blocks after the first return blocksize_1 / 2 each), so that the last packet keeps all its samples."""
    hdr = [spec.ident_packet(), spec.comment_packet(), spec.setup_packet()]
    half = (1 << spec.bs1) // 2
    granules = [half * min(k + 3, len(packets) - 1) for k in range(0, len(packets), 4)]
    return vp.ogg_stream(serial, hdr, packets, granules, packets_per_page=4)


def distinct_files(corpus, n_packets):
    """[(file bytes, [(spec, [audio packets of the stream])] per logical stream)]"""
    kinds = {c: kind_spec(90 + c, c) for c in (1, 2, 6)}
    out = []
    for v in range(4):
        plan = [(2, n_packets)] if corpus == "uniform" else [[(1, n_packets)], [(2, n_packets)], [(6, n_packets)]][v % 3]
        if corpus == "mixed" and v == 3:
            plan = [(2, n_packets // 3), (1, n_packets)]         # chained: stereo, then mono
        data, streams = b"", []
        for s, (ch, n) in enumerate(plan):
            spec, distinct = kinds[ch]
            pk = [distinct[(v * 5 + k * 3) % len(distinct)] for k in range(n)]
            data += ogg_file(10 * v + s + 1, spec, pk)
            streams.append((spec, pk))
        out.append((data, streams))
    return out


def corpus_files(corpus, n_files, n_packets):
    d = distinct_files(corpus, n_packets)
    if corpus == "uniform":
        return [d[f % 4] for f in range(n_files)]
    return [d[3] if f % 8 == 7 else d[f % 3] for f in range(n_files)]


def layout(files):
    """element offset of each file's PCM (max channels of its streams x stride), total elements"""
    stride = P * 1024 + (2048 - 256) // 4        # the most 16 packets of a 256/2048 stream return (lwf_readers_read)
    offs, at = [], 0
    for _, streams in files:
        offs.append(at)
        at += max(s.channels for s, _ in streams) * stride
    return offs, at, stride


def buffers(ctx, memory, total):
    """Two zeroed PCM buffers: both ways leave the same elements unwritten, so their last steps compare whole."""
    if memory == "host":
        out = [ctx.host_alloc(total, np.float32) for _ in range(2)]
        for b in out:
            b[...] = 0
        return out
    return [torch.zeros(total, dtype=torch.float32, device="cuda") for _ in range(2)]


def addr(buf):
    return buf.ctypes.data if isinstance(buf, np.ndarray) else buf.data_ptr()


def run_readers(ctx, files, memory, steps, warmup, threads):
    lib = fe.lib()
    rs = fe.OggStreamReaders(ctx, threads=threads)
    for data, _ in files:
        rs.add(data)
    offs, total, stride = layout(files)
    jobs = (fe._ReadJob * len(files))()
    for j in range(len(files)):
        jobs[j].reader, jobs[j].max_packets, jobs[j].out_offset, jobs[j].out_stride = j, P, offs[j], stride
    bufs = buffers(ctx, memory, total)
    mem = cabi.MEM_HOST if memory == "host" else cabi.MEM_DEVICE
    tickets, samples, t = [], 0, C.c_uint64()
    pg, en = C.c_double(), C.c_double()
    for k in range(warmup + steps):
        if k == warmup:
            ctx.synchronize()
            t0, samples, host = time.perf_counter(), 0, [0.0, 0.0]
        if len(tickets) >= 2:
            ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, tickets[-2]))
        ctx.check(lib.lwf_readers_read(rs._h, jobs, len(files), cabi.OUT_F32_PLANAR, addr(bufs[k % 2]), mem, C.byref(t)))
        tickets.append(t.value)
        lib.lwf_readers_last_timing(rs._h, C.byref(pg), C.byref(en), None)
        if k >= warmup:
            host[0] += pg.value
            host[1] += en.value
        samples += sum(jobs[j].n_samples * jobs[j].channels for j in range(len(files)))
        assert all(jobs[j].status == 0 and not jobs[j].ended for j in range(len(files)))
    ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, tickets[-1]))
    wall = time.perf_counter() - t0
    last = bufs[(warmup + steps - 1) % 2]
    last = last if isinstance(last, np.ndarray) else last.cpu().numpy()
    rs.close()
    return wall, samples, last, host


def run_batcher(ctx, files, memory, steps, warmup, threads):
    """The hand glue: every stream de-paged up front, a PreviousWindowRight per logical stream, a header set per
    distinct setup; per step each file's next (up to) 16 packets, a job never spanning two streams and a chained
    stream's first packet decoded with the packets of its first step (it returns no samples, as a fresh state's first
    packet never does) and left out of the count of packets returned."""
    lib = fe.lib()
    offs, total, stride = layout(files)
    setups, bt = {}, None
    plans = {}
    for data, _ in files:
        if id(data) in plans:
            continue
        rd = fe.OggPacketReader(data)
        streams, cur = [], None
        while True:
            pk = rd.read_packet()
            if pk is None:
                break
            if pk.first_in_stream:
                ident, serial = pk.data, pk.stream_serial
                comment, setup = rd.read_packet().data, rd.read_packet().data
                cur = [(ident, setup, comment), serial, []]
                streams.append(cur)
            elif pk.stream_serial == cur[1]:
                cur[2].append(pk.data)
        plans[id(data)] = streams
    for streams in plans.values():
        for (ident, setup, comment), _, _ in streams:
            key = (ident, setup)
            if key not in setups:
                h = fe.Headers(ident, comment, setup)
                su = h.make_setup(ctx)
                if bt is None:
                    bt = fe.StreamBatcher(ctx, h, threads=threads)
                bt.add_headers(h, su)
                setups[key] = (h, su)
    # per file: its streams' states, then the per-step packet lists
    step_jobs = [[] for _ in range(warmup + steps)]
    pwrs = []
    for f, (data, _) in enumerate(files):
        streams = plans[id(data)]
        si, at, pwr = 0, 0, None
        for k in range(warmup + steps):
            ident, setup, _ = streams[si][0]
            pk = streams[si][2]
            if pwr is None:
                pwr = L.PreviousWindowRight(setups[(ident, setup)][1])
                pwrs.append(pwr)
            take = pk[at: at + P + (1 if si and at == 0 else 0)]       # a chained stream: its first packet is dropped
            step_jobs[k].append((pwr, take))
            at += len(take)
            if at >= len(pk) and si + 1 < len(streams):
                si, at, pwr = si + 1, 0, None
    prepared = []
    for k in range(warmup + steps):
        arr = (fe._StreamJob * len(files))()
        keep = []
        for j, (pwr, take) in enumerate(step_jobs[k]):
            pk = (C.c_char_p * max(1, len(take)))(*take)
            ln = (C.c_size_t * max(1, len(take)))(*[len(p) for p in take])
            keep.append((pk, ln))
            arr[j].stream, arr[j].n_packets, arr[j].packets, arr[j].lengths = pwr._h, len(take), pk, ln
            arr[j].out_offset, arr[j].out_stride = offs[j], stride
        prepared.append((arr, keep))
    bufs = buffers(ctx, memory, total)
    mem = cabi.MEM_HOST if memory == "host" else cabi.MEM_DEVICE
    tickets, samples, t = [], 0, C.c_uint64()
    pg, en = C.c_double(), C.c_double()
    chans = [[pwr.setup.output_channels for pwr, _ in step_jobs[k]] for k in range(warmup + steps)]
    for k in range(warmup + steps):
        if k == warmup:
            ctx.synchronize()
            t0, samples, host = time.perf_counter(), 0, [0.0, 0.0]
        if len(tickets) >= 2:
            ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, tickets[-2]))
        arr = prepared[k][0]
        ctx.check(lib.lwf_batcher_submit(bt._h, arr, len(files), cabi.OUT_F32_PLANAR, addr(bufs[k % 2]), mem, C.byref(t)))
        tickets.append(t.value)
        lib.lwf_batcher_last_timing(bt._h, C.byref(en), None)
        if k >= warmup:
            host[1] += en.value
        samples += sum(arr[j].n_samples * chans[k][j] for j in range(len(files)))
    ctx.check(cabi.lib().lwb_ticket_wait(ctx._h, tickets[-1]))
    wall = time.perf_counter() - t0
    last = bufs[(warmup + steps - 1) % 2]
    last = last if isinstance(last, np.ndarray) else last.cpu().numpy()
    bt.close()
    for p in pwrs:
        p.close()
    return wall, samples, last, host


def run_single(ctx, files, steps, warmup):
    lib = fe.lib()
    rds = [fe.OggStreamReader(ctx, data) for data, _ in files]
    buf = ctx.host_alloc(8 * 2048, np.float32)
    n = C.c_size_t()
    samples = 0
    for k in range(warmup + steps):
        if k == warmup:
            t0, samples = time.perf_counter(), 0
        for rd in rds:
            for _ in range(P):
                ctx.check(lib.lwf_reader_read_dec_packet(rd._h, cabi.OUT_F32_PLANAR, buf.ctypes.data, buf.size, C.byref(n)))
                samples += n.value * rd.headers.audio_channels
    wall = time.perf_counter() - t0
    for rd in rds:
        rd.close()
    return wall, samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--single-files", type=int, default=64)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=0)
    args = ap.parse_args()
    cabi.lib().lwb_bind_host_to_device(0)
    ctx = L.Context(0)
    n_packets = (args.steps + args.warmup) * P + 8
    result = {}
    for corpus in ("uniform", "mixed"):
        files = corpus_files(corpus, args.files, n_packets)
        wall, samples = run_single(ctx, files[: args.single_files], args.steps, args.warmup)
        result[f"{corpus}_single"] = {"ms_per_step": wall / args.steps * 1e3 * args.files / args.single_files,
                                      "gsamples_per_s": samples / wall / 1e9, "files_measured": args.single_files}
        for memory in ("host", "device"):
            last = {}
            for way, fn in (("batcher", run_batcher), ("readers", run_readers)):
                wall, samples, last[way], host = fn(ctx, files, memory, args.steps, args.warmup, args.threads)
                result[f"{corpus}_{way}_{memory}"] = {"ms_per_step": wall / args.steps * 1e3, "gsamples_per_s": samples / wall / 1e9,
                                                      "paging_s_per_step": host[0] / args.steps, "entropy_s_per_step": host[1] / args.steps}
            differ = np.nonzero(last["batcher"].view(np.uint32) != last["readers"].view(np.uint32))[0]
            result[f"{corpus}_{memory}_readers_pcm_equals_batcher"] = not differ.size
            if differ.size:
                offs = layout(files)[0]
                result[f"{corpus}_{memory}_first_differing_file"] = int(np.searchsorted(offs, differ[0], "right") - 1)
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "files": args.files, "packets_per_step": P,
                      "steps": args.steps, "host_cpus": os.cpu_count(), **result}))
    ctx.close()


if __name__ == "__main__":
    main()

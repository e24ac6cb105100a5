"""Random access into many Ogg Vorbis files: a step seeks every file to a random granule position, skips a random
number of samples and reads 8 packets, two ways:
  single    OggStreamReader.seek_absgp_pg, skip_samples_linear and 8 read_dec_packet calls per file, on --single-files
            files only (one lwb_decode_packet and a synchronise per packet); its ms per step is scaled to the corpus.
  readers   one OggStreamReaders: lwf_readers_seek_absgp_pg for every file, one lwf_readers_skip_samples_linear call and
            one lwf_readers_read call of 8 packets, f32 planar PCM in device memory, waited for at the end of the step.
The corpus is readers_bench.py's uniform one (2048 stereo 256/2048 files of one setup by default, 48 packets each).  The
goals and skip counts of a step are the same for both ways.  Prints one JSON line: ms per step of each way (median, min
and max over the timed steps), the readers' seek-pass seconds and skip paging seconds (the walk that counts samples,
lwf_readers_last_timing) per step, and the GPU's name and power limit read in the same run; and whether the readers'
skipped and read PCM of the last step equals the single readers' on the files both ran.
Run from the repository root: python profiles/readers_seek_bench.py"""
import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

import lewton_b200 as L  # noqa: E402
from lewton_b200 import frontend as fe  # noqa: E402
from readers_bench import corpus_files, gpu_info  # noqa: E402

READ = 8


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--single-files", type=int, default=64)
    ap.add_argument("--packets", type=int, default=48)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=0)
    a = ap.parse_args()
    name, power = gpu_info()
    ctx = L.Context(0)
    files = [d for d, _ in corpus_files("uniform", a.files, a.packets)]
    total = (a.packets - 4) * 1024
    rng = np.random.default_rng(7)
    steps = [(rng.integers(0, total, a.files), rng.integers(0, 4096, a.files)) for _ in range(a.steps + 1)]

    rs = fe.OggStreamReaders(ctx, threads=a.threads)
    idx = [rs.add(d) for d in files]
    _, skip_stride = rs.skip_room(0)
    read_stride = rs.stride(0, READ)
    skip_buf = torch.zeros(2 * a.files * skip_stride, dtype=torch.float32, device="cuda")
    read_buf = torch.zeros(2 * a.files * read_stride, dtype=torch.float32, device="cuda")
    t_readers, t_seek, t_walk = [], [], []
    for s, (goals, skips) in enumerate(steps):
        t0 = time.perf_counter()
        errs = rs.seek_absgp_pg(idx, goals.tolist())
        t1 = time.perf_counter()
        sk = rs.skip_samples_linear(list(zip(idx, skips.tolist())), skip_buf, skip_stride)
        walk = rs.paging_seconds
        rd = rs.read([(i, READ) for i in idx], read_buf, read_stride)
        rd.wait()
        t2 = time.perf_counter()
        assert not any(errs) and all(r.got_packet for r in sk.results)
        if s:                                  # the first step warms up
            t_readers.append((t2 - t0) * 1e3)
            t_seek.append(t1 - t0)
            t_walk.append(walk)
    skip_host, read_host = skip_buf.cpu().numpy(), read_buf.cpu().numpy()

    n1 = min(a.single_files, a.files)
    singles = [fe.OggStreamReader(ctx, files[i]) for i in range(n1)]
    t_single, same = [], True
    for s, (goals, skips) in enumerate(steps):
        t0 = time.perf_counter()
        out = []
        for i, rd1 in enumerate(singles):
            rd1.seek_absgp_pg(int(goals[i]))
            pk, left = rd1.skip_samples_linear(int(skips[i]))
            out.append((pk, [rd1.read_dec_packet_f32() for _ in range(READ)]))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if s:
            t_single.append((t1 - t0) * 1e3 * a.files / n1)
    for i, (pk, reads) in enumerate(out):       # the last step, file by file
        r = sk.results[i]
        got = np.stack([skip_host[r.out_offset + c * skip_stride: r.out_offset + c * skip_stride + r.n_samples] for c in range(2)])
        same &= np.array_equal(got.view(np.uint32), np.stack(pk).view(np.uint32))
        rr = rd.results[i]
        want = np.concatenate([np.stack(p) for p in reads if p is not None], axis=1)
        got = np.stack([read_host[rr.out_offset + c * read_stride: rr.out_offset + c * read_stride + rr.n_samples] for c in range(2)])
        same &= got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "files": a.files, "single_files": n1,
                      "packets_read_per_file": READ, "steps": a.steps,
                      "readers_ms_per_step": stats(t_readers), "single_ms_per_step_scaled": stats(t_single),
                      "readers_seek_pass_s": stats(t_seek), "readers_skip_paging_s": stats(t_walk),
                      "speedup_median": float(np.median(t_single) / np.median(t_readers)), "pcm_equal": bool(same)}))
    for rd1 in singles:
        rd1.close()
    rs.close()
    ctx.close()


if __name__ == "__main__":
    main()

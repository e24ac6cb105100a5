"""Output sample type against speed: f32, i16, f16, i32 and packed i24 planar PCM on bench.py's shape.

Workload: 4096 stereo streams x 16 long packets per step (spectrum entry, the one-launch k_long path), in two arms:
  device  device-resident spectrum and PCM (bench.py's headline arm), timed with CUDA events on the context's stream;
  e2e     page-locked host arenas (bench.py's e2e arm, --e2e-streams streams), synchronous calls timed on the wall clock.
The formats alternate round by round in one process, so drift of clocks or power hits all five alike.  Prints one JSON
line: per arm and format ms/step, Msamples/s (PCM samples, all channels), the algorithmic bytes per sample (device: 4 B
spectrum in + 4 / 2 / 2 / 4 / 3 B PCM out; e2e: the H2D and D2H bytes per step), with the card's name, its power limit and the
SM clock read in the same run.  Run from the repository root: python profiles/int_out_bench.py"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import lewton_b200 as L  # noqa: E402
from lewton_b200 import _cabi as cabi  # noqa: E402

N2 = 1024
FORMATS = {"f32": (cabi.OUT_F32_PLANAR, 4), "i16": (cabi.OUT_I16_PLANAR, 2), "f16": (cabi.OUT_F16_PLANAR, 2),
           "i32": (cabi.OUT_I32_PLANAR, 4), "i24": (cabi.OUT_I24_PLANAR, 3)}


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--packets", type=int, default=16)
    ap.add_argument("--e2e-streams", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=20, help="timed steps per round and format (device arm)")
    ap.add_argument("--e2e-steps", type=int, default=5, help="timed steps per round and format (e2e arm)")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    S, P, Ch = args.streams, args.packets, 2
    ctx = L.Context(0)
    su = L.Setup(ctx, Ch, 8, 11, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(Ch)], [L.ModeInfo(False), L.ModeInfo(True)])
    stream = torch.cuda.ExternalStream(ctx.cuda_stream, device=torch.device("cuda", 0))
    modes = np.ones(P, np.uint8)
    stride = P * N2
    samples = S * P * Ch * N2

    gen = torch.Generator(device="cuda").manual_seed(1234)
    spec = torch.randn((S, P, Ch, N2), generator=gen, device="cuda", dtype=torch.float32) * 1e-2
    dev = {}
    for name, (fmt, esz) in FORMATS.items():
        pcm = torch.empty((S * Ch * stride * esz,), device="cuda", dtype=torch.uint8)        # raw bytes: i24 has no torch dtype
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        chains = [L.ChainSpec(pwrs[s], modes, coeff_offset=s * P * Ch * N2, out_offset=s * Ch * stride, out_stride=stride)
                  for s in range(S)]
        dev[name] = (L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, spec.data_ptr(), pcm.data_ptr(), fmt), pcm, pwrs)

    Se = min(args.e2e_streams, S)
    h_spec = ctx.host_alloc(Se * P * Ch * N2, np.float32)
    h_spec[:] = (np.random.default_rng(99).standard_normal(h_spec.size) * 1e-2).astype(np.float32)
    e2e = {}
    for name, (fmt, esz) in FORMATS.items():
        h_pcm = ctx.host_alloc(Se * Ch * stride * esz, np.uint8)
        pwrs = [L.PreviousWindowRight(su) for _ in range(Se)]
        chains = [L.ChainSpec(pwrs[s], modes, coeff_offset=s * P * Ch * N2, out_offset=s * Ch * stride, out_stride=stride)
                  for s in range(Se)]
        e2e[name] = (L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, h_spec, h_pcm, fmt), h_pcm, pwrs)

    for name in FORMATS:                                  # warm-up: plans captured, arenas grown
        for _ in range(3):
            dev[name][0].run()
            e2e[name][0].run()
    ctx.synchronize()
    torch.cuda.synchronize()

    dev_ms = {n: [] for n in FORMATS}
    e2e_ms = {n: [] for n in FORMATS}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name in FORMATS:
            run = dev[name][0].run
            ev0.record(stream)
            for _ in range(args.steps):
                run()
            ev1.record(stream)
            ev1.synchronize()
            dev_ms[name].append(ev0.elapsed_time(ev1) / args.steps)
        for name in FORMATS:
            run = e2e[name][0].run
            t0 = time.perf_counter()
            for _ in range(args.e2e_steps):
                run()
            e2e_ms[name].append((time.perf_counter() - t0) * 1e3 / args.e2e_steps)
    card, limits = gpu_info()

    out = {"workload": f"{S} stereo streams x {P} long packets per step (device arm), {Se} streams (e2e arm), spectrum "
                       "entry, planar output", "card": card, "power_limit,sm_clock,sm_clock_max": limits,
           "rounds": args.rounds, "device": {}, "e2e": {}}
    e_samples = Se * P * Ch * N2
    for name, (_, esz) in FORMATS.items():
        ms = float(np.median(dev_ms[name]))
        out["device"][name] = {"ms_per_step": ms, "msamples_per_s": samples / (ms * 1e-3) / 1e6,
                               "bytes_per_sample": 4 + esz, "rounds_ms": dev_ms[name]}
        ms = float(np.median(e2e_ms[name]))
        out["e2e"][name] = {"ms_per_step": ms, "msamples_per_s": e_samples / (ms * 1e-3) / 1e6,
                            "h2d_bytes_per_step": e_samples * 4, "d2h_bytes_per_step": e_samples * esz, "rounds_ms": e2e_ms[name]}
    print(json.dumps(out))
    for d in (dev, e2e):
        for b, _, pwrs in d.values():
            b.close()
            for p in pwrs:
                p.close()
    ctx.close()


if __name__ == "__main__":
    main()

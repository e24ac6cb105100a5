"""What output windows (lwb_stream_set_window) cost: bench.py's device-resident shape (stereo streams of long packets,
n = 2048, spectrum entry, f32 planar, on k_long) with every chain clipped at both ends by up to one packet, against the
same batches unclipped.  Both variants set a window on every stream before every step (the unclipped one the default
window), so both plan every step alike; the clipped one adds the scratch placement and one k_row_copy.

Device-memory batches: CUDA events around lwb_plan_execute, with the stream held by a sleep kernel while the host
plans, so the events time the GPU's work only.  Host-memory batches: the host clock around the synchronous call (planning,
H2D, kernels and D2H), and the bytes their D2H copies move per step (the written samples: dropped ones never cross
PCIe).  The variants alternate step by step.  Prints one JSON line with
the GPU's name and power limit.

    python profiles/window_bench.py [--streams 4096] [--packets 16] [--steps 30]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lewton_b200 as L  # noqa: E402
from lewton_b200 import _cabi as cabi  # noqa: E402

N2 = 1024


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=20).stdout.strip().splitlines()[0]
        name, power, clock = (v.strip() for v in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--packets", type=int, default=16)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    S, P, C = args.streams, args.packets, 2
    ctx = L.Context(0)
    su = L.Setup(ctx, C, 8, 11, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(C)], [L.ModeInfo(False), L.ModeInfo(True)])
    stream = torch.cuda.ExternalStream(ctx.cuda_stream, device=torch.device("cuda", 0))
    gen = torch.Generator(device="cuda").manual_seed(1234)
    spec = torch.randn((S, P, C, N2), generator=gen, device="cuda", dtype=torch.float32) * 1e-2
    stride = P * N2
    rng = np.random.default_rng(0)
    modes = np.ones(P, np.uint8)
    result = {"gpu": gpu_info(), "streams": S, "packets_per_stream": P, "channels": C}

    for memory in (cabi.MEM_DEVICE, cabi.MEM_HOST):
        if memory == cabi.MEM_DEVICE:
            pcm = torch.empty((S, C, stride), device="cuda", dtype=torch.float32)
            co, out = spec.data_ptr(), pcm.data_ptr()
        else:
            h_spec = ctx.host_alloc(spec.numel(), np.float32)
            h_spec[...] = spec.cpu().numpy().ravel()
            h_pcm = ctx.host_alloc(S * C * stride, np.float32)
            co, out = h_spec, h_pcm
        torch.cuda.synchronize()
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        chains = [L.ChainSpec(pwrs[s], modes, coeff_offset=s * P * C * N2, out_offset=s * C * stride, out_stride=stride) for s in range(S)]
        batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, memory, co, out, cabi.OUT_F32_PLANAR)
        produced = P * N2            # per chain and step once the streams are warm (the first step produces (P - 1) * N2)
        times = {"unclipped": [], "clipped": []}
        d2h = {"unclipped": [], "clipped": []}
        launches = {}
        for it in range(2 * (args.warmup + args.steps)):
            variant = ("unclipped", "clipped")[it % 2]
            for p in pwrs:
                if variant == "clipped":
                    skip = int(rng.integers(0, N2 + 1))
                    p.set_window(skip, produced - skip - int(rng.integers(0, N2 + 1)))
                else:
                    p.set_window(0, None)
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            k0 = ctx.kernel_launches()
            if memory == cabi.MEM_DEVICE:
                with torch.cuda.stream(stream):
                    torch.cuda._sleep(50_000_000)      # holds the stream while the host plans the batch
                    ev0.record(stream)
                    batch.run()
                    ev1.record(stream)
            else:
                t0 = time.perf_counter()
                batch.run()                            # returns once the PCM has landed in h_pcm
                ms = (time.perf_counter() - t0) * 1e3
            ctx.synchronize()
            torch.cuda.synchronize()
            k1 = ctx.kernel_launches()
            if it >= 2 * args.warmup:
                times[variant].append(ev0.elapsed_time(ev1) if memory == cabi.MEM_DEVICE else ms)
                d2h[variant].append(sum(c.n_samples for c in batch.collect()) * C * 4)
                launches[variant] = {k: k1[k] - k0[k] for k in k1 if k1[k] != k0[k]}
        key = "device" if memory == cabi.MEM_DEVICE else "host"
        result[key] = {v: {"ms_per_step_median": float(np.median(t)), "ms_per_step_min": float(np.min(t)), "ms_per_step_max": float(np.max(t)),
                           "d2h_bytes_per_step": int(np.median(d2h[v])) if memory == cabi.MEM_HOST else 0, "launches": launches[v]}
                       for v, t in times.items()}
        result[key]["clipped_over_unclipped"] = result[key]["clipped"]["ms_per_step_median"] / result[key]["unclipped"]["ms_per_step_median"]
        del batch, chains, pwrs
    print(json.dumps(result))


if __name__ == "__main__":
    main()

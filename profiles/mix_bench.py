"""Cost of the output channel mix (lwb_setup_set_output_mix).

1. Device-resident, bench.py's shape (S stereo streams x P long 2048-point packets, spectrum entry, f32 planar): no mix
   (k_long), an identity mix (the same bytes through k_chain: what leaving the fused kernel costs) and stereo -> mono.
   CUDA events on the context's stream around `--steps` replays of a prepared batch; the three configurations are
   alternated `--rounds` times, so the spread of each is visible next to the differences between them.
2. Host PCM, 6-channel 256/2048 streams (10 % short blocks) downmixed to stereo: the unmixed batch (six planes cross
   PCIe) followed by a numpy downmix of its PCM, against the mixed batch (two planes cross).  Host wall clock around
   synchronous calls, which return once the PCM has landed in page-locked memory; D2H bytes per step counted from the
   chains' results.

Prints one JSON line per configuration and writes them, with the GPU's name and power limit, to --out."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lewton_b200 as L  # noqa: E402
from lewton_b200 import _cabi as cabi  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                      # (the numbers are then reported without it)
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def make_setup(ctx, C, bs0, bs1):
    return L.Setup(ctx, C, bs0, bs1, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(C)], [L.ModeInfo(False), L.ModeInfo(True)])


def device_part(ctx, args, out):
    S, P, C, N2 = args.streams, args.packets, 2, 1024
    gen = torch.Generator(device="cuda").manual_seed(1234)
    spec = torch.randn((S, P, C, N2), generator=gen, device="cuda", dtype=torch.float32) * 1e-2
    stride = P * N2
    stream = torch.cuda.ExternalStream(ctx.cuda_stream, device=torch.device("cuda", 0))
    configs = {"no_mix": None, "identity_mix": L.mix_select(2, [0, 1]), "stereo_to_mono": L.mix_mono(2)}
    runs = {}
    for name, M in configs.items():
        su = make_setup(ctx, C, 8, 11)
        if M is not None:
            su.set_output_mix(M)
        K = su.output_channels
        pcm = torch.empty((S, K, stride), device="cuda", dtype=torch.float32)
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        chains = [L.ChainSpec(pwrs[s], np.ones(P, np.uint8), coeff_offset=s * P * C * N2, out_offset=s * K * stride,
                              out_stride=stride) for s in range(S)]
        b = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, spec.data_ptr(), pcm.data_ptr(), cabi.OUT_F32_PLANAR)
        k0 = ctx.kernel_launches()
        for _ in range(args.warmup):
            b.run()
        ctx.synchronize()
        k1 = ctx.kernel_launches()
        runs[name] = (b, pcm, pwrs, K, sorted(k for k in k1 if k1[k] > k0[k]))
    ms = {name: [] for name in configs}
    for _ in range(args.rounds):
        for name, (b, _, _, _, _) in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ctx.synchronize()
            e0.record(stream)
            for _ in range(args.steps):
                b.run()
            e1.record(stream)
            ctx.synchronize()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1) / args.steps)
    # the identity mix writes exactly the unmixed bytes
    same = torch.equal(runs["no_mix"][1].view(torch.int32), runs["identity_mix"][1].view(torch.int32))
    for name, (_, _, _, K, kernels) in runs.items():
        m = float(np.median(ms[name]))
        rec = {"part": "device", "config": name, "kernels": kernels, "streams": S, "packets_per_stream": P, "channels_in": C,
               "channels_out": K, "ms_per_step_median": m, "ms_per_step_min": min(ms[name]), "ms_per_step_max": max(ms[name]),
               "rounds": args.rounds, "steps_per_round": args.steps,
               "gsamples_per_s": S * P * C * N2 / (m * 1e-3) / 1e9,
               "hbm_pcm_bytes_per_step": S * P * K * N2 * 4,
               "note": "samples counted per input channel; timer: CUDA events around prepared-batch replays"}
        if name == "identity_mix":
            rec["bytes_equal_no_mix"] = bool(same)
        out.append(rec)
        print(json.dumps(rec), flush=True)
    for b, _, pwrs, _, _ in runs.values():
        b.close()
        for p in pwrs:
            p.close()


def host_part(ctx, args, out):
    S, P, C, bs0, bs1 = args.host_streams, args.packets, 6, 8, 11
    rng = np.random.default_rng(99)
    M = np.array([[1, 0.70710677, 0, 0.70710677, 0, 0], [0, 0.70710677, 1, 0, 0.70710677, 0]], np.float32)
    seqs = []
    for _ in range(S):
        bf = (rng.random(P) >= 0.1).astype(np.uint8)
        prev, nxt = np.ones(P, np.uint8), np.ones(P, np.uint8)
        for i in range(P):
            if bf[i]:
                prev[i] = bf[i - 1] if i else 1
                nxt[i] = bf[i + 1] if i + 1 < P else 1
        seqs.append((bf, prev, nxt))
    n_coeff = sum(C * ((1 << (bs1 if b else bs0)) // 2) for bf, _, _ in seqs for b in bf)
    coeffs = ctx.host_alloc(n_coeff, np.float32)
    coeffs[...] = (rng.standard_normal(n_coeff) * 1e-2).astype(np.float32)
    stride = P * (1 << bs1)
    runs = {}
    for name, mix in (("unmixed_plus_numpy_downmix", None), ("device_mix", M)):
        su = make_setup(ctx, C, bs0, bs1)
        if mix is not None:
            su.set_output_mix(mix)
        K = su.output_channels
        pcm = ctx.host_alloc(S * K * stride, np.float32)
        pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
        chains, coff = [], 0
        for s, (bf, prev, nxt) in enumerate(seqs):
            chains.append(L.ChainSpec(pwrs[s], bf, prev, nxt, coeff_offset=coff, out_offset=s * K * stride, out_stride=stride))
            coff += sum(C * ((1 << (bs1 if b else bs0)) // 2) for b in bf)
        runs[name] = (chains, pcm, pwrs, K)
    stereo = np.empty((S, 2, stride), np.float32)

    def step(name):
        chains, pcm, _, K = runs[name]
        L.decode_chains(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, coeffs, pcm, cabi.OUT_F32_PLANAR)
        if K == C:               # the caller's downmix of the six planes
            x = pcm.reshape(S, C, stride)
            np.matmul(M, x, out=stereo)
        return chains

    for name in runs:
        for _ in range(args.warmup):
            step(name)
    sec = {name: [] for name in runs}
    for _ in range(args.rounds):
        for name in runs:
            t0 = time.perf_counter()
            for _ in range(args.host_steps):
                chains = step(name)
            sec[name].append((time.perf_counter() - t0) / args.host_steps)
    for name, (chains, _, _, K) in runs.items():
        n = sum(int(c.n_samples) for c in chains)
        m = float(np.median(sec[name]))
        rec = {"part": "host", "config": name, "streams": S, "packets_per_stream": P, "channels_in": C, "channels_out": K,
               "short_block_share": 0.1, "d2h_bytes_per_step": n * K * 4, "ms_per_step_median": m * 1e3,
               "ms_per_step_min": min(sec[name]) * 1e3, "ms_per_step_max": max(sec[name]) * 1e3,
               "gsamples_per_s": n * C / m / 1e9, "rounds": args.rounds, "steps_per_round": args.host_steps,
               "note": "samples counted per input channel; timer: host wall clock around synchronous host-memory calls"
                       + ("; includes np.matmul of the 6 planes to stereo" if K == C else "")}
        out.append(rec)
        print(json.dumps(rec), flush=True)
    for chains, _, pwrs, _ in runs.values():
        for p in pwrs:
            p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--packets", type=int, default=16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-streams", type=int, default=512)
    ap.add_argument("--host-steps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "mix_bench.json"))
    args = ap.parse_args()
    ctx = L.Context(0)
    out = []
    device_part(ctx, args, out)
    host_part(ctx, args, out)
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"device": gpu_info(), "results": out}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Mixed short/long streams (256/2048, stereo): throughput of the segmented path (k_long for long runs, k_short
for the short bursts, k_chain for the rest; csrc/path_mixed.cuh) against the same without k_short
(LWB_NO_SHORT=1: short bursts through the chain kernel, the round-1 state) and the chain kernel alone
(LWB_NO_MIXED=1).  Spectrum entry, f32 planar, device-resident, state carried between steps.
One JSON line per (p_short, path)."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch

    import lewton_b200 as L
    from lewton_b200 import _cabi as cabi
    from helpers import mode_sequence

    peak = 3350.0          # H100 SXM data sheet (HBM3), when no measured peak is present
    pth = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pth):
        peak = float(json.load(open(pth))["hbm_gbs"])
    S, P, C = int(os.environ.get("MB_STREAMS", 4096)), int(os.environ.get("MB_PACKETS", 64)), 2
    ctx = L.Context(0)
    stream = torch.cuda.ExternalStream(ctx.cuda_stream)
    su = L.Setup(ctx, C, 8, 11, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(C)], [L.ModeInfo(False), L.ModeInfo(True)])
    rng = np.random.default_rng(1)
    for p_short in [float(x) for x in os.environ.get("MB_PSHORT", "0.02,0.1,0.3").split(",")]:
        seqs, coeff_off, out_off, offs = [], 0, 0, []
        for s in range(S):
            # the same packets are decoded every step on top of the previous step's state: the
            # sequence must close on itself (first and last block long) for that to be a legal stream
            bf = (rng.random(P) >= p_short).astype(np.uint8)
            bf[0] = bf[-1] = 1
            prev, nxt = np.ones(P, np.uint8), np.ones(P, np.uint8)
            for i in range(P):
                if bf[i]:
                    prev[i] = bf[i - 1] if i else 1
                    nxt[i] = bf[i + 1] if i + 1 < P else 1
            # steady state: the stream's saved half matches the first packet's previous window
            n_coeff = int(sum(C * (1024 if b else 128) for b in bf))
            seqs.append((bf.astype(np.uint8), prev, nxt))
            offs.append((coeff_off, out_off))
            coeff_off += n_coeff
            out_off += C * P * 1024          # upper bound per chain
        spec = torch.randn(coeff_off, device="cuda") * 1e-2
        pcm = torch.empty(out_off, device="cuda")
        for path, env in (("segmented", None), ("segmented_noshort", "LWB_NO_SHORT"), ("chain_only", "LWB_NO_MIXED")):
            if env:
                os.environ[env] = "1"
            pw = [L.PreviousWindowRight(su) for _ in range(S)]
            chains = [L.ChainSpec(pw[s], seqs[s][0], seqs[s][1], seqs[s][2], coeff_offset=offs[s][0], out_offset=offs[s][1],
                                  out_stride=P * 1024) for s in range(S)]
            batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, spec.data_ptr(), pcm.data_ptr(),
                            cabi.OUT_F32_PLANAR)
            l0 = ctx.launch_count
            batch.run()
            launches = ctx.launch_count - l0
            for _ in range(2):
                batch.run()
            ctx.synchronize()
            batch.collect()
            samples = sum(ch.n_samples for ch in chains) * C
            reps = 5
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            t0 = time.perf_counter()
            for _ in range(reps):
                batch.run()
            host_ms = (time.perf_counter() - t0) / reps * 1e3
            e1.record(stream)
            ctx.synchronize()
            ms = e0.elapsed_time(e1) / reps
            print(json.dumps({"p_short": p_short, "path": path, "streams": S, "packets": P, "ms": ms, "host_enqueue_ms": host_ms, "launches": launches,
                              "msamples_per_s": samples / ms / 1e3, "achieved_gbs": samples * 8 / ms / 1e6,
                              "frac_of_hbm_peak": samples * 8 / ms / 1e6 / peak}), flush=True)
            batch.close()
            for p in pw:
                p.close()
            if env:
                del os.environ[env]
        del spec, pcm
    su.close()
    ctx.close()


if __name__ == "__main__":
    main()

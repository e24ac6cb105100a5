#!/usr/bin/env python3
"""BASELINE.json configs[4]: synthetic IMDCT(+window+OLA) sweep, n = 64..8192, batch = 1..65536 blocks.

Every point goes through lwb_decode_chains (spectrum entry, f32 planar, device-resident): mono
streams whose setup has blocksize_0 == blocksize_1 == log2(n), one packet-chain per stream.  Long
uniform batches of n = 2048 take the fused kernel (k_long), everything else the generic path.
Prints one JSON line per point: Msamples/s, achieved GB/s on the 8 B/sample algorithmic traffic,
fraction of the HBM peak."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    import lewton_b200 as L
    from lewton_b200 import _cabi as cabi

    peak = 3350.0          # H100 SXM data sheet (HBM3), when no measured peak is present
    pth = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pth):
        peak = float(json.load(open(pth))["hbm_gbs"])
    ctx = L.Context(0)
    stream = torch.cuda.ExternalStream(ctx.cuda_stream)
    P = 8                                   # packets per chain
    for bs in [int(x) for x in os.environ.get("SWEEP_BS", "6,7,8,9,10,11,12,13").split(",")]:
        n = 1 << bs
        su = L.Setup(ctx, 1, bs, bs, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(1)], [L.ModeInfo(True)])
        for log_b in [int(x) for x in os.environ.get("SWEEP_LOGB", "0,4,8,12,16").split(",")]:
            blocks = 1 << log_b
            chains_n = max(1, blocks // P)
            pk = min(P, blocks)
            n2 = n // 2
            total = chains_n * pk * n2
            if total * 8 > (6 << 30):
                continue
            spec = torch.randn(total, device="cuda") * 1e-2
            pcm = torch.empty(total, device="cuda")
            pw = [L.PreviousWindowRight(su) for _ in range(chains_n)]
            modes = np.zeros(pk, np.uint8)
            chains = [L.ChainSpec(pw[i], modes, coeff_offset=i * pk * n2, out_offset=i * pk * n2, out_stride=pk * n2)
                      for i in range(chains_n)]
            batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, spec.data_ptr(), pcm.data_ptr(),
                            cabi.OUT_F32_PLANAR)
            for _ in range(3):
                batch.run()
            ctx.synchronize()
            reps = 5 if total > (1 << 22) else 20
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(reps):
                batch.run()
            e1.record(stream)
            ctx.synchronize()
            ms = e0.elapsed_time(e1) / reps
            samples = chains_n * pk * n2          # steady state: every packet emits n/2 samples
            line = {"n": n, "blocks": chains_n * pk, "ms": ms, "msamples_per_s": samples / ms / 1e3,
                    "achieved_gbs": samples * 8 / ms / 1e6, "frac_of_hbm_peak": samples * 8 / ms / 1e6 / peak,
                    "path": "fused k_long" if bs == 11 else "fused k_short" if bs == 8 else "fused k_mid" if bs in (9, 10) else "chain kernel"}
            print(json.dumps(line), flush=True)
            batch.close()
            for p in pw:
                p.close()
            del spec, pcm
        su.close()
    ctx.close()


if __name__ == "__main__":
    main()

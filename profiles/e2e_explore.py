#!/usr/bin/env python3
"""How close is `e2e` (host buffers through lwb_decode_chains) to what the PCIe link gives?
Measures on one H100: pinned H2D alone, D2H alone, both directions at once (256 MiB each, two
streams, CUDA events), then the e2e call with f32 and with i16 PCM.  One JSON line."""
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

    nbytes = 256 << 20
    h_a = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    h_b = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    d_a = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    d_b = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    out = {}

    def timeit(fn, reps=8):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps

    def h2d():
        with torch.cuda.stream(s1):
            d_a.copy_(h_a, non_blocking=True)

    def d2h():
        with torch.cuda.stream(s2):
            h_b.copy_(d_b, non_blocking=True)

    def both():
        h2d()
        d2h()

    out["h2d_alone_gbs"] = nbytes / timeit(h2d) / 1e9
    out["d2h_alone_gbs"] = nbytes / timeit(d2h) / 1e9
    out["duplex_each_way_gbs"] = nbytes / timeit(both) / 1e9

    ctx = L.Context(0)
    S, P, C, N2 = 2048, 16, 2, 1024
    su = L.Setup(ctx, C, 8, 11, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(C)], [L.ModeInfo(False), L.ModeInfo(True)])
    lib = cabi.lib()
    h_spec = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_float * (S * P * C * N2)).from_address(lib.lwb_host_alloc(S * P * C * N2 * 4)))
    h_spec[:] = (np.random.default_rng(5).standard_normal(h_spec.size) * 1e-2).astype(np.float32)
    stride = P * N2
    modes = np.ones(P, np.uint8)
    for name, fmt, ct, esz in (("f32", cabi.OUT_F32_PLANAR, np.ctypeslib.ctypes.c_float, 4),
                               ("i16", cabi.OUT_I16_PLANAR, np.ctypeslib.ctypes.c_int16, 2)):
        h_pcm = np.ctypeslib.as_array((ct * (S * C * stride)).from_address(lib.lwb_host_alloc(S * C * stride * esz)))
        pw = [L.PreviousWindowRight(su) for _ in range(S)]
        chains = [L.ChainSpec(pw[s], modes, coeff_offset=s * P * C * N2, out_offset=s * C * stride, out_stride=stride) for s in range(S)]
        batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, h_spec, h_pcm, fmt)
        for _ in range(3):
            batch.run()
        t0 = time.perf_counter()
        for _ in range(10):
            batch.run()
        sec = (time.perf_counter() - t0) / 10
        out[f"e2e_{name}_msamples_per_s"] = S * P * C * N2 / sec / 1e6
        out[f"e2e_{name}_h2d_gbs"] = S * P * C * N2 * 4 / sec / 1e9
        out[f"e2e_{name}_d2h_gbs"] = S * P * C * N2 * esz / sec / 1e9
        batch.close()
        for p in pw:
            p.close()
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

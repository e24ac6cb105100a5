import os, sys, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import lewton_b200 as L
from lewton_b200 import _cabi as cabi
ctx = L.Context(0)
S, P, C, N2 = 2048, 16, 2, 1024
su = L.Setup(ctx, C, 8, 11, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(C)], [L.ModeInfo(False), L.ModeInfo(True)])
lib = cabi.lib()
ct = np.ctypeslib.ctypes
h_spec = np.ctypeslib.as_array((ct.c_float * (S * P * C * N2)).from_address(lib.lwb_host_alloc(S * P * C * N2 * 4)))
h_spec[:] = (np.random.default_rng(5).standard_normal(h_spec.size) * 1e-2).astype(np.float32)
stride = P * N2
modes = np.ones(P, np.uint8)
out = {}
for name, fmt, cty, esz in (("f32", cabi.OUT_F32_PLANAR, ct.c_float, 4), ("i16", cabi.OUT_I16_PLANAR, ct.c_int16, 2)):
    h_pcm = np.ctypeslib.as_array((cty * (S * C * stride)).from_address(lib.lwb_host_alloc(S * C * stride * esz)))
    for mode, mem in (("staged", cabi.MEM_HOST), ("zero_copy", cabi.MEM_DEVICE)):
        pw = [L.PreviousWindowRight(su) for _ in range(S)]
        chains = [L.ChainSpec(pw[s], modes, coeff_offset=s * P * C * N2, out_offset=s * C * stride, out_stride=stride) for s in range(S)]
        if mem == cabi.MEM_HOST:
            batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, mem, h_spec, h_pcm, fmt)
        else:
            batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, mem, h_spec.ctypes.data, h_pcm.ctypes.data, fmt)
        for _ in range(3):
            batch.run(); ctx.synchronize()
        ref = h_pcm.copy()
        t0 = time.perf_counter()
        for _ in range(10):
            batch.run(); ctx.synchronize()
        sec = (time.perf_counter() - t0) / 10
        out[f"{name}_{mode}_msamples_per_s"] = S * P * C * N2 / sec / 1e6
        out[f"{name}_{mode}_checksum"] = float(np.abs(h_pcm.astype(np.float64)).sum())
        batch.close()
        for p in pw: p.close()
print(json.dumps(out))

#!/usr/bin/env python3
"""End-to-end style line for the residue entries (SURVEY.md 8f rank 2): host (pinned) buffers in, PCM in host buffers out,
through lwb_decode_chains / lwb_plan_execute, one H100.  The packets are real Vorbis audio packets made by
tests/vorbis_packer.py (stereo, residue type 2, one coupling step, ~365 bytes per 2048-sample long packet = the size of a
128 kbit/s stream), entropy-decoded ONCE on the host; what is timed is everything behind the entropy decode:

  residue_f32 / residue_i16 : dense residue vectors cross PCIe (8 B per coefficient in), LWB_ENTRY_RESIDUE
  vq_f32 / vq_i16           : VQ runs + 16-bit codebook entries cross PCIe instead, the device accumulates, LWB_ENTRY_VQ

One JSON line per case; h2d / d2h bytes per step counted from the arrays handed over."""
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pinned(shape, dtype):
    from lewton_b200 import _cabi as cabi
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = cabi.lib().lwb_host_alloc(max(n, 16))
    buf = (C.c_char * max(n, 16)).from_address(p)
    return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)


def main():
    import lewton_b200 as L
    import vorbis_packer as vp
    from lewton_b200 import _cabi as cabi
    from lewton_b200 import frontend as fe

    S, P, D = int(os.environ.get("VQ_STREAMS", 2048)), 16, 32
    cabi.lib().lwb_bind_host_to_device(0)
    ctx = L.Context(0)
    rng = np.random.default_rng(12)
    spec = vp.StreamSpec(rng, channels=2, cascade_p=0.3, residue_types=[2], n_modes=2)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    assert hdr.vq_capable()
    su = hdr.make_setup(ctx)
    mode = [i for i, (bf, _) in enumerate(spec.modes) if bf][0]
    dist = []
    for d in range(D):
        pk, _ = spec.audio_packet(mode, 1, 1, p_unused=0.0)
        dense = hdr.decode_packet(pk)
        _, runs, ents = hdr.decode_packet_vq(pk)
        k, y, _ = dense.pack()
        dist.append((len(pk), dense.residue, k, y, runs, ents))
    rows = S * P
    pick = np.random.default_rng(5).integers(0, D, rows)
    res = pinned((rows, 2, 1024), np.float32)
    kinds = pinned((rows, 2), np.uint8)
    ys = pinned((rows, 2, cabi.MAX_POSTS), np.uint32)
    nrun = np.array([len(dist[d][4]) for d in pick]); nent = np.array([len(dist[d][5]) for d in pick])
    roff = pinned((rows + 1,), np.uint64); eoff = pinned((rows + 1,), np.uint64)
    roff[0] = eoff[0] = 0
    roff[1:] = np.cumsum(nrun); eoff[1:] = np.cumsum(nent)
    runs = pinned((int(roff[-1]),), fe.VQ_RUN_DTYPE); ents = pinned((int(eoff[-1]),), np.uint16)
    for r, d in enumerate(pick):
        _, rr, k, y, ru, en = dist[d]
        res[r], kinds[r], ys[r] = rr, k, y
        runs[int(roff[r]):int(roff[r + 1])] = ru
        ents[int(eoff[r]):int(eoff[r + 1])] = en
    stride = P * 1024
    modes = np.full(P, mode, np.uint8)
    pkt_bytes = float(np.mean([dist[d][0] for d in pick]))
    for case, entry, fmt, dt in (("residue_f32", cabi.ENTRY_RESIDUE, cabi.OUT_F32_PLANAR, np.float32),
                                 ("residue_i16", cabi.ENTRY_RESIDUE, cabi.OUT_I16_PLANAR, np.int16),
                                 ("vq_f32", cabi.ENTRY_VQ, cabi.OUT_F32_PLANAR, np.float32),
                                 ("vq_i16", cabi.ENTRY_VQ, cabi.OUT_I16_PLANAR, np.int16)):
        pcm = pinned((S, 2, stride), dt)
        pw = [L.PreviousWindowRight(su) for _ in range(S)]
        chains = [L.ChainSpec(pw[s], modes, coeff_offset=s * P * 2048, packet_index=s * P, out_offset=s * 2 * stride, out_stride=stride)
                  for s in range(S)]
        kw = dict(floor_kind=kinds, floor1_y=ys)
        h2d = kinds.nbytes + ys.nbytes
        if entry == cabi.ENTRY_VQ:
            kw["vq"] = (runs, roff, ents, eoff)
            h2d += runs.nbytes + ents.nbytes + roff.nbytes + eoff.nbytes
        else:
            h2d += res.nbytes
        batch = L.Batch(ctx, chains, entry, cabi.MEM_HOST, None if entry == cabi.ENTRY_VQ else res, pcm, fmt, **kw)
        for _ in range(3):
            batch.run()
        reps = 8
        t0 = time.perf_counter()
        for _ in range(reps):
            batch.run()
        sec = (time.perf_counter() - t0) / reps
        samples = S * P * 2 * 1024
        print(json.dumps({"case": case, "streams": S, "packets_per_stream": P, "ms_per_step": sec * 1e3, "msamples_per_s": samples / sec / 1e6,
                          "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(pcm.nbytes),
                          "h2d_bytes_per_packet": h2d / rows, "bitstream_bytes_per_packet": pkt_bytes,
                          "vq_runs_per_packet": float(nrun.mean()), "vq_vectors_per_packet": float(nent.mean()),
                          "note": "host pinned buffers in and out, synchronous call, entropy decode not included"}), flush=True)
        batch.close()
        for p in pw:
            p.close()
    ctx.close()


if __name__ == "__main__":
    main()

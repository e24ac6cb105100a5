#!/usr/bin/env python3
"""Throughput of the other shapes SURVEY.md section 8(d) asks to be reported beside the headline
(device-resident, one H100, CUDA events on the library's stream, one JSON line per case):

  long_f32        S x P stereo long packets, spectrum entry, f32 planar           8 B / sample (the headline)
  long_i16        same, i16 planar output                                          6 B / sample
  long_residue    same, residue entry: coupling (0,1) + floor-1 + multiply; floor posts device-resident
                  (lwb_batch_io::floor_memory); k_floor1_segments + k_prologue_fused + k_long, captured plan   18 B / sample moved, 8 algorithmic
  long_residue_hostfloors   same with host floor arrays (uploaded every step)
  streaming_p1    one packet per stream per call (state round-trips HBM)           16 B / sample
  config3_6ch     BASELINE.json configs[2] shape: 6 channels, Bernoulli(0.25) short blocks, coupling chain
                  (0,1),(2,3),(0,4), floor-1, residue entry; segmented path (k_prologue + k_long, k_chain)
Inputs are synthetic (N(0,1)*1e-2 residues, random valid floor-1 posts drawn from a pool of 64 rows)."""
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
    from helpers import make_setup, random_floor1_y

    peak = 3350.0          # H100 SXM data sheet (HBM3), when no measured peak is present
    pth = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pth):
        peak = float(json.load(open(pth))["hbm_gbs"])
    ctx = L.Context(0)
    stream = torch.cuda.ExternalStream(ctx.cuda_stream)
    rng = np.random.default_rng(1234)
    floors = [(1, [0, 1024] + [int(v) for v in rng.permutation(np.arange(1, 1024))[:30]])]

    def timed(batch, reps=10, warm=3):
        l0 = ctx.launch_count
        batch.run()
        launches = ctx.launch_count - l0
        for _ in range(warm - 1):
            batch.run()
        ctx.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t0 = time.perf_counter()
        for _ in range(reps):
            batch.run()
        host_ms = (time.perf_counter() - t0) / reps * 1e3
        e1.record(stream)
        ctx.synchronize()
        return e0.elapsed_time(e1) / reps, host_ms, launches

    def report(case, samples, ms, host_ms, launches, bytes_per_sample, note):
        print(json.dumps({"case": case, "ms": ms, "host_enqueue_ms": host_ms, "launches": launches,
                          "msamples_per_s": samples / ms / 1e3, "algorithmic_bytes_per_sample": bytes_per_sample,
                          "achieved_gbs": samples * bytes_per_sample / ms / 1e6,
                          "frac_of_hbm_peak": samples * bytes_per_sample / ms / 1e6 / peak, "note": note}), flush=True)

    def floor_rows(rows, nposts, mult):
        pool = np.zeros((64, cabi.MAX_POSTS), np.uint32)
        for i in range(64):
            pool[i, :nposts] = random_floor1_y(rng, mult, nposts)
        return pool[rng.integers(0, 64, rows)]

    # ---- uniform long batches ------------------------------------------------------------------
    S, P, C = 4096, 16, 2
    su = make_setup(ctx, C, 8, 11, mappings=[{"coupling": [(0, 1)], "floor_of_channel": [0, 0]}], floors=floors)
    spec = torch.randn(S * P * C * 1024, device="cuda") * 1e-2
    modes = np.ones(P, np.uint8)
    for case, fmt, entry, bps in (("long_f32", cabi.OUT_F32_PLANAR, cabi.ENTRY_SPECTRUM, 8),
                                  ("long_i16", cabi.OUT_I16_PLANAR, cabi.ENTRY_SPECTRUM, 6),
                                  ("long_residue", cabi.OUT_F32_PLANAR, cabi.ENTRY_RESIDUE, 8),
                                  ("long_residue_i16", cabi.OUT_I16_PLANAR, cabi.ENTRY_RESIDUE, 6),
                                  ("long_residue_hostfloors", cabi.OUT_F32_PLANAR, cabi.ENTRY_RESIDUE, 8)):
        pcm = torch.empty(S * C * P * 1024, device="cuda", dtype=torch.float32 if fmt == cabi.OUT_F32_PLANAR else torch.int16)
        pw = [L.PreviousWindowRight(su) for _ in range(S)]
        chains = [L.ChainSpec(pw[s], modes, coeff_offset=s * P * C * 1024, packet_index=s * P, out_offset=s * C * P * 1024,
                              out_stride=P * 1024) for s in range(S)]
        kw, keep = {}, None
        if entry == cabi.ENTRY_RESIDUE:
            h_kinds, h_ys = np.full(S * P * C, cabi.FLOOR_ONE, np.uint8), floor_rows(S * P * C, len(floors[0][1]), 1)
            if case.endswith("hostfloors"):
                kw = dict(floor_kind=h_kinds, floor1_y=h_ys)
            else:
                keep = (torch.from_numpy(h_kinds).cuda(), torch.from_numpy(h_ys.view(np.int32)).cuda())
                kw = dict(floor_kind=keep[0].data_ptr(), floor1_y=keep[1].data_ptr(), floor_memory=cabi.MEM_DEVICE)
        batch = L.Batch(ctx, chains, entry, cabi.MEM_DEVICE, spec.data_ptr(), pcm.data_ptr(), fmt, **kw)
        ms, host_ms, launches = timed(batch)
        report(case, S * P * C * 1024, ms, host_ms, launches, bps,
               f"{S} stereo streams x {P} long packets" +
               (", floor posts in host arrays, uploaded every step" if case.endswith("hostfloors") else
                ", floor posts device-resident, front stages + fused kernel replayed from the plan" if kw else ""))
        del keep
        batch.close()
        for p in pw:
            p.close()
        del pcm
    del spec

    # ---- one packet per stream per call ----------------------------------------------------------
    S1 = 65536
    spec = torch.randn(S1 * C * 1024, device="cuda") * 1e-2
    pcm = torch.empty(S1 * C * 1024, device="cuda")
    pw = [L.PreviousWindowRight(su) for _ in range(S1)]
    one = np.ones(1, np.uint8)
    chains = [L.ChainSpec(pw[s], one, coeff_offset=s * C * 1024, out_offset=s * C * 1024, out_stride=1024) for s in range(S1)]
    batch = L.Batch(ctx, chains, cabi.ENTRY_SPECTRUM, cabi.MEM_DEVICE, spec.data_ptr(), pcm.data_ptr(), cabi.OUT_F32_PLANAR)
    ms, host_ms, launches = timed(batch)
    report("streaming_p1", S1 * C * 1024, ms, host_ms, launches, 16, f"{S1} stereo streams x 1 long packet per call")
    batch.close()
    for p in pw:
        p.close()
    del spec, pcm
    su.close()

    # ---- config 3: 6 channels, mixed blocks, coupling chain, floor-1, residue entry ----------------
    S3, P3, C3 = 1024, 64, 6
    su3 = make_setup(ctx, C3, 8, 11, mappings=[{"coupling": [(0, 1), (2, 3), (0, 4)], "floor_of_channel": [0] * C3}], floors=floors)
    seqs, coeff_off, offs, total_rows = [], 0, [], 0
    for s in range(S3):
        bf = (rng.random(P3) >= 0.25).astype(np.uint8)
        bf[0] = bf[-1] = 1
        prev, nxt = np.ones(P3, np.uint8), np.ones(P3, np.uint8)
        for i in range(P3):
            if bf[i]:
                prev[i] = bf[i - 1] if i else 1
                nxt[i] = bf[i + 1] if i + 1 < P3 else 1
        seqs.append((bf, prev, nxt))
        offs.append(coeff_off)
        coeff_off += int(sum(C3 * (1024 if b else 128) for b in bf))
    res = torch.randn(coeff_off, device="cuda") * 1e-2
    pcm = torch.empty(S3 * C3 * P3 * 1024, device="cuda")
    pw = [L.PreviousWindowRight(su3) for _ in range(S3)]
    chains = [L.ChainSpec(pw[s], seqs[s][0], seqs[s][1], seqs[s][2], coeff_offset=offs[s], packet_index=s * P3,
                          out_offset=s * C3 * P3 * 1024, out_stride=P3 * 1024) for s in range(S3)]
    rows = S3 * P3 * C3
    h_kinds, h_ys = np.full(rows, cabi.FLOOR_ONE, np.uint8), floor_rows(rows, len(floors[0][1]), 1)
    d_kinds, d_ys = torch.from_numpy(h_kinds).cuda(), torch.from_numpy(h_ys.view(np.int32)).cuda()
    batch = L.Batch(ctx, chains, cabi.ENTRY_RESIDUE, cabi.MEM_DEVICE, res.data_ptr(), pcm.data_ptr(), cabi.OUT_F32_PLANAR,
                    floor_kind=d_kinds.data_ptr(), floor1_y=d_ys.data_ptr(), floor_memory=cabi.MEM_DEVICE)
    # output check on a sample of the streams: a fresh batch run from empty states against the oracle
    from helpers import RefStream, bits_equal
    from oracle import oracle
    oracle.build()
    pcm.zero_()
    batch.run()
    ctx.synchronize()
    batch.collect()
    checked = 0
    for s in (0, 1, S3 // 2, S3 - 1):
        ref = RefStream(oracle, C3, 8, 11, [(0, 0), (1, 0)], [{"coupling": [(0, 1), (2, 3), (0, 4)], "floor_of_channel": [0] * C3}], floors)
        bf, prev, nxt = seqs[s]
        h_res = res[offs[s]:(offs[s + 1] if s + 1 < S3 else coeff_off)].cpu().numpy()
        pos, parts = 0, []
        for i in range(P3):
            n2 = 1024 if bf[i] else 128
            r = h_res[pos:pos + C3 * n2].reshape(C3, n2)
            pos += C3 * n2
            fl = [[int(v) for v in h_ys[(s * P3 + i) * C3 + c][:len(floors[0][1])]] for c in range(C3)]
            rc, o = ref.packet(int(bf[i]), int(prev[i]), int(nxt[i]), r, fl)
            assert rc == 0
            parts.append(o)
        want = np.concatenate(parts, axis=1)
        got = pcm[s * C3 * P3 * 1024:(s + 1) * C3 * P3 * 1024].cpu().numpy().reshape(C3, P3 * 1024)[:, :want.shape[1]]
        assert chains[s].n_samples == want.shape[1] and bits_equal(got, want), f"config3_6ch stream {s} differs from the oracle"
        checked += 1
    ms, host_ms, launches = timed(batch, reps=5)
    batch.collect()
    samples = sum(ch.n_samples for ch in chains) * C3
    report("config3_6ch", samples, ms, host_ms, launches, 8,
           f"{S3} streams x {P3} packets x 6 ch, 25 % short blocks, residue entry, device floor arrays, captured plan; "
           f"{checked} streams of the first run checked bit-exact against the oracle")
    batch.close()
    ctx.close()


if __name__ == "__main__":
    main()

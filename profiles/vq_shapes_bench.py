"""LWB_ENTRY_VQ against LWB_ENTRY_RESIDUE on the batch shapes the fused long-block path does not take, from page-locked
host memory, one GPU.

Shapes (real Vorbis packets made by tests/vorbis_packer.py, entropy-decoded once on the host and tiled over the streams):
  itl_256_2048   stereo 256/2048 streams, 10 % short blocks, i16 interleaved output   (k_chain)
  mid_1024       uniform stereo 1024-point streams, f32 planar                        (front stages + k_mid)
  six_512_4096   6-channel 512/4096 streams, f32 planar                               (k_chain)
Modes, in rounds that alternate in one process:
  residue        dense residue vectors cross PCIe
  vq             VQ runs and 16-bit codebook entries cross PCIe instead; the device accumulates the vectors
  vq_four_kernel the same VQ batch on the four-kernel path (LWB_FORCE_GENERIC=1), where such batches went before
Each mode is timed two ways: synchronous lwb_decode_chains steps (ms per step, wall), and lwb_submit_chains two deep
over two output arenas (ms per step, wall, and how long lwb_submit_chains holds the caller).  One JSON line per shape,
with the GPU's name and power limit read in the same run.  Run from the repository root: python profiles/vq_shapes_bench.py"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lewton_b200 as L  # noqa: E402
import vorbis_packer as vp  # noqa: E402
from lewton_b200 import _cabi as cabi  # noqa: E402
from lewton_b200 import frontend as fe  # noqa: E402
from lewton_b200.api import _marshal  # noqa: E402

# name: channels, bs0, bs1, share of short blocks, output format, streams
SHAPES = {
    "itl_256_2048": (2, 8, 11, 0.1, cabi.OUT_I16_INTERLEAVED, 1024),
    "mid_1024": (2, 10, 10, 0.0, cabi.OUT_F32_PLANAR, 2048),
    "six_512_4096": (6, 9, 12, 0.1, cabi.OUT_F32_PLANAR, 256),
}


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def distinct_streams(channels, bs0, bs1, p_short, D, P, seed):
    """D packer streams of P packets of one VQ-capable setup: headers and, per stream, the packets' bytes."""
    for k in range(40):
        rng = np.random.default_rng(seed + 1000 * k)
        spec = vp.StreamSpec(rng, channels=channels, bs0=bs0, bs1=bs1, cascade_p=0.3)
        hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        if not hdr.vq_capable():
            hdr.close()
            continue
        long_modes = [i for i, (bf, _) in enumerate(spec.modes) if bf]
        short_modes = [i for i, (bf, _) in enumerate(spec.modes) if not bf]
        streams = []
        for _ in range(D):
            bf = rng.random(P) >= p_short
            bf[0] = bf[-1] = True
            pk = []
            for i in range(P):
                mode = int(rng.choice(long_modes if bf[i] else short_modes))
                prev = int(bf[i - 1]) if i else 1
                nxt = int(bf[(i + 1) % P])           # (the stream repeats: the last packet's neighbour is the first)
                pk.append(spec.audio_packet(mode, prev, nxt, p_unused=0.05)[0])
            streams.append(pk)
        return hdr, streams
    raise AssertionError("no VQ-capable draw")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packets", type=int, default=16, help="packets per stream and step")
    ap.add_argument("--distinct", type=int, default=16, help="distinct packet streams, tiled over the batch's streams")
    ap.add_argument("--seconds", type=float, default=1.0, help="least duration of one round of one mode")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    lib = cabi.lib()
    lib.lwb_bind_host_to_device(0)
    ctx = L.Context(0)
    name, power = gpu_info()
    P, D = args.packets, args.distinct

    def check(rc):
        if rc:
            raise L.AudioReadError(rc, lib.lwb_last_error(ctx._h).decode())

    for shape in args.shapes.split(","):
        Ch, bs0, bs1, p_short, fmt, S = SHAPES[shape]
        hdr, dist = distinct_streams(Ch, bs0, bs1, p_short, D, P, 31)
        su = hdr.make_setup(ctx)
        # host decode of the distinct streams, once: per packet (dense residue, kinds, ys, VQ runs, VQ entries, mode bytes)
        dec = []
        for pk in dist:
            rows = []
            for p in pk:
                d = hdr.decode_packet(p)
                v, rr, ee = hdr.decode_packet_vq(p)
                k, y, _ = d.pack()
                rows.append((d.residue.ravel(), k, y, rr, ee, (v.mode_number, v.prev_window_flag, v.next_window_flag),
                             hdr.decoded_sample_count(p)))
            dec.append(rows)
        pick = [s % D for s in range(S)]
        n_coeff = sum(sum(r[0].size for r in dec[d]) for d in pick)
        coeffs = ctx.host_alloc(n_coeff, np.float32)
        kinds = ctx.host_alloc((S * P, Ch), np.uint8)
        ys = ctx.host_alloc((S * P, Ch, cabi.MAX_POSTS), np.uint32)
        nrun = [len(r[3]) for d in pick for r in dec[d]]
        nent = [len(r[4]) for d in pick for r in dec[d]]
        roff, eoff = ctx.host_alloc(S * P + 1, np.uint64), ctx.host_alloc(S * P + 1, np.uint64)
        roff[0] = eoff[0] = 0
        roff[1:], eoff[1:] = np.cumsum(nrun), np.cumsum(nent)
        runs = ctx.host_alloc(max(int(roff[-1]), 1), fe.VQ_RUN_DTYPE)
        ents = ctx.host_alloc(max(int(eoff[-1]), 1), np.uint16)
        planar = fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_I16_PLANAR)
        dt = np.float32 if fmt in (cabi.OUT_F32_PLANAR, cabi.OUT_F32_INTERLEAVED) else np.int16
        stride = (max(sum(r[6] for r in rows) for rows in dec) + 3) // 4 * 4
        chains = {m: [] for m in ("residue", "vq", "vq_four_kernel")}
        pwrs = {m: [] for m in chains}
        coff = row = 0
        for s, d in enumerate(pick):
            c0 = coff
            for r in dec[d]:
                coeffs[coff:coff + r[0].size] = r[0]
                kinds[row], ys[row] = r[1], r[2]
                runs[int(roff[row]):int(roff[row + 1])] = r[3]
                ents[int(eoff[row]):int(eoff[row + 1])] = r[4]
                coff += r[0].size
                row += 1
            modes, prev, nxt = (np.array([r[5][j] for r in dec[d]], np.uint8) for j in range(3))
            for m in chains:
                pw = L.PreviousWindowRight(su)
                pwrs[m].append(pw)
                chains[m].append(L.ChainSpec(pw, modes, prev, nxt, coeff_offset=c0, packet_index=s * P, out_offset=s * Ch * stride,
                                             out_stride=stride if planar else 0))
        outs = [ctx.host_alloc(S * Ch * stride, dt) for _ in range(2)]
        marshalled = {}
        for m in chains:
            vq = m != "residue"
            for k in range(2):
                marshalled[m, k] = _marshal(chains[m], cabi.ENTRY_VQ if vq else cabi.ENTRY_RESIDUE, cabi.MEM_HOST, None if vq else coeffs,
                                            outs[k], fmt, kinds, ys, None, cabi.MEM_HOST, (runs, roff, ents, eoff) if vq else None)
        h2d = {"residue": coeffs.nbytes + kinds.nbytes + ys.nbytes}
        h2d["vq"] = h2d["vq_four_kernel"] = kinds.nbytes + ys.nbytes + runs.nbytes + ents.nbytes + roff.nbytes + eoff.nbytes

        def run(mode, how, seconds):
            """Back-to-back steps for >= seconds: (steps, wall seconds, host seconds inside the library calls)."""
            if mode == "vq_four_kernel":
                os.environ["LWB_FORCE_GENERIC"] = "1"
            steps, host, tickets, t = 0, 0.0, [], C.c_uint64()
            t0 = time.perf_counter()
            try:
                while True:
                    arr, io = marshalled[mode, steps % 2]
                    if how == "sync":
                        h0 = time.perf_counter()
                        check(lib.lwb_decode_chains(ctx._h, arr, S, C.byref(io)))
                    else:
                        if len(tickets) >= 2:
                            check(lib.lwb_ticket_wait(ctx._h, tickets[-2]))
                        h0 = time.perf_counter()
                        check(lib.lwb_submit_chains(ctx._h, arr, S, C.byref(io), C.byref(t)))
                        tickets.append(t.value)
                    host += time.perf_counter() - h0
                    steps += 1
                    if time.perf_counter() - t0 >= seconds:
                        break
                if tickets:
                    check(lib.lwb_ticket_wait(ctx._h, tickets[-1]))
            finally:
                os.environ.pop("LWB_FORCE_GENERIC", None)
            return steps, time.perf_counter() - t0, host

        for m in chains:
            for how in ("sync", "async"):
                run(m, how, 0.2)                   # warm-up: arenas, staging and stream states in their steady state
        # the PCM of one step, all three modes: the same bytes
        ref = None
        for m in chains:
            outs[0].fill(0)
            arr, io = marshalled[m, 0]
            if m == "vq_four_kernel":
                os.environ["LWB_FORCE_GENERIC"] = "1"
            check(lib.lwb_decode_chains(ctx._h, arr, S, C.byref(io)))
            os.environ.pop("LWB_FORCE_GENERIC", None)
            assert ref is None or outs[0].tobytes() == ref, f"{shape}: {m} differs from the residue entry"
            ref = outs[0].tobytes()
        samples = Ch * sum(int(arr[i].n_samples) for i in range(S))
        acc = {(m, how): [0, 0.0, 0.0] for m in chains for how in ("sync", "async")}
        for _ in range(args.rounds):
            for key in acc:
                steps, wall, host = run(*key, args.seconds)
                acc[key][0] += steps
                acc[key][1] += wall
                acc[key][2] += host
        result = {}
        for (m, how), (steps, wall, host) in acc.items():
            result[f"{m}_{how}"] = {"ms_per_step": wall / steps * 1e3, "host_ms_per_call": host / steps * 1e3,
                                    "msamples_per_s": samples * steps / wall / 1e6, "steps": steps}
        print(json.dumps({"shape": shape, "gpu": name, "power_limit_and_max_sm_clock": power, "streams": S, "packets_per_stream": P,
                          "channels": Ch, "blocksizes": [1 << bs0, 1 << bs1], "pcm_samples_per_step": samples,
                          "h2d_bytes_per_step": {m: int(v) for m, v in h2d.items()}, **result}), flush=True)
        for m in pwrs:
            for pw in pwrs[m]:
                pw.close()
        marshalled = outs = coeffs = kinds = ys = runs = ents = roff = eoff = None
    ctx.close()


if __name__ == "__main__":
    main()

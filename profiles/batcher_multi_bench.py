"""The stream batcher over a mixed corpus: one batcher with several header sets (lwf_batcher_add_headers) against one
batcher per header set, submitted in turn.

Workload: five header sets of tests/vorbis_packer.py, --streams streams each, --packets long packets per stream and step
(~300 bytes per channel and packet): mono 256/2048, two stereo 256/2048 sets, stereo 1024/1024 and 6-channel 512/4096.
A decode server with one set of headers per quality, rate and channel layout meets this mix.
  multi      one batcher, every set added to it: one lwf_batcher_submit per step, whose entropy decode is one parallel
             pass over all jobs, then one batch per group (channels, blocksizes): four batches.
  separate   one batcher per header set (each with its own thread pool, sized to every host CPU): five lwf_batcher_submit
             calls per step, one after the other.
Both submit two deep: step k waits for the tickets of step k - 2 before it reuses that PCM arena.  The PCM goes to
page-locked host memory (host_f32) or to device memory (device_f32), for the dense residue entry and the VQ-record entry.
Each round runs back-to-back steps for at least --seconds; the ways alternate in one process.  Prints one JSON line with,
per entry, memory and way: ms per step, Gsamples/s (PCM samples of all channels), entropy seconds per step (summed over
the calls of a step) and the kernels launched per step, with the GPU's name and power limit and the host CPU count read in
the same run.  One step of each way on fresh streams is checked to give the same PCM, byte for byte.
Run from the repository root: python profiles/batcher_multi_bench.py"""
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

import torch  # noqa: E402

import lewton_b200 as L  # noqa: E402
import vorbis_packer as vp  # noqa: E402
from lewton_b200 import _cabi as cabi  # noqa: E402
from lewton_b200 import frontend as fe  # noqa: E402

# (seed, channels, blocksize_0, blocksize_1)
SETS = [(71, 1, 8, 11), (72, 2, 8, 11), (73, 2, 8, 11), (74, 2, 10, 10), (75, 6, 9, 12)]
MEMS = {"host_f32": cabi.MEM_HOST, "device_f32": cabi.MEM_DEVICE}


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=512, help="streams per header set")
    ap.add_argument("--packets", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=1.0, help="least duration of one round of one way")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    S, P = args.streams, args.packets
    lib = fe.lib()
    cabi.lib().lwb_bind_host_to_device(0)
    ctx = L.Context(0)
    corpus = []                 # (headers, channels, distinct long packets)
    for seed, ch, bs0, bs1 in SETS:
        rng = np.random.default_rng(seed)
        spec = vp.StreamSpec(rng, channels=ch, bs0=bs0, bs1=bs1, residue_types=[1, 2], cascade_p=0.12)
        hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        assert hdr.vq_capable()
        long_modes = [m for m, (b, _) in enumerate(spec.modes) if b]
        corpus.append((hdr, ch, [spec.audio_packet(int(rng.choice(long_modes)), 1, 1, p_unused=0.02)[0] for _ in range(32)]))
    stride = P * 2048                                   # the largest long block yields 2048 samples per channel
    offs, off = [], 0
    for _, ch, _ in corpus:
        offs.append([off + s * ch * stride for s in range(S)])
        off += S * ch * stride
    n_out = off

    def check(rc):
        ctx.check(rc)

    def packets(k, s):
        return [corpus[k][2][(s * 7 + i) % len(corpus[k][2])] for i in range(P)]

    result = {}
    for entry, ename in ((cabi.ENTRY_RESIDUE, "dense"), (cabi.ENTRY_VQ, "vq")):
        setups = [hdr.make_setup(ctx) for hdr, _, _ in corpus]
        multi = fe.StreamBatcher(ctx, corpus[0][0], entry=entry)
        for k in range(1, len(corpus)):
            multi.add_headers(corpus[k][0], setups[k])
        separate = [fe.StreamBatcher(ctx, hdr, entry=entry) for hdr, _, _ in corpus]

        def calls(way):
            """The (batcher, job array, packet arrays, n) of one step of `way`, on fresh streams."""
            pwrs = [[L.PreviousWindowRight(setups[k]) for _ in range(S)] for k in range(len(corpus))]
            groups = [[(pwrs[k][s], packets(k, s)) for s in range(S)] for k in range(len(corpus))]
            if way == "multi":
                parts = [(multi, [j for g in groups for j in g], [o for k in range(len(corpus)) for o in offs[k]])]
            else:
                parts = [(separate[k], groups[k], offs[k]) for k in range(len(corpus))]
            out = []
            for bt, jobs, o in parts:
                arr, keep, n = bt._jobs(jobs, stride)       # built once: per-step marshalling would be timed too
                for j in range(n):
                    arr[j].out_offset = o[j]
                out.append((bt, arr, keep, n))
            return pwrs, out

        for mname, mem in MEMS.items():
            if mem == cabi.MEM_HOST:
                outs = [ctx.host_alloc(n_out, np.float32) for _ in range(2)]
                addrs = [o.ctypes.data for o in outs]
            else:
                outs = [torch.empty(n_out, dtype=torch.float32, device="cuda") for _ in range(2)]
                addrs = [o.data_ptr() for o in outs]
            state = {way: calls(way) for way in ("multi", "separate")}

            def run(way, seconds):
                """Back-to-back steps for >= seconds: (steps, wall seconds, entropy seconds)."""
                steps, ent, last = 0, 0.0, []
                t = C.c_uint64()
                e, s = C.c_double(), C.c_double()
                t0 = time.perf_counter()
                while True:
                    if len(last) >= 2:
                        check(cabi.lib().lwb_ticket_wait(ctx._h, last[-2]))
                    for bt, arr, _, n in state[way][1]:
                        check(lib.lwf_batcher_submit(bt._h, arr, n, cabi.OUT_F32_PLANAR, addrs[steps % 2], mem, C.byref(t)))
                        lib.lwf_batcher_last_timing(bt._h, C.byref(e), C.byref(s))
                        ent += e.value
                    last.append(t.value)
                    steps += 1
                    if time.perf_counter() - t0 >= seconds:
                        break
                check(cabi.lib().lwb_ticket_wait(ctx._h, last[-1]))
                return steps, time.perf_counter() - t0, ent

            def step_samples(way):
                """PCM samples (all channels) of the last step of `way`; job j of a call is stream j % S of its set."""
                chs = [ch for _, ch, _ in corpus]
                total = 0
                for k, (_, arr, _, n) in enumerate(state[way][1]):
                    for j in range(n):
                        assert arr[j].status == 0 and arr[j].packets_done == P
                        total += arr[j].n_samples * chs[k if way == "separate" else j // S]
                return total

            for way in state:
                run(way, 0.3)               # warm-up: arenas, staging and streams in their steady state
            acc = {w: [0, 0.0, 0.0] for w in state}
            kernels = {w: {} for w in state}
            for _ in range(args.rounds):
                for way in state:
                    k0 = ctx.kernel_launches()
                    steps, wall, ent = run(way, args.seconds)
                    k1 = ctx.kernel_launches()
                    for name in k1:
                        kernels[way][name] = kernels[way].get(name, 0) + k1[name] - k0[name]
                    acc[way][0] += steps
                    acc[way][1] += wall
                    acc[way][2] += ent
            for way, (steps, wall, ent) in acc.items():
                total = step_samples(way)
                result[f"{ename}_{mname}_{way}"] = {
                    "ms_per_step": wall / steps * 1e3, "gsamples_per_s": total * steps / wall / 1e9,
                    "entropy_s_per_step": ent / steps,
                    "kernels_per_step": {n: round(v / steps, 2) for n, v in kernels[way].items() if v}, "steps": steps}
            # one step of each way on fresh streams into arena 0: the same PCM
            pcm = {}
            for way in state:
                if mem == cabi.MEM_HOST:
                    outs[0][:] = 0
                else:
                    outs[0].zero_()
                pwrs, parts = calls(way)
                t = C.c_uint64()
                for bt, arr, _, n in parts:
                    check(lib.lwf_batcher_submit(bt._h, arr, n, cabi.OUT_F32_PLANAR, addrs[0], mem, C.byref(t)))
                check(cabi.lib().lwb_ticket_wait(ctx._h, t.value))
                assert all(arr[j].status == 0 and arr[j].packets_done == P for _, arr, _, n in parts for j in range(n))
                pcm[way] = (outs[0].copy() if mem == cabi.MEM_HOST else outs[0].cpu().numpy())
                for ps in pwrs:
                    for p in ps:
                        p.close()
            assert np.array_equal(pcm["multi"].view(np.uint8), pcm["separate"].view(np.uint8)), f"{ename} {mname}: PCM differs"
            for way in state:
                for ps in state[way][0]:
                    for p in ps:
                        p.close()
        multi.close()
        for bt in separate:
            bt.close()
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "streams_per_set": S, "packets": P,
                      "host_cpus": os.cpu_count(), **result}))
    ctx.close()


if __name__ == "__main__":
    main()

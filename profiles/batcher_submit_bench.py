"""The stream batcher from packets to PCM: synchronous lwf_batcher_decode against lwf_batcher_submit two deep, with the
PCM in page-locked host memory or in device memory.

Workload: 2048 stereo streams x 16 long packets per step (packets of tests/vorbis_packer.py, ~300 bytes each, one set
of headers), for the dense residue entry and the VQ-record entry.  Each step runs one of these ways, in rounds that
alternate in one process:
  decode       lwf_batcher_decode into page-locked host f32 PCM; it returns once the PCM has landed.
  host_f32     lwf_batcher_submit into page-locked host f32 PCM, two arenas used in turn: step k waits for the ticket of
               step k - 2 before it reuses that arena, so the entropy decode of step k overlaps the GPU work of step k - 1.
  device_f32   the same into device memory: the PCM never crosses back to the host.
  device_f16   the same with f16 PCM.
Each round runs back-to-back steps for at least --seconds.  Prints one JSON line with, per entry and way: ms per step,
Gsamples/s (PCM samples of all channels), the entropy seconds and the hold per step (lwf_batcher_last_timing: for decode, its synthesis call;
for a submit, the arena-set wait, uploads and lwb_submit_chains), and the H2D and D2H bytes per packet, with the GPU's
name and power limit read in the same run.  The final PCM of every way is checked against decode's.
Run from the repository root: python profiles/batcher_submit_bench.py"""
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

WAYS = {"decode": (cabi.OUT_F32_PLANAR, np.float32, cabi.MEM_HOST), "host_f32": (cabi.OUT_F32_PLANAR, np.float32, cabi.MEM_HOST),
        "device_f32": (cabi.OUT_F32_PLANAR, torch.float32, cabi.MEM_DEVICE),
        "device_f16": (cabi.OUT_F16_PLANAR, torch.float16, cabi.MEM_DEVICE)}


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
    ap.add_argument("--streams", type=int, default=2048)
    ap.add_argument("--packets", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=1.0, help="least duration of one round of one way")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    S, P, Ch = args.streams, args.packets, 2
    lib = fe.lib()
    cabi.lib().lwb_bind_host_to_device(0)
    ctx = L.Context(0)
    rng = np.random.default_rng(77)
    spec = vp.StreamSpec(rng, channels=Ch, residue_types=[1, 2], cascade_p=0.12)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    assert hdr.vq_capable()
    long_modes = [m for m, (b, _) in enumerate(spec.modes) if b]
    distinct = [spec.audio_packet(int(rng.choice(long_modes)), 1, 1, p_unused=0.02)[0] for _ in range(64)]
    n_half = (1 << spec.bs1) // 2
    stride = P * n_half
    n_out = S * Ch * stride
    su = hdr.make_setup(ctx)

    def check(rc):
        ctx.check(rc)

    result = {}
    for entry, ename in ((cabi.ENTRY_RESIDUE, "dense"), (cabi.ENTRY_VQ, "vq")):
        bt = fe.StreamBatcher(ctx, hdr, entry=entry)
        state = {}
        for way, (fmt, dt, mem) in WAYS.items():
            pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
            jobs = [(pwrs[s], [distinct[(s * 7 + k) % len(distinct)] for k in range(P)]) for s in range(S)]
            arr, keep, n = bt._jobs(jobs, stride)          # built once: per-step marshalling of 2048 jobs would be timed too
            if mem == cabi.MEM_HOST:
                outs = [ctx.host_alloc(n_out, dt) for _ in range(1 if way == "decode" else 2)]
                addrs = [o.ctypes.data for o in outs]
            else:
                outs = [torch.empty(n_out, dtype=dt, device="cuda") for _ in range(2)]
                addrs = [o.data_ptr() for o in outs]
            state[way] = (pwrs, arr, keep, n, outs, addrs)

        def run(way, seconds):
            """Back-to-back steps for >= seconds: (steps, wall seconds, entropy seconds, rest of the calls' seconds)."""
            fmt, _, mem = WAYS[way]
            _, arr, _, n, _, addrs = state[way]
            steps, ent, rest, tickets = 0, 0.0, 0.0, []
            t = C.c_uint64()
            e, s = C.c_double(), C.c_double()
            t0 = time.perf_counter()
            while True:
                if way == "decode":
                    check(lib.lwf_batcher_decode(bt._h, arr, n, fmt, addrs[0]))
                else:
                    if len(tickets) >= 2:
                        check(cabi.lib().lwb_ticket_wait(ctx._h, tickets[-2]))
                    check(lib.lwf_batcher_submit(bt._h, arr, n, fmt, addrs[steps % 2], mem, C.byref(t)))
                    tickets.append(t.value)
                lib.lwf_batcher_last_timing(bt._h, C.byref(e), C.byref(s))
                ent += e.value
                rest += s.value
                steps += 1
                if time.perf_counter() - t0 >= seconds:
                    break
            if tickets:
                check(cabi.lib().lwb_ticket_wait(ctx._h, tickets[-1]))
            return steps, time.perf_counter() - t0, ent, rest

        for way in WAYS:
            run(way, 0.3)                   # warm-up: arenas, staging and streams in their steady state
        acc = {w: [0, 0.0, 0.0, 0.0] for w in WAYS}
        for _ in range(args.rounds):
            for way in WAYS:
                for i, v in enumerate(run(way, args.seconds)):
                    acc[way][i] += v
        # one more step each, into arena 0: what a step moves (the batch's inputs up, host PCM down) and its PCM
        h2d = {}
        for way in WAYS:
            run(way, 0.0)
            h2d[way] = lib.lwf_batcher_last_input_bytes(bt._h)
        _, arr, _, n, _, _ = state["decode"]
        samples = sum(arr[j].n_samples for j in range(n)) * Ch
        assert all(arr[j].status == 0 and arr[j].packets_done == P for j in range(n))
        want = state["decode"][4][0].view(np.uint8)
        for way, (fmt, dt, mem) in WAYS.items():
            last = state[way][4][0]
            got = last.cpu().numpy() if mem == cabi.MEM_DEVICE else last
            if fmt == cabi.OUT_F32_PLANAR:
                assert np.array_equal(got.view(np.uint8), want), f"{ename} {way}: PCM differs from decode's"
            else:
                ref = state["decode"][4][0].astype(np.float16)
                assert np.array_equal(got.view(np.uint16), ref.view(np.uint16)), f"{ename} {way}: f16 PCM differs"
        for way, (steps, wall, ent, rest) in acc.items():
            fmt, dt, mem = WAYS[way]
            esz = 2 if fmt == cabi.OUT_F16_PLANAR else 4
            result[f"{ename}_{way}"] = {
                "ms_per_step": wall / steps * 1e3, "gsamples_per_s": samples * steps / wall / 1e9,
                "entropy_s_per_step": ent / steps, "hold_s_per_step": rest / steps,
                "h2d_bytes_per_packet": h2d[way] / (S * P), "d2h_bytes_per_packet": samples * esz / (S * P) if mem == cabi.MEM_HOST else 0,
                "steps": steps}
        bt.close()
        for way in WAYS:
            for p in state[way][0]:
                p.close()
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "streams": S, "packets": P, "host_cpus": os.cpu_count(),
                      **result}))
    ctx.close()


if __name__ == "__main__":
    main()

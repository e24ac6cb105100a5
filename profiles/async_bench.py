"""Host-memory batches: synchronous lwb_decode_chains against lwb_submit_chains two deep.

Workload: bench.py's e2e shape at 4096 stereo streams x 16 long packets per step (spectrum entry, page-locked host
arenas), for f32 and i16 planar output.  Each step runs two ways, in rounds that alternate in one process:
  sync   lwb_decode_chains; it returns once the step's PCM has landed.
  async  lwb_submit_chains with two arena pairs used in turn: step k waits for the ticket of step k - 2 before it
         reuses that pair, so the H2D of one step overlaps the kernels and the D2H of the step before.
Each round runs back-to-back steps for at least --seconds.  Prints one JSON line: Msamples/s (PCM samples per second,
all channels) and host milliseconds per call (sync: the whole call; async: lwb_submit_chains alone, without the ticket
wait) for each mode and format, with the GPU's name and power limit read in the same run.  Run from the repository root: python profiles/async_bench.py"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import lewton_b200 as L  # noqa: E402
from lewton_b200 import _cabi as cabi  # noqa: E402
from lewton_b200.api import _marshal  # noqa: E402

N2 = 1024


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--packets", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=1.0, help="least duration of one round of one mode")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    S, P, Ch = args.streams, args.packets, 2
    lib = cabi.lib()
    lib.lwb_bind_host_to_device(0)
    ctx = L.Context(0)
    su = L.Setup(ctx, Ch, 8, 11, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(Ch)], [L.ModeInfo(False), L.ModeInfo(True)])
    stride = P * N2
    n_in, n_out = S * P * Ch * N2, S * Ch * stride
    spec = [ctx.host_alloc(n_in, np.float32) for _ in range(2)]
    spec[0][:] = (np.random.default_rng(99).standard_normal(n_in) * 1e-2).astype(np.float32)
    spec[1][:] = spec[0]
    outs = {fmt: [ctx.host_alloc(n_out, dt) for _ in range(2)]
            for fmt, dt in ((cabi.OUT_F32_PLANAR, np.float32), (cabi.OUT_I16_PLANAR, np.int16))}
    modes = np.ones(P, np.uint8)
    pwrs = {m: [L.PreviousWindowRight(su) for _ in range(S)] for m in ("sync", "async")}
    chains = {m: [L.ChainSpec(pwrs[m][s], modes, coeff_offset=s * P * Ch * N2, out_offset=s * Ch * stride, out_stride=stride)
                  for s in range(S)] for m in pwrs}
    # the lwb_chain arrays and io blocks, built once (per-step Python marshalling of 4096 chains would be timed too)
    marshalled = {}
    for m in pwrs:
        for fmt in outs:
            for k in range(2):
                marshalled[m, fmt, k] = _marshal(chains[m], cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, spec[k], outs[fmt][k], fmt,
                                                 None, None, None, cabi.MEM_HOST, None)

    def check(rc):
        if rc:
            raise L.AudioReadError(rc, lib.lwb_last_error(ctx._h).decode())

    def run(mode, fmt, seconds):
        """Back-to-back steps for >= seconds; returns (steps, wall seconds, host seconds inside the library calls)."""
        steps, host, t0 = 0, 0.0, time.perf_counter()
        tickets = []
        t = C.c_uint64()
        while True:
            arr, io = marshalled[mode, fmt, steps % 2]
            if mode == "sync":
                h0 = time.perf_counter()
                check(lib.lwb_decode_chains(ctx._h, arr, S, C.byref(io)))
            else:
                if len(tickets) >= 2:
                    check(lib.lwb_ticket_wait(ctx._h, tickets[-2]))
                h0 = time.perf_counter()            # (the submit alone: the wait above is time the caller may spend)
                check(lib.lwb_submit_chains(ctx._h, arr, S, C.byref(io), C.byref(t)))
                tickets.append(t.value)
            host += time.perf_counter() - h0
            steps += 1
            if time.perf_counter() - t0 >= seconds:
                break
        if tickets:
            check(lib.lwb_ticket_wait(ctx._h, tickets[-1]))
        return steps, time.perf_counter() - t0, host

    samples = S * P * Ch * N2
    result = {}
    for fmt, fname in ((cabi.OUT_F32_PLANAR, "f32"), (cabi.OUT_I16_PLANAR, "i16")):
        for mode in ("sync", "async"):
            run(mode, fmt, 0.2)                  # warm-up: arenas, staging, streams in their steady state
        acc = {m: [0, 0.0, 0.0] for m in ("sync", "async")}
        for _ in range(args.rounds):
            for mode in ("sync", "async"):
                steps, wall, host = run(mode, fmt, args.seconds)
                acc[mode][0] += steps
                acc[mode][1] += wall
                acc[mode][2] += host
        for mode, (steps, wall, host) in acc.items():
            result[f"{fname}_{mode}"] = {"msamples_per_s": samples * steps / wall / 1e6, "host_ms_per_call": host / steps * 1e3,
                                         "steps": steps, "seconds": wall}
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "streams": S, "packets": P, **result}))
    ctx.close()


if __name__ == "__main__":
    main()

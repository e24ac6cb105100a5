"""Checkpointing stream states: one stream at a time against lwb_streams_save / lwb_streams_load.

Workload: 4096 stereo streams after a long block (blocksizes 256 / 2048), so each holds [2][1024] f32 of state: 32 MiB
in all.  Measured three ways, in one process:
  per_stream  lwb_stream_export_state / lwb_stream_import_state for every stream into one page-locked buffer (each call
              synchronises); host clock around the 4096 calls.
  device      one lwb_streams_save / lwb_streams_load into device memory; CUDA events on the context's stream, around the
              call on an idle stream (host queuing included) and around its device work alone (queued behind a sleep).
  host        the same into page-locked host memory (staged in the context's arena, one copy of the extent).
GB/s is the 32 MiB of state over the call's time (a device copy also reads as many bytes as it writes).  Then the cost of
a checkpoint taken every step in async_bench.py's loop (4096 streams x 16 long packets, f32 planar, lwb_submit_chains two
deep on page-locked arenas): the loop with a device-memory lwb_streams_save after every submit, against the loop
without, in alternating rounds.  Prints one JSON line, with the GPU's name, power limit and SM clocks read in the same run,
and with --out FILE also writes it to FILE.  Run from the repository root: python profiles/state_bench.py"""
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
from lewton_b200.api import _marshal, _slot_array  # noqa: E402

N2 = 1024


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--packets", type=int, default=16, help="long packets per step of the checkpoint loop")
    ap.add_argument("--rounds", type=int, default=20, help="timed calls of each bulk measurement")
    ap.add_argument("--seconds", type=float, default=1.0, help="least duration of one round of the checkpoint loop")
    ap.add_argument("--out", help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    S, P, Ch = args.streams, args.packets, 2
    lib = cabi.lib()
    ctx = L.Context(0)
    su = L.Setup(ctx, Ch, 8, 11, [L.FloorTypeOne(1, [0, 128])], [L.Mapping(Ch)], [L.ModeInfo(False), L.ModeInfo(True)])

    def check(rc):
        if rc:
            raise L.AudioReadError(rc, lib.lwb_last_error(ctx._h).decode())

    pwrs = [L.PreviousWindowRight(su) for _ in range(S)]
    rng = np.random.default_rng(5)
    one = (rng.standard_normal(S * Ch * N2) * 1e-2).astype(np.float32)
    L.decode_chains(ctx, [L.ChainSpec(p, [1], coeff_offset=s * Ch * N2, out_offset=0, out_stride=1) for s, p in enumerate(pwrs)],
                    cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, one, np.zeros(Ch, np.float32), cabi.OUT_F32_PLANAR)
    assert all(len(p) == N2 for p in pwrs)
    state_bytes = S * Ch * N2 * 4
    offsets, total = L.state_offsets(pwrs)
    stream = torch.cuda.ExternalStream(ctx.cuda_stream, device=torch.device("cuda", 0))
    result = {"gpu_power_limit_clocks": gpu_info(), "streams": S, "state_mib": state_bytes / 2**20}

    # per stream: one export / import per stream, each synchronising
    host = ctx.host_alloc(total, np.float32)
    per = {"export": [], "import": []}
    for r in range(3):
        t0 = time.perf_counter()
        for s, p in enumerate(pwrs):
            check(lib.lwb_stream_export_state(p._h, host.ctypes.data + 4 * offsets[s]))
        t1 = time.perf_counter()
        for s, p in enumerate(pwrs):
            check(lib.lwb_stream_import_state(p._h, host.ctypes.data + 4 * offsets[s], N2))
        t2 = time.perf_counter()
        if r:                                   # round 0 warms up
            per["export"].append(t1 - t0)
            per["import"].append(t2 - t1)
    for k, v in per.items():
        ms = float(np.median(v)) * 1e3
        result[f"per_stream_{k}"] = {"ms_per_call": ms, "gb_per_s": state_bytes / (ms * 1e-3) / 1e9, "calls": S}

    # bulk, device and page-locked host memory: CUDA events around each call on the context's stream
    dev = torch.empty(total, dtype=torch.float32, device="cuda:0")
    torch.cuda.synchronize()
    t = C.c_uint64()
    slots = [L.StateSlot(p, o) for p, o in zip(pwrs, offsets)]
    for memory, mname, buf in ((cabi.MEM_DEVICE, "device", dev.data_ptr()), (cabi.MEM_HOST, "host", host.ctypes.data)):
        save_arr = _slot_array(slots)
        check(lib.lwb_streams_save(ctx._h, save_arr, S, memory, buf, C.byref(t)))
        check(lib.lwb_ctx_synchronize(ctx._h))
        load_arr = (cabi.StateSlot * S)()
        C.memmove(load_arr, save_arr, C.sizeof(save_arr))
        for kind, fn, arr in (("save", lib.lwb_streams_save, save_arr), ("load", lib.lwb_streams_load, load_arr)):
            # call: the events bracket the call on an idle stream, so the host's time to queue it counts too; gpu: the
            # stream is held behind a ~2 ms sleep while the call is queued, so only the device work is timed
            times = {"call": [], "gpu": []}
            for r in range(args.rounds + 3):
                for how in times:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    if how == "gpu":
                        with torch.cuda.stream(stream):
                            torch.cuda._sleep(4_000_000)
                    e0.record(stream)
                    check(fn(ctx._h, arr, S, memory, buf, C.byref(t)))
                    e1.record(stream)
                    check(lib.lwb_ticket_wait(ctx._h, t.value))
                    e1.synchronize()
                    if r >= 3:
                        times[how].append(e0.elapsed_time(e1))
            for how, v in times.items():
                ms = float(np.median(v))
                result[f"bulk_{mname}_{kind}_{how}"] = {"ms_per_call": ms, "min_ms": float(np.min(v)), "gb_per_s": state_bytes / (ms * 1e-3) / 1e9,
                                                        "rounds": len(v)}
    # the round trips above left every state as it was
    check(lib.lwb_ctx_synchronize(ctx._h))
    assert all(len(p) == N2 and not p.is_empty() for p in pwrs)

    # a checkpoint every step of the two-deep submit loop
    stride = P * N2
    n_in, n_out = S * P * Ch * N2, S * Ch * stride
    spec = [ctx.host_alloc(n_in, np.float32) for _ in range(2)]
    spec[0][:] = (rng.standard_normal(n_in) * 1e-2).astype(np.float32)
    spec[1][:] = spec[0]
    outs = [ctx.host_alloc(n_out, np.float32) for _ in range(2)]
    modes = np.ones(P, np.uint8)
    chains = [L.ChainSpec(pwrs[s], modes, coeff_offset=s * P * Ch * N2, out_offset=s * Ch * stride, out_stride=stride) for s in range(S)]
    marshalled = [_marshal(chains, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, spec[k], outs[k], cabi.OUT_F32_PLANAR, None, None, None,
                           cabi.MEM_HOST, None) for k in range(2)]
    ck = [torch.empty(total, dtype=torch.float32, device="cuda:0") for _ in range(2)]
    ck_arr = _slot_array(slots)
    torch.cuda.synchronize()

    def run(checkpoint, seconds):
        steps, tickets, t0 = 0, [], time.perf_counter()
        while True:
            arr, io = marshalled[steps % 2]
            if len(tickets) >= 2:
                check(lib.lwb_ticket_wait(ctx._h, tickets[-2]))
            check(lib.lwb_submit_chains(ctx._h, arr, S, C.byref(io), C.byref(t)))
            if checkpoint:                       # the states this step leaves, into the older of two checkpoint buffers
                check(lib.lwb_streams_save(ctx._h, ck_arr, S, cabi.MEM_DEVICE, ck[steps % 2].data_ptr(), C.byref(t)))
            tickets.append(t.value)
            steps += 1
            if time.perf_counter() - t0 >= seconds:
                break
        check(lib.lwb_ticket_wait(ctx._h, tickets[-1]))
        return steps, time.perf_counter() - t0

    for c in (False, True):
        run(c, 0.3)
    acc = {False: [0, 0.0], True: [0, 0.0]}
    for _ in range(3):
        for c in (False, True):
            steps, wall = run(c, args.seconds)
            acc[c][0] += steps
            acc[c][1] += wall
    samples = S * P * Ch * N2
    for c, (steps, wall) in acc.items():
        result["loop_with_checkpoint" if c else "loop_without_checkpoint"] = {"ms_per_step": wall / steps * 1e3,
                                                                             "msamples_per_s": samples * steps / wall / 1e6, "steps": steps}
    result["checkpoint_cost_pct"] = (result["loop_with_checkpoint"]["ms_per_step"] / result["loop_without_checkpoint"]["ms_per_step"] - 1) * 100
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()

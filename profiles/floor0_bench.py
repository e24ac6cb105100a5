#!/usr/bin/env python3
"""Floor-0 streams through the host front half and the batched synthesis (lwf_batcher), with floor-0 curves rendered on
the host and sent dense (LWB_FLOOR_DENSE) against floor-0 records rendered on the device (LWB_FLOOR_ZERO,
StreamBatcher(floor0=True)), for the residue and the VQ entries.  The packets are Vorbis audio packets made by
tests/vorbis_packer.py: stereo, a type-0 floor on every channel, long blocks.  FLOOR0_STREAMS streams x 16 packets
(default 2048), host pinned memory in and out.

One JSON line per case: the bytes handed to the device per packet (lwf_batcher_last_input_bytes), host entropy-decode
seconds per packet (the pool's wall time over the packets), and Msamples/s of the whole call (entropy + synthesis +
copies).  Device-memory batches are not part of the batcher and are not measured here."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def floor0_stream():
    """A stereo packer stream whose channels all use its type-0 floor in a long mode, and that qualifies for VQ."""
    import vorbis_packer as vp
    from lewton_b200 import frontend as fe
    for seed in range(200):
        rng = np.random.default_rng(seed)
        spec = vp.StreamSpec(rng, channels=2, floor0=True, residue_types=[2], n_modes=2)
        hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        long_modes = [i for i, (bf, _) in enumerate(spec.modes) if bf]
        mp = spec.mappings[spec.modes[long_modes[0]][1]]
        if hdr.vq_capable() and all(isinstance(spec.floors[mp["floors"][mp["mux"][c]]], vp.Floor0) for c in range(2)):
            return spec, hdr, long_modes[0]
    raise RuntimeError("no stereo floor-0 stream found")


def main():
    import lewton_b200 as L
    from lewton_b200 import _cabi as cabi
    from lewton_b200 import frontend as fe

    S, P, D = int(os.environ.get("FLOOR0_STREAMS", 2048)), 16, 64
    cabi.lib().lwb_bind_host_to_device(0)
    ctx = L.Context(0)
    spec, hdr, mode = floor0_stream()
    dist = [spec.audio_packet(mode, 1, 1, p_unused=0.0)[0] for _ in range(D)]
    pick = np.random.default_rng(5).integers(0, D, (S, P))
    n = 1 << spec.bs1
    stride = P * n
    samples = S * (P - 1) * n                            # 2 channels x n/2 per packet after each stream's first
    pcm = np.asarray(ctx.host_alloc((S * 2 * stride,), np.float32))
    ref = {}
    for entry_name, entry in (("residue", cabi.ENTRY_RESIDUE), ("vq", cabi.ENTRY_VQ)):
        for records in (False, True):
            su = hdr.make_setup(ctx, floor0=records)
            b = fe.StreamBatcher(ctx, hdr, threads=0, entry=entry, floor0=records)
            pw = [L.PreviousWindowRight(su) for _ in range(S)]
            jobs = [(pw[s], [dist[d] for d in pick[s]]) for s in range(S)]
            b.decode(jobs, pcm, stride)                  # warm-up (arenas, module load)
            times, ent = [], []
            k0 = ctx.kernel_launches()
            for _ in range(5):
                for p in pw:
                    p.reset()
                t0 = time.perf_counter()
                res = b.run(pcm)
                times.append(time.perf_counter() - t0)
                ent.append(b.entropy_seconds)
            assert all(r[2] == 0 for r in res)
            key = entry_name
            if records:
                assert pcm.tobytes() == ref[key], "records and dense curves decoded differently"
            else:
                ref[key] = pcm.tobytes()
            sec = float(np.median(times))
            print(json.dumps({"case": f"{entry_name}_{'records' if records else 'dense'}", "streams": S, "packets_per_stream": P,
                              "blocksize": n, "h2d_bytes_per_packet": b.input_bytes / (S * P),
                              "host_entropy_us_per_packet": float(np.median(ent)) / (S * P) * 1e6,
                              "ms_per_call": sec * 1e3, "msamples_per_s": samples / sec / 1e6,
                              "launches": {k: v - k0[k] for k, v in ctx.kernel_launches().items() if v - k0[k]},
                              "memory": "host pinned in and out (device memory: not measured)"}), flush=True)
            b.close()
            for p in pw:
                p.close()
            su.close()
    gpu = os.popen("nvidia-smi --query-gpu=name,power.limit --format=csv,noheader").read().strip()
    print(json.dumps({"gpu": gpu}))
    ctx.close()


if __name__ == "__main__":
    main()

"""Worker for tests/test_stream_states_gpu.py's migrate_streams tests: run under torch.distributed.run with two ranks and
the backend named by argv[1] (gloo: both ranks on GPU 0, each with its own context; nccl: rank r on GPU r).

Every rank builds the same random packets.  Rank 0 decodes the first part of all streams, migrate_streams moves the
second half of them to rank 1, each rank decodes the rest of its streams, and rank 0 checks every stream's PCM, the
migrated ones' from rank 1 included, against the oracle run straight through."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import lewton_b200 as L  # noqa: E402
from helpers import bits_equal, mismatch_report  # noqa: E402
from lewton_b200.sharding import _p2p, migrate_streams  # noqa: E402
from oracle import oracle  # noqa: E402
from test_stream_states_gpu import SPECTRUM, Track, decode, setup_of  # noqa: E402

NAME, S, P1, P2 = "stereo_256_2048", 8, 3, 4


def main():
    backend = sys.argv[1]
    dist.init_process_group(backend)
    rank = dist.get_rank()
    device = rank if backend == "nccl" else 0
    torch.cuda.set_device(device)
    oracle.build()
    rng = np.random.default_rng(77)
    tracks = [Track(oracle, rng, NAME, SPECTRUM, P1 + P2 + k % 3) for k in range(S)]
    ctx = L.Context(device)
    moved = list(range(S // 2, S))
    if rank == 0:
        su = setup_of(ctx, NAME)
        pwrs = [L.PreviousWindowRight(su) for _ in tracks]
        first = decode(ctx, [(p, t, 0, P1) for p, t in zip(pwrs, tracks)], SPECTRUM)
        for got, tr in zip(first, tracks):
            assert bits_equal(got, tr.want_pcm(0, P1)), mismatch_report(got, tr.want_pcm(0, P1))
        migrate_streams(ctx, 0, 1, pwrs=[pwrs[k] for k in moved])
        for k in moved:
            pwrs[k].close()
        mine = {k: pwrs[k] for k in range(S) if k not in moved}
    else:
        su = setup_of(ctx, NAME)
        new = migrate_streams(ctx, 0, 1, setups=[su] * len(moved))
        mine = dict(zip(moved, new))
    keys = sorted(mine)
    rest = decode(ctx, [(mine[k], tracks[k], P1, len(tracks[k].packets)) for k in keys], SPECTRUM)
    # rank 1's PCM goes to rank 0, in one flat f32 transfer of known size
    dev = torch.device("cuda", device) if backend == "nccl" else torch.device("cpu")
    if rank == 1:
        _p2p([dist.P2POp(dist.isend, torch.from_numpy(np.concatenate([r.ravel() for r in rest])).to(dev), 0)])
    else:
        sizes = [tracks[k].want_pcm(P1, len(tracks[k].packets)).size for k in moved]
        flat = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        _p2p([dist.P2POp(dist.irecv, flat, 1)])
        flat = flat.cpu().numpy()
        got = dict(zip(keys, rest))
        off = 0
        for k, n in zip(moved, sizes):
            got[k] = flat[off: off + n].reshape(2, -1)
            off += n
        for k in range(S):
            want = tracks[k].want_pcm(P1, len(tracks[k].packets))
            assert bits_equal(got[k], want), (k, mismatch_report(got[k], want))
    for k in keys:
        assert bits_equal(mine[k].data(), tracks[k].end_state), k
    dist.barrier()
    if rank == 0:
        print(f"MIGRATE_OK {backend}")
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

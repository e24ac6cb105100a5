"""Stream sharding for multi-GPU runs (SURVEY.md section 8e).

The synthesis path has no cross-stream dependency: the only couplings are packet k <-> k+1 of one
stream (overlap-add) and the channels of one packet (inverse coupling), so streams are partitioned
by contiguous ranges over the ranks and the COMPUTE needs no collective.  When a batch originates and
terminates on one rank (a front end that entropy-decodes on one socket, a sink that wants all PCM in one
place), the batch is scattered and the PCM gathered over NVLink with grouped NCCL send / receive
(`scatter_streams` / `gather_streams`: torch.distributed's batch_isend_irecv = ncclGroupStart ..
ncclSend / ncclRecv .. ncclGroupEnd) -- the only NCCL traffic of the path, timed separately by bench.py."""


def stream_range(n_streams, world_size, rank):
    """Contiguous, balanced [lo, hi) of the streams rank `rank` owns (sizes differ by at most 1)."""
    if not (0 <= rank < world_size) or n_streams < 0:
        raise ValueError("bad rank / world size / stream count")
    base, extra = divmod(n_streams, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def owner_of(stream, n_streams, world_size):
    """Rank that owns `stream` under stream_range."""
    base, extra = divmod(n_streams, world_size)
    cut = extra * (base + 1)
    if stream < cut:
        return stream // (base + 1)
    return extra + (stream - cut) // base if base else world_size - 1


def _p2p(ops):
    import torch.distributed as dist
    if not ops:
        return
    if dist.get_backend() == "nccl":
        for w in dist.batch_isend_irecv(ops):      # one ncclGroupStart/End around all sends and receives
            w.wait()
    else:                                          # gloo (CPU tests): the same transfers one by one
        for w in [op.op(op.tensor, op.peer) for op in ops]:
            w.wait()


def scatter_streams(root_tensor, local_tensor, n_streams, root=0):
    """Rows [lo, hi) = stream_range(n_streams, world, rank) of `root_tensor` (first dimension = streams, present on
    `root` only) land in `local_tensor` on every rank.  Grouped point-to-point: the root sends each peer its slice."""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    if rank == root:
        ops = []
        for r in range(world):
            lo, hi = stream_range(n_streams, world, r)
            if r == root:
                local_tensor.copy_(root_tensor[lo:hi])
            elif hi > lo:
                ops.append(dist.P2POp(dist.isend, root_tensor[lo:hi], r))
        _p2p(ops)
    else:
        lo, hi = stream_range(n_streams, world, rank)
        if hi > lo:
            _p2p([dist.P2POp(dist.irecv, local_tensor, root)])


def gather_streams(local_tensor, root_tensor, n_streams, root=0):
    """Inverse of scatter_streams: every rank's rows return to their place in `root_tensor` on `root`."""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    if rank == root:
        ops = []
        for r in range(world):
            lo, hi = stream_range(n_streams, world, r)
            if r == root:
                root_tensor[lo:hi].copy_(local_tensor)
            elif hi > lo:
                ops.append(dist.P2POp(dist.irecv, root_tensor[lo:hi], r))
        _p2p(ops)
    else:
        lo, hi = stream_range(n_streams, world, rank)
        if hi > lo:
            _p2p([dist.P2POp(dist.isend, local_tensor, root)])


def migrate_streams(ctx, src, dst, pwrs=(), setups=()):
    """Moves live streams from rank `src` to rank `dst` mid-decode, without a gap or a changed sample: a long-lived server
    rebalances its ranks, or hands a context's streams over before it goes.  Both ranks call it; any other rank returns []
    at once.  ctx: this rank's Context.
      src: pwrs are the streams to move, in order, called after the batches that decoded them so far have been queued.
        Their states are saved in one call (Context.save_states) and waited for; the streams may be closed afterwards.
        Returns [].
      dst: setups holds one Setup of ctx per stream, in the same order, each with the channel count of the stream it
        receives and a blocksize_1 whose half holds its state.  Returns the new streams, loaded (Context.load_states): the
        next batch queued on ctx decodes from them exactly as the source streams would have.
    The state buffer crosses with its slot metadata in grouped point-to-point transfers, as scatter_streams' rows do: in
    device memory over NCCL, in page-locked host memory over gloo."""
    import numpy as np
    import torch
    import torch.distributed as dist

    from . import _cabi as cabi
    from .api import PreviousWindowRight, StateSlot, state_offsets
    rank = dist.get_rank()
    if rank not in (src, dst) or src == dst:
        return []
    nccl = dist.get_backend() == "nccl"
    dev = torch.device("cuda", ctx.device) if nccl else torch.device("cpu")
    memory = cabi.MEM_DEVICE if nccl else cabi.MEM_HOST

    def state_buffer(n):
        if nccl:
            return torch.empty(max(n, 1), dtype=torch.float32, device=dev)
        return torch.from_numpy(ctx.host_alloc(max(n, 1), np.float32))

    if rank == src:
        pwrs = list(pwrs)
        offsets, total = state_offsets(pwrs)
        buf = state_buffer(total)
        slots, ticket = ctx.save_states(pwrs, buf, memory, offsets)
        ticket.wait()                         # the transfers below run on torch's streams, not on ctx's
        meta = torch.tensor([[s.offset, s.len, int(s.has)] for s in slots] or [[0, 0, 0]], dtype=torch.int64, device=dev)
        _p2p([dist.P2POp(dist.isend, torch.tensor([len(slots), total], dtype=torch.int64, device=dev), dst)])
        _p2p([dist.P2POp(dist.isend, meta, dst), dist.P2POp(dist.isend, buf, dst)])
        return []
    setups = list(setups)
    head = torch.zeros(2, dtype=torch.int64, device=dev)
    _p2p([dist.P2POp(dist.irecv, head, src)])
    n, total = (int(v) for v in head.tolist())
    if n != len(setups):
        raise ValueError(f"migrate_streams: rank {src} sends {n} streams, rank {dst} has {len(setups)} setups for them")
    meta = torch.zeros((max(n, 1), 3), dtype=torch.int64, device=dev)
    buf = state_buffer(total)
    _p2p([dist.P2POp(dist.irecv, meta, src), dist.P2POp(dist.irecv, buf, src)])
    if nccl:
        torch.cuda.current_stream(dev).synchronize()      # the load runs on ctx's stream
    new = [PreviousWindowRight(su) for su in setups]
    slots = [StateSlot(p, o, ln, h) for p, (o, ln, h) in zip(new, meta.tolist())]
    ctx.load_states(slots, buf, memory).wait()
    return new

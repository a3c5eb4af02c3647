"""Multi-GPU layout of a stream batch: contiguous blocks of streams per rank, no data-path collective.

Streams never interact and their state stays resident on the GPU that owns them (SURVEY.md 8(e)), so the only traffic
between ranks is I/O when a deployment has a single ingest point: rank `src` scatters int16[N][640] PCM rows and gathers
uint8[N][cap] payloads + int16[N][2] length fields (decoder: the mirror image).  Both are grouped point-to-point
transfers (ncclSend/ncclRecv under the "nccl" backend, i.e. NVLink 5 / NVSwitch peer copies; "gloo" on CPU for tests).
Ranks that ingest their own streams (the layout bench.py times) never call into this module.

Two ways to serve a single ingest point:
  * scatter_streams / gather_streams -- explicit transfers before / after the codec kernels (NCCL point-to-point);
  * share_from_root                  -- no transfer step at all: the root's device buffers are mapped into every rank (CUDA
    IPC) and handed to the *_device entry points as they are; the band-split kernel pulls its PCM rows over NVLink and the
    entropy-coding / decoder kernels push their rows back (`solo_b200_enable_peer_access`)."""
import torch
import torch.distributed as dist


def _bytes(t):
    """Raw byte view of a contiguous tensor: NCCL has no int16 type, and these transfers are plain byte moves anyway."""
    return t.view(torch.uint8)


def _run(ops):
    """Post the point-to-point operations of one scatter / gather, one dist.send / dist.recv each (asynchronous on NCCL's
    stream, so the transfers to different peers still overlap).  The grouped form (dist.batch_isend_irecv,
    SOLO_B200_P2P=grouped) was far slower than separate sends in an earlier measurement; neither has been timed on H100."""
    import os
    if not ops:
        return
    if os.environ.get("SOLO_B200_P2P") == "grouped":
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        return
    for op in ops:
        (dist.send if op.op is dist.isend else dist.recv)(op.tensor, op.peer, group=op.group)


def shard_bounds(n_streams, world):
    """[(lo, hi)) per rank: rank r owns streams r*N//W .. (r+1)*N//W (contiguous so every transfer is one message)."""
    return [(r * n_streams // world, (r + 1) * n_streams // world) for r in range(world)]


def local_count(n_streams, rank, world):
    lo, hi = shard_bounds(n_streams, world)[rank]
    return hi - lo


def scatter_streams(full, n_streams, row_shape, dtype, device, src=0, group=None):
    """Rank `src` passes `full` = tensor [N, *row_shape]; every rank (src included) gets its own rows [n_local, *row_shape]."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    bounds = shard_bounds(n_streams, world)
    lo, hi = bounds[rank]
    out = torch.empty((hi - lo,) + tuple(row_shape), dtype=dtype, device=device)
    ops = []
    if rank == src:
        assert full.shape[0] == n_streams and full.dtype == dtype
        for r, (a, b) in enumerate(bounds):
            if r == src:
                out.copy_(full[a:b])
            elif b > a:
                ops.append(dist.P2POp(dist.isend, _bytes(full[a:b].contiguous()), r, group))
    elif hi > lo:
        ops.append(dist.P2POp(dist.irecv, _bytes(out), src, group))
    _run(ops)
    return out


def gather_streams(local, n_streams, dst=0, group=None):
    """Inverse of scatter_streams: rank `dst` returns [N, *row_shape], the others None."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    bounds = shard_bounds(n_streams, world)
    lo, hi = bounds[rank]
    assert local.shape[0] == hi - lo
    ops = []
    full = None
    if rank == dst:
        full = torch.empty((n_streams,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        full[lo:hi].copy_(local)
        for r, (a, b) in enumerate(bounds):
            if r != dst and b > a:
                ops.append(dist.P2POp(dist.irecv, _bytes(full[a:b]), r, group))
    elif hi > lo:
        ops.append(dist.P2POp(dist.isend, _bytes(local.contiguous()), dst, group))
    _run(ops)
    return full


def share_from_root(t, src=0, group=None):
    """Rank `src` passes a CUDA tensor; every rank returns a tensor that aliases the root's memory (the root: the tensor
    itself).  Kernels of the local GPU reach it through NVLink / NVSwitch peer access, which this call enables."""
    from torch.multiprocessing.reductions import reduce_tensor
    import solo_b200
    rank = dist.get_rank(group)
    box = [None]
    if rank == src:
        fn, args = reduce_tensor(t)
        box = [(fn, args, t.device.index)]
    dist.broadcast_object_list(box, src=src, group=group)
    fn, args, root_dev = box[0]
    local = torch.cuda.current_device()
    if rank == src:
        return t
    solo_b200.enable_peer_access(local, root_dev)
    # open the IPC handle from the LOCAL device: cudaIpcOpenMemHandle then sets up (lazy) peer access between this GPU and
    # the exporting one, and the returned addresses are valid in kernels of the local GPU.  (torch would open it under the
    # exporter's ordinal; index 6 of the rebuild arguments is that ordinal.)
    args = list(args)
    args[6] = local
    peer = fn(*args)
    torch.cuda.set_device(local)
    return peer

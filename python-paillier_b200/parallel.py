"""Multi-GPU plumbing: one process per GPU (torchrun), batches shard by contiguous row ranges.

The hot path has no exchange step -- every element is independent -- so the only
collectives are (1) a broadcast of the key limbs from rank 0 and (2) an optional all-gather of result
limbs when a caller wants the whole vector on every rank.  NCCL on GPUs, gloo in the CPU tests.
"""
import numpy as np

from .engine import ints_to_limbs, limbs_to_ints


def shard_range(batch, rank, world):
    """Rows [lo, hi) of a batch owned by `rank`: contiguous, sizes differ by at most one."""
    base, extra = divmod(batch, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def broadcast_ints(values, limbs, src=0, device=None):
    """Broadcast a list of big integers (e.g. n, p, q) from `src` as a [len, limbs] limb matrix."""
    import torch
    import torch.distributed as dist
    arr = ints_to_limbs(values, limbs).view(np.int32).copy()
    t = torch.from_numpy(arr)
    if device is not None:
        t = t.to(device)
    dist.broadcast(t, src)
    return limbs_to_ints(t.cpu().numpy().view(np.uint32))


def all_gather_rows(local_rows, batch):
    """All-gather row shards (torch int32 tensor [rows_r, L], contiguous split of `batch`) into the full
    [batch, L] matrix on every rank.  Shards are padded to the largest shard for the collective."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    sizes = [shard_range(batch, r, world) for r in range(world)]
    maxrows = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros((maxrows, local_rows.shape[1]), dtype=local_rows.dtype, device=local_rows.device)
    pad[: local_rows.shape[0]] = local_rows
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad)
    return torch.cat([o[: hi - lo] for o, (lo, hi) in zip(out, sizes)], dim=0)

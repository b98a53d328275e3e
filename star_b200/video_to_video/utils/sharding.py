"""Work split over the ranks of a torch.distributed job (one process per GPU) and the all-gathers that reassemble it."""
import torch
import torch.distributed as dist


def _dist_info():
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def _shard_bounds(n, world):
    """contiguous, balanced split of n items over `world` ranks: [(lo, hi)] (empty shards when n < world)"""
    base, extra = divmod(n, world)
    out, lo = [], 0
    for r in range(world):
        hi = lo + base + (1 if r < extra else 0)
        out.append((lo, hi))
        lo = hi
    return out


def _all_gather_varlen(local, counts, dim):
    """all-gather of per-rank tensors whose extent along `dim` is counts[rank] (padded to the longest share);
    returns the concatenation in rank order.  ONE collective."""
    world, rank = _dist_info()
    pad = max(counts)
    shape = list(local.shape)
    shape[dim] = pad
    send = local.new_zeros(shape)
    if counts[rank]:
        send.narrow(dim, 0, counts[rank]).copy_(local)
    recv = [torch.empty_like(send) for _ in range(world)]
    dist.all_gather(recv, send)
    return torch.cat([recv[r].narrow(dim, 0, counts[r]) for r in range(world) if counts[r]], dim=dim)


def _all_gather_owned(local, sizes, dim):
    """all-gather of items owned round-robin: item i, of extent sizes[i] along `dim`, is on rank i % world, and `local`
    is this rank's items concatenated in item order (extent 0 when it owns none; every rank passes the same dtype).
    Returns all items concatenated in item order.  ONE collective."""
    world, _ = _dist_info()
    order = [i for r in range(world) for i in range(r, len(sizes), world)]          # rank-major, as the gather returns them
    gathered = _all_gather_varlen(local, [sum(sizes[r::world]) for r in range(world)], dim)
    item = dict(zip(order, gathered.split([sizes[i] for i in order], dim=dim)))
    return torch.cat([item[i] for i in range(len(sizes))], dim=dim)

"""Batch sharding for multi-GPU inference (SURVEY.md §8e): one process per GPU, each rank runs an independent replica
on its slice of the batch; there is NO collective on the data path (pairs are independent, evaluate.py:121-131).
The only communication is the optional gather of results and the max-over-ranks reduction of timings.

Replaces the reference's single-process nn.DataParallel scatter/gather (evaluate.py:246-252, train.py:175).
"""
import torch
import torch.distributed as dist


def shard_range(n, world, rank):
    """Contiguous, balanced slice [lo, hi) of n items for `rank` of `world` (first n % world ranks get one extra)."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad world/rank")
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def world_rank():
    """(world size, rank) of the initialised process group, or (1, 0)."""
    if dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def strided_items(items, world, rank):
    """The items of index = rank (mod world), in order (validate's samples, create_kitti_submission's pairs).  A sequence (len
    and indexing, such as the reference's FlowDataset) is indexed, so only this rank's items are loaded; any other iterable is
    walked and filtered."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad world/rank")
    if world == 1:
        return iter(items)
    if hasattr(items, "__len__") and hasattr(items, "__getitem__") and not isinstance(items, dict):
        return (items[i] for i in range(rank, len(items), world))
    return (it for i, it in enumerate(items) if i % world == rank)


def greedy_assignment(sizes, world):
    """Rank of each item for `world` ranks by longest-first greedy on `sizes` (create_sintel_submission: whole sequences by pair
    count): items in decreasing size, ties by index, each to the least loaded rank, ties to the lowest rank."""
    if world <= 0:
        raise ValueError("bad world")
    load = [0] * world
    owner = [0] * len(sizes)
    for i in sorted(range(len(sizes)), key=lambda i: (-sizes[i], i)):
        r = min(range(world), key=lambda r: (load[r], r))
        owner[i] = r
        load[r] += sizes[i]
    return owner


def gather_strided(local, world):
    """Every rank's list of `local` objects (rank r's holding the items of index = r (mod world), in order), all-gathered and
    interleaved back into the global order.  Returns `local` itself at world 1."""
    if world == 1:
        return local
    parts = [None] * world
    dist.all_gather_object(parts, local)
    out = []
    for k in range(max(len(p) for p in parts)):
        out.extend(p[k] for p in parts if k < len(p))
    return out


def barrier():
    """dist.barrier() when more than one rank runs."""
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()


def infer_sharded(fn, image1, image2, gather=True, **kw):
    """Run `fn(image1_shard, image2_shard, **kw) -> (flow_low, flow_up)` on this rank's slice of the batch.
    With gather=True every rank returns the full-batch results (all_gather of the per-rank outputs, padded to the
    largest shard); otherwise only the local shard is returned."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    n = image1.shape[0]
    lo, hi = shard_range(n, world, rank)
    outs = fn(image1[lo:hi], image2[lo:hi], **kw) if hi > lo else None
    if world == 1 or not gather:
        return outs
    sizes = [shard_range(n, world, r) for r in range(world)]
    cap = max(h - l for l, h in sizes)
    # every rank needs the output shapes even if its own shard is empty
    meta = [None] * world
    dist.all_gather_object(meta, None if outs is None else [tuple(o.shape[1:]) for o in outs])
    shapes = next(m for m in meta if m is not None)
    ref = outs[0] if outs is not None else None
    device = ref.device if ref is not None else image1.device
    full = []
    for i, shp in enumerate(shapes):
        pad = torch.zeros((cap,) + tuple(shp), dtype=torch.float32, device=device)
        if outs is not None:
            pad[: hi - lo] = outs[i]
        parts = [torch.empty_like(pad) for _ in range(world)]
        dist.all_gather(parts, pad)
        full.append(torch.cat([parts[r][: sizes[r][1] - sizes[r][0]] for r in range(world)], 0))
    return tuple(full)


def max_over_ranks(value, device="cpu"):
    """Max over ranks of a host float (device timings are reported as the slowest rank's)."""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()

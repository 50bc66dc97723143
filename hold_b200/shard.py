"""Multi-GPU partitioning of the path (SURVEY.md §8e): rays/frames are independent units, so ranks take disjoint
ray ranges with NO data-path collective (render.py has no gradients, SURVEY D4).  Shards are aligned to the
reference's 512-pixel render chunks (datasets/eval_datasets.py:13) so that a sharded render reproduces the
reference's own chunked semantics of the batch-global sampler flag (engine/ray_sampler.py:244)."""
from __future__ import annotations


def shard_range(n: int, rank: int, world: int, align: int = 512) -> tuple[int, int]:
    """[start, stop) of `n` units for `rank` of `world`, boundaries on multiples of `align` (last shard takes the tail)."""
    assert 0 <= rank < world and n >= 0 and align >= 1
    blocks = (n + align - 1) // align
    per, rem = divmod(blocks, world)
    b0 = rank * per + min(rank, rem)
    b1 = b0 + per + (1 if rank < rem else 0)
    return min(b0 * align, n), min(b1 * align, n)


def shard_frames(n_frames: int, rank: int, world: int) -> list[int]:
    """Round-robin frames, the reference's own `--agent_id` farming idea (datasets/eval_datasets.py:43-50)."""
    return list(range(rank, n_frames, world))


def allreduce_flat_(tensors, group=None, average: bool = False):
    """ONE all-reduce (sum) over a single flat bucket holding every tensor of `tensors` — the "single NCCL all-reduce on
    gradients per step" of the north star / SURVEY §8e for data-parallel steps (frame-sharded pose refinement,
    optimize_ckpt.py: shared parameters — betas, scene_scale, obj_scale — receive gradient terms from every rank's frames;
    per-frame parameters stay local).  In place; `None` entries are skipped.  Backend-agnostic plumbing
    (torch.distributed: nccl on GPUs, gloo in the CPU tests)."""
    import torch
    import torch.distributed as dist

    ts = [t for t in tensors if t is not None]
    if not ts or not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return tensors
    flat = torch.cat([t.reshape(-1).to(torch.float32) for t in ts])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    if average:
        flat /= dist.get_world_size(group)
    o = 0
    for t in ts:
        n = t.numel()
        t.copy_(flat[o:o + n].view_as(t))
        o += n
    return tensors


def allreduce_grads_(params, group=None, average: bool = False):
    """`allreduce_flat_` over the `.grad` of `params` — ALL of them, in the given (rank-invariant) order: a parameter without a
    gradient on this rank (e.g. a node none of this rank's rays hit) contributes zeros and receives the sum, so that the bucket has
    the same layout on every rank (ranks that disagreed on which gradients exist would otherwise reduce mismatched buckets)."""
    import torch

    params = [p for p in params if p.requires_grad]
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
    allreduce_flat_([p.grad for p in params], group=group, average=average)


def gather_rays(local, n_total: int, rank: int, world: int, align: int = 512, group=None, dst: int = 0):
    """Assemble a per-ray output ([n_local, ...] on every rank, shards from `shard_range`) on rank `dst`: the only
    collective of a sharded render, and only for image assembly (SURVEY §8e).  Returns the full [n_total, ...] tensor on
    `dst`, None elsewhere."""
    import torch
    import torch.distributed as dist

    if world == 1:
        return local
    sizes = [shard_range(n_total, r, world, align) for r in range(world)]
    pad = max(e - s for s, e in sizes)
    buf = torch.zeros((pad,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    buf[: local.shape[0]] = local
    out = [torch.empty_like(buf) for _ in range(world)] if rank == dst else None
    dist.gather(buf, out, dst=dst, group=group)
    if rank != dst:
        return None
    return torch.cat([o[: e - s] for o, (s, e) in zip(out, sizes)], 0)

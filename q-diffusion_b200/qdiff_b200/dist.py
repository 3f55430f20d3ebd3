"""Multi-GPU plumbing of the sampling path (SURVEY 8e): the batch shards by images, weights are replicated,
nothing is exchanged inside the denoising loop; the only collective is the final gather of latents.

To make an N-rank run produce exactly the 1-rank result, every rank draws the FULL-batch noise from the same
seed (the reference draws one torch.randn(shape) for the whole batch: ldm/models/diffusion/plms.py:124,
ddim.py:126) and keeps its contiguous slice.
"""
import torch


def shard_bounds(global_batch, rank, world):
    if global_batch % world:
        raise ValueError(f"global batch {global_batch} is not divisible by world size {world}")
    per = global_batch // world
    return rank * per, (rank + 1) * per


def shard_like_single_process(shape, seed, rank, world, extra_shapes=()):
    """Full-batch tensors drawn from one CPU generator, sliced to this rank.  shape[0] is the GLOBAL batch.
    Returns [x_T shard, *extra shards] (extras share the generator, in order)."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = shard_bounds(shape[0], rank, world)
    out = []
    for s in (tuple(shape),) + tuple(tuple(e) for e in extra_shapes):
        full = torch.randn(s, generator=g)
        out.append(full[lo:hi].contiguous())
    return out


def step_noise_fn(shape, seed, rank, world):
    """noise_fn(k, size, device) for the stochastic samplers: every call draws the next FULL-batch noise tensor from one
    CPU generator seeded with `seed` and returns this rank's slice on `device`.  One step's noise is drawn when the step
    needs it, so nothing is precomputed for the whole loop (1000 steps of CIFAR batch 64 would be ~0.8 GB).
    shape[0] is the GLOBAL batch."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = shard_bounds(shape[0], rank, world)

    def noise_fn(k, size, device):
        return torch.randn(tuple(shape), generator=g)[lo:hi].to(device)
    return noise_fn


def gather_latents(local, world):
    """Final image gather: all_gather of the per-rank latents, concatenated in rank order (rank 0 saves)."""
    if world == 1:
        return local
    import torch.distributed as dist
    parts = [torch.empty_like(local) for _ in range(world)]
    dist.all_gather(parts, local.contiguous())
    return torch.cat(parts, dim=0)

"""Utterance sharding across GPUs: batch rows are independent for the whole
K-step loop, so each rank samples a contiguous slice of the batch with no per-step communication and
ONE all-gather of the finished mel shards at the end (NCCL over NVLink / NVSwitch; gloo on CPU tests).
"""
import torch
import torch.distributed as dist

from . import _capi


def shard_bounds(n_items, world_size, rank):
    """Contiguous, balanced split: the first (n % world) ranks hold one extra item."""
    base, extra = divmod(n_items, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(tensor, world_size=None, rank=None, dim=0):
    world_size = dist.get_world_size() if world_size is None else world_size
    rank = dist.get_rank() if rank is None else rank
    lo, hi = shard_bounds(tensor.shape[dim], world_size, rank)
    return tensor.narrow(dim, lo, hi - lo)


def all_gather_batch(local, n_items, group=None):
    """local: this rank's [b_r, ...] shard -> [n_items, ...] on every rank (one collective).  Equal shards (n_items % world
    == 0, the usual case) gather straight into the result; ragged shards go through one padded staging buffer."""
    world = dist.get_world_size(group)
    cap = (n_items + world - 1) // world
    tail = tuple(local.shape[1:])
    fused = hasattr(dist, "all_gather_into_tensor") and local.is_cuda
    if n_items % world == 0:
        out = torch.empty((n_items,) + tail, dtype=local.dtype, device=local.device)
        src = local.contiguous()
        dist.all_gather_into_tensor(out, src, group=group) if fused else _all_gather_list(out, src, world, group)
        return out
    pad = torch.zeros((cap,) + tail, dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = torch.empty((world * cap,) + tail, dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad, group=group) if fused else _all_gather_list(out, pad, world, group)
    parts = []
    for r in range(world):
        lo, hi = shard_bounds(n_items, world, r)
        parts.append(out[r * cap: r * cap + (hi - lo)])
    return torch.cat(parts, 0)


def _all_gather_list(out, pad, world, group):
    chunks = list(out.chunk(world, 0))
    dist.all_gather(chunks, pad, group=group)


def sharded_infer(sampler, cond, K_step, spec_min, spec_max, group=None, **kw):
    """Runs DsxSampler.infer on this rank's utterances and all-gathers mel_out [B,T,M].
    Per-utterance keyword tensors (fs2_mel, x_start, start_noise, mel2ph) are sliced like cond;
    step_noise [K,B,...] is sliced on dim 1."""
    B = cond.shape[0]
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    lo, hi = shard_bounds(B, world, rank)
    sl = {}
    for k, v in kw.items():
        if torch.is_tensor(v) and k in ("fs2_mel", "x_start", "start_noise", "mel2ph"):
            sl[k] = v[lo:hi]
        elif torch.is_tensor(v) and k == "step_noise":
            sl[k] = v[:, lo:hi]
        else:
            sl[k] = v
    if hi > lo:
        # in-kernel Philox noise is indexed by the GLOBAL utterance number: one seed gives every rank's utterances their own
        # noise, and the sharded result equals the unsharded one
        sampler.ensure_weights(cond.device)
        sampler.set_option(_capi.OPT_BATCH_OFFSET, lo)
        try:
            local = sampler.infer(cond[lo:hi], K_step, spec_min, spec_max, **sl)
        finally:
            sampler.set_option(_capi.OPT_BATCH_OFFSET, 0)
    else:
        local = torch.zeros((0, cond.shape[2], spec_min.numel()), device=cond.device)
    return all_gather_batch(local, B, group)

"""Batch-sharded generation over the GPUs of one node (SURVEY.md 8e): every sequence is independent through the whole
of generate(), so rank r generates a contiguous slice of the batch with replicated weights and the decoded images are
assembled with ONE all-gather at the end.  No collective runs inside the decode loop.  The sampler's Philox counters are
keyed on the global sequence index (MaskGit.row_offset), so token ids do not depend on the number of ranks."""
import numbers

import torch
import torch.distributed as dist

PER_IMAGE_SETTINGS = ("temperature", "cond_scale", "critic_noise_scale")


def shard_bounds(total, rank, world):
    """Contiguous balanced split: the first (total % world) ranks get one extra item."""
    base, extra = divmod(total, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def gather_batch(local, total, group=None):
    """All-gather row-sharded tensors (shards from shard_bounds, possibly uneven) into the full batch on every rank."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local
    rank = dist.get_rank(group)
    per = -(-total // world)
    if total % world == 0:
        out = torch.empty((total,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    pad = torch.zeros((per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    out = torch.empty((world * per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    pieces = []
    for r in range(world):
        lo, hi = shard_bounds(total, r, world)
        pieces.append(out[r * per:r * per + (hi - lo)])
    return torch.cat(pieces, 0)


def generate_sharded(maskgit, texts, text_embeds=None, cond_images=None, group=None, *, text_embeds_shard=None, cond_images_shard=None,
                     seed=None, **generate_kwargs):
    """maskgit.generate over this rank's slice of `texts`, then one all-gather.  Returns the full batch on every rank.

    Inputs indexed by GLOBAL row (`text_embeds` [B, L, D], `cond_images` [B, ...]) are sliced here; a caller whose loader already
    holds only its own rows passes `text_embeds_shard` / `cond_images_shard` (rows [lo, hi) of shard_bounds) instead.

    The sampler noise is keyed on the global sequence index, so the token ids do not depend on the number of ranks:
    "mmg" mode uses ONE seed for all ranks — `seed` when the caller passes the same value on every rank (no communication), else rank
    0's `sampler_seed` or its draw from torch's generator, broadcast; "aten" mode is told the size of the whole batch the reference would
    have drawn noise for (`global_batch`)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    total = len(texts)
    lo, hi = shard_bounds(total, rank, world)
    for name in PER_IMAGE_SETTINGS:       # per-image settings (a sequence or 1-D tensor of `total` values) are sliced like text_embeds
        value = generate_kwargs.get(name)
        if value is None or isinstance(value, numbers.Real) or (isinstance(value, torch.Tensor) and value.dim() == 0):
            continue
        if len(value) != total:
            raise ValueError(f"{name} has {len(value)} values for {total} texts")
        generate_kwargs[name] = value[lo:hi]
    tr = maskgit.transformer
    saved = (tr.encode_text, maskgit.row_offset, maskgit.global_batch, maskgit.sampler_seed)
    try:
        if seed is None:
            seed = maskgit.sampler_seed if maskgit.sampler_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
            if world > 1:
                box = [seed]
                dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
                seed = box[0]
        maskgit.sampler_seed, maskgit.row_offset, maskgit.global_batch = seed, lo, total
        if text_embeds_shard is None and text_embeds is not None:
            text_embeds_shard = text_embeds[lo:hi]
        if text_embeds_shard is not None:
            assert text_embeds_shard.shape[0] == hi - lo, "text_embeds_shard must hold exactly this rank's rows"
            shard = text_embeds_shard
            tr.encode_text = lambda t: shard
        if cond_images_shard is None and cond_images is not None:
            cond_images_shard = cond_images[lo:hi]
        if hi > lo:
            local = maskgit.generate(texts[lo:hi], cond_images=cond_images_shard, **generate_kwargs)
        else:       # more ranks than sequences: this rank contributes an empty shard of the right shape / dtype / device
            size = maskgit.image_size
            local = torch.empty((0, maskgit.vae.channels, size, size), dtype=torch.float32, device=next(maskgit.parameters()).device)
    finally:
        tr.encode_text, maskgit.row_offset, maskgit.global_batch, maskgit.sampler_seed = saved
    return gather_batch(local, total, group)

"""Batch-sharded generation and editing over the GPUs of one node (SURVEY.md 8e): every sequence is independent through the whole
of generate(), inpaint(), edit(), extrapolate() and the Muse cascade, so rank r runs a contiguous slice of the batch with replicated weights and the
results are assembled with all-gathers at the end.  No collective runs inside the decode loop.  The sampler's Philox counters are
keyed on the global sequence index (MaskGit.row_offset), so token ids do not depend on the number of ranks; with `image_seeds` (one seed
per image, sliced by global row like the per-image settings) each image's noise depends on its own seed alone."""
import numbers

import torch
import torch.distributed as dist

from .muse_maskgit import MaskGit, _image_seeds, _is_scalar, _muse_result

PER_IMAGE_SETTINGS = ("temperature", "cond_scale", "critic_noise_scale", "topk_filter_thres", "timesteps", "superres_timesteps")
ROW_INPUTS = ("images", "mask", "cond_images")      # call inputs indexed by global row, sliced like `texts`


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


def _gather(local, total, group):
    """gather_batch of a call's result: one tensor, or each tensor of an (images, ids) tuple."""
    if isinstance(local, tuple):
        return tuple(gather_batch(t, total, group) for t in local)
    return gather_batch(local, total, group)


def _empty_result(maskgit, return_ids=False, fmap_size=None, image_hw=None):
    """What a rank without rows contributes: (0, C, S, S) fp32 images and, with return_ids, (0, f, f) int64 ids, on the model's device.
    image_hw: the (H, W) of a call whose images are not S x S (extrapolate); its ids are then (0, H / p, W / p)."""
    device = next(maskgit.parameters()).device
    size = maskgit.image_size
    H, W = image_hw if image_hw is not None else (size, size)
    images = torch.empty((0, maskgit.vae.channels, H, W), dtype=torch.float32, device=device)
    if not return_ids:
        return images
    if image_hw is not None:
        shape = (H // maskgit.vae.dim_divisor, W // maskgit.vae.dim_divisor)
    else:
        f = fmap_size if fmap_size is not None else maskgit.vae.get_encoded_fmap_size(size)
        shape = (f, f)
    return images, torch.empty((0,) + shape, dtype=torch.int64, device=device)


def _run_shard(method, maskgits, texts, lo, hi, total, empty, *, group=None, seeds=None, text_embeds=None, text_embeds_shard=None,
               cond_images_shard=None, **kwargs):
    """method(texts[lo:hi], **kwargs) as the holder of rows [lo, hi) of a batch of `total` images; returns this rank's result, or
    empty() when lo == hi.  Every rank of `group` must call it, with its own (lo, hi): the seeds are one broadcast.

    maskgits: the MaskGits `method` samples with, in the order one process draws their seeds.  Each gets row_offset = lo, global_batch =
    total and one seed shared by every rank: seeds[i] when given (no communication), else its sampler_seed or a draw from torch's
    generator, as rank 0 of `group` has them.  text_embeds (rows of the whole batch) or text_embeds_shard (rows [lo, hi)) replace every
    maskgit transformer's encode_text.  kwargs named in ROW_INPUTS and per-image settings given per image are indexed by global row and
    sliced here; cond_images_shard replaces the slice of cond_images.  image_seeds (per-image seeds in any form generate() takes, for the
    whole batch) become this rank's rows' seeds; no call seed is then drawn or broadcast, since no kernel reads it.  The attributes are
    restored on return, also when the call raises.

    Per-image timesteps and top-k thresholds are checked on the whole batch first, by every maskgit, so every rank raises the same
    ValueError before any collective: checked on its own slice only, a rank could pass where another raises and wait in the all-gather,
    or (sampler_rng = "aten", mixed counts that are uniform per slice) run and advance its CUDA generator differently from the others."""
    for name in ("timesteps", "superres_timesteps"):
        if kwargs.get(name) is not None and not _is_scalar(kwargs[name]):
            for m in maskgits:
                m._steps_arg(kwargs[name], total)
    if kwargs.get("topk_filter_thres") is not None and not _is_scalar(kwargs["topk_filter_thres"]):
        for m in maskgits:
            m._thres_arg(kwargs["topk_filter_thres"], total)
    for name in PER_IMAGE_SETTINGS:       # per-image settings (a sequence or 1-D tensor of `total` values) are sliced like text_embeds
        value = kwargs.get(name)
        if value is None or isinstance(value, numbers.Real) or (isinstance(value, torch.Tensor) and value.dim() == 0):
            continue
        if len(value) != total:
            raise ValueError(f"{name} has {len(value)} values for {total} texts")
        kwargs[name] = value[lo:hi]
    for name in ROW_INPUTS:
        value = kwargs.get(name)
        if value is None:
            continue
        if len(value) != total:
            raise ValueError(f"{name} has {len(value)} rows for {total} texts")
        kwargs[name] = value[lo:hi]
    if cond_images_shard is not None:
        kwargs["cond_images"] = cond_images_shard
    if kwargs.get("image_seeds") is not None:
        kwargs["image_seeds"] = _image_seeds(kwargs["image_seeds"], total)[lo:hi]
        if seeds is None:
            seeds = [m.sampler_seed for m in maskgits]
    if seeds is None:
        seeds = [m.sampler_seed if m.sampler_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item()) for m in maskgits]
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            box = [seeds]
            dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
            seeds = box[0]
    if text_embeds_shard is None and text_embeds is not None:
        text_embeds_shard = text_embeds[lo:hi]
    if text_embeds_shard is not None:
        assert text_embeds_shard.shape[0] == hi - lo, "text_embeds_shard must hold exactly this rank's rows"
    saved = [(m.transformer.encode_text, m.row_offset, m.global_batch, m.sampler_seed) for m in maskgits]
    try:
        for m, seed in zip(maskgits, seeds):
            m.sampler_seed, m.row_offset, m.global_batch = seed, lo, total
            if text_embeds_shard is not None:
                m.transformer.encode_text = lambda t, shard=text_embeds_shard: shard
        if hi > lo:
            return method(texts[lo:hi], **kwargs)
        return empty()            # more ranks than sequences: an empty shard of the right shape / dtype / device
    finally:
        for m, (encode_text, row_offset, global_batch, sampler_seed) in reversed(list(zip(maskgits, saved))):
            m.transformer.encode_text, m.row_offset, m.global_batch, m.sampler_seed = encode_text, row_offset, global_batch, sampler_seed


def _sharded_call(maskgit, method, texts, group, seed, kwargs, image_hw=None):
    """A MaskGit call over this rank's rows, then the all-gather of its result (image_hw: as _empty_result's)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    total = len(texts)
    lo, hi = shard_bounds(total, rank, world)
    empty = lambda: _empty_result(maskgit, kwargs.get("return_ids", False), kwargs.get("fmap_size"), image_hw)
    local = _run_shard(method, (maskgit,), texts, lo, hi, total, empty, group=group, seeds=None if seed is None else (seed,), **kwargs)
    return _gather(local, total, group)


def generate_sharded(maskgit, texts, text_embeds=None, cond_images=None, group=None, *, text_embeds_shard=None, cond_images_shard=None,
                     seed=None, **generate_kwargs):
    """maskgit.generate over this rank's slice of `texts`, then one all-gather.  Returns the full batch on every rank (with
    return_ids=True, the (images, ids) of the whole batch).

    Inputs indexed by GLOBAL row (`text_embeds` [B, L, D], `cond_images` [B, ...], per-image settings) are sliced here; a caller whose
    loader already holds only its own rows passes `text_embeds_shard` / `cond_images_shard` (rows [lo, hi) of shard_bounds) instead.

    The sampler noise is keyed on the global sequence index, so the token ids do not depend on the number of ranks:
    "mmg" mode uses ONE seed for all ranks — `seed` when the caller passes the same value on every rank (no communication), else rank
    0's `sampler_seed` or its draw from torch's generator, broadcast; "aten" mode is told the size of the whole batch the reference would
    have drawn noise for (`global_batch`).  Not with `sampler_noise_fn`: the callable sees only this rank's shape.  `image_seeds` (one
    seed per image of the whole batch, a keyword separate from the call-wide `seed`) is sliced by global row; each image's result then
    depends on its own seed, not on `seed`, its rank or row_offset."""
    return _sharded_call(maskgit, maskgit.generate, texts, group, seed,
                         dict(generate_kwargs, text_embeds=text_embeds, text_embeds_shard=text_embeds_shard, cond_images=cond_images,
                              cond_images_shard=cond_images_shard))


def inpaint_sharded(maskgit, texts, images, mask, text_embeds=None, cond_images=None, group=None, *, text_embeds_shard=None,
                    cond_images_shard=None, seed=None, **inpaint_kwargs):
    """maskgit.inpaint over this rank's rows, then the all-gather of the images (and ids with return_ids=True).  `images` and `mask`
    (every form inpaint takes) are indexed by global row and sliced here, as are text_embeds, cond_images and per-image settings.  Each
    rank counts the regenerated tokens of its own rows only, and samples mask_schedule(its largest count) rows per image and step.

    Seeds and the rank-count invariance of the token ids are generate_sharded's: one seed for every rank in "mmg" mode, `global_batch`
    in "aten" mode; not with `sampler_noise_fn`.  `image_seeds` is sliced by global row, as for generate_sharded."""
    return _sharded_call(maskgit, maskgit.inpaint, texts, group, seed,
                         dict(inpaint_kwargs, images=images, mask=mask, text_embeds=text_embeds, text_embeds_shard=text_embeds_shard,
                              cond_images=cond_images, cond_images_shard=cond_images_shard))


def edit_sharded(maskgit, texts, images, mask=None, text_embeds=None, cond_images=None, group=None, *, text_embeds_shard=None,
                 cond_images_shard=None, seed=None, **edit_kwargs):
    """maskgit.edit over this rank's rows, then the all-gather, sliced as inpaint_sharded (`mask` may be None: every token editable).
    The selection keys are keyed on the global position too, so with one seed for every rank ("mmg" mode) the token ids do not depend
    on the number of ranks.  sampler_rng = "aten" raises ValueError on every rank, as edit() does; `sampler_noise_fn` is not covered.
    `image_seeds` is sliced by global row, as for generate_sharded."""
    if maskgit.sampler_rng == "aten":          # raised here, before any collective, so that ranks without rows raise it too
        raise ValueError('edit() has no "aten" noise stream (the reference has no editing): use sampler_rng = "mmg" or sampler_noise_fn')
    MaskGit._round_steps("edit", edit_kwargs.get("timesteps", 4))
    return _sharded_call(maskgit, maskgit.edit, texts, group, seed,
                         dict(edit_kwargs, images=images, mask=mask, text_embeds=text_embeds, text_embeds_shard=text_embeds_shard,
                              cond_images=cond_images, cond_images_shard=cond_images_shard))


def extrapolate_sharded(maskgit, texts, images, direction="right", amount=256, text_embeds=None, group=None, *, text_embeds_shard=None,
                        seed=None, **extrapolate_kwargs):
    """maskgit.extrapolate over this rank's rows, then the all-gather of the grown images (and canvases with return_ids=True).  `images`
    is indexed by global row and sliced here, as are text_embeds and per-image settings; a rank without rows contributes the grown
    (0, C, H', W') / (0, H'/p, W'/p) shapes.  The arguments are checked on the whole batch before any collective, so every rank raises the
    same ValueError.  The sampler noise is keyed on the global row and the window-local position, so with one seed for every rank ("mmg"
    mode) the token ids do not depend on the number of ranks; sampler_rng = "aten" raises ValueError, as extrapolate() does, and
    `sampler_noise_fn` is not covered.  `image_seeds` is sliced by global row, as for generate_sharded."""
    MaskGit._round_steps("extrapolate", extrapolate_kwargs.get("timesteps", 18))
    window = maskgit._extrapolate_plan(images, len(texts), direction, amount, extrapolate_kwargs.get("stride"))
    p = maskgit.vae.dim_divisor
    return _sharded_call(maskgit, maskgit.extrapolate, texts, group, seed,
                         dict(extrapolate_kwargs, images=images, direction=direction, amount=amount, text_embeds=text_embeds,
                              text_embeds_shard=text_embeds_shard),
                         image_hw=(window.canvas[0] * p, window.canvas[1] * p))


def muse_sharded(muse, texts, text_embeds=None, group=None, *, text_embeds_shard=None, **forward_kwargs):
    """Muse.forward over this rank's texts: the base stage makes this rank's low-res images and the super-resolution stage, on the same
    rank, is conditioned on them, so nothing is exchanged between the stages.  One all-gather of the super-resolution images (and one of
    the low-res images with return_lowres) at the end; PIL conversion follows the gather, so every rank returns what Muse.forward returns.

    Seeds: each stage's own `sampler_seed`, else a draw from torch's generator, base first, as one process draws them; rank 0's pair
    reaches every rank in one broadcast.  text_embeds / text_embeds_shard are handed to both stages' transformers.  Per-image
    cond_scale / temperature / timesteps / superres_timesteps are sliced by global row.  Token ids do not depend on the number of ranks, as for generate_sharded.
    `image_seeds` is sliced by global row; Muse.forward derives the super-resolution seeds from each rank's slice."""
    return_lowres = forward_kwargs.pop("return_lowres", False)
    return_pil_images = forward_kwargs.pop("return_pil_images", True)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    total = len(texts)
    lo, hi = shard_bounds(total, rank, world)
    base, superres = muse.base_maskgit, muse.superres_maskgit
    empty = lambda: (_empty_result(superres), _empty_result(base))
    hi_res, low_res = _run_shard(muse.forward, (base, superres), texts, lo, hi, total, empty, group=group, text_embeds=text_embeds,
                                 text_embeds_shard=text_embeds_shard, return_lowres=True, return_pil_images=False, **forward_kwargs)
    hi_res = gather_batch(hi_res, total, group)
    low_res = gather_batch(low_res, total, group) if return_lowres else None
    return _muse_result(hi_res, low_res, return_lowres, return_pil_images)

"""CPU oracle of MaskGit.edit's token loop: an fp32 restatement on torch CPU, composed from tests/inpaint_oracle.inpaint_ids.  The reference has
no editing; the loop restated here is:

  ids = ids0, E = editable positions, N_b = E[b].sum(), r_b = max(int(fraction * N_b), 1) (0 when N_b = 0)
  per iteration i: keys = noise_fn(i * timesteps, (b, n)); image b selects the r_b largest keys among its editable positions (ties: lowest
  position); then inpaint_ids with regen = the selection and the noise of its step s drawn as noise_fn(i * timesteps + s, shape)."""
import numpy as np
import torch

from oracle import philox
from tests import inpaint_oracle as IO

KEY_C0 = 0xFFFFFFFE          # first Philox counter word of the selection keys (gumbel noise: vocabulary index, critic noise: 0xFFFFFFFF)


def select_counts(editable, fraction):
    """[b] r_b: max(int(fraction * N_b), 1) in Python floats, 0 when image b has no editable token."""
    return [max(int(fraction * int(c)), 1) if int(c) else 0 for c in editable.sum(dim=1)]


def select(keys, editable, counts):
    """(b, n) bool: the counts[b] largest keys among row b's editable positions, ties to the lowest position."""
    sel = torch.zeros(keys.shape, dtype=torch.bool)
    for i, c in enumerate(counts):
        free = editable[i].nonzero().flatten()
        order = free[torch.argsort(-keys[i, free], stable=True)]
        sel[i, order[:c]] = True
    return sel


def philox_keys(seed, iteration, b, n, row_offset=0):
    """(b, n) fp32 keys of mmg_edit_select's Philox mode: counter (0xFFFFFFFE, iteration, grow_lo, grow_hi), key = seed,
    grow = (row_offset + b) * n + p."""
    grow = np.arange(row_offset * n, (row_offset + b) * n, dtype=np.uint64)
    w0, _, _, _ = philox.philox4(np.full(grow.shape, KEY_C0, dtype=np.uint64), np.full(grow.shape, iteration & 0xFFFFFFFF, dtype=np.uint64),
                                 grow & np.uint64(0xFFFFFFFF), grow >> np.uint64(32), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    u = (w0 >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / (1 << 24))
    return torch.from_numpy(u.reshape(b, n))


def edit_ids(sd, cfg, text_embeds, ids0, editable, mask_id, noise_fn, iterations=8, fraction=0.1, timesteps=4, trace=None, **kw):
    """ids0 (b, n) int64: the encoded image tokens; editable (b, n) bool.  noise_fn as in inpaint_ids, called in the order of the GPU path:
    each iteration's keys, then the draws of its decode steps.  kw goes to inpaint_ids (cond_ids, cond_scale, temperature, critic, ...).
    trace (list) receives one dict per iteration: keys, selected, ids (after the iteration)."""
    b, n = ids0.shape
    editable = editable.reshape(b, n).bool()
    counts = select_counts(editable, fraction)
    ids = ids0
    for i in range(iterations):
        keys = noise_fn(i * timesteps, (b, n))
        sel = select(keys, editable, counts)
        ids = IO.inpaint_ids(sd, cfg, text_embeds, ids, sel, mask_id, lambda s, shape, i=i: noise_fn(i * timesteps + s, shape),
                             timesteps=timesteps, **kw)
        if trace is not None:
            trace.append(dict(keys=keys, selected=sel, ids=ids))
    return ids

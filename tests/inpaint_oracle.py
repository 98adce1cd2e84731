"""CPU oracle of MaskGit.inpaint's token loop: an fp32 restatement on torch CPU, built from the pinned pieces of oracle/muse_oracle.py
(forward, sampling tail, critic) in the same way as muse_oracle.generate_ids.  The reference has no inpainting; the loop restated here is:

  ids = where(regen, mask_id, known_ids), scores = 0, frozen = ~regen, N_b = regen[b].sum()
  per step: image b re-masks the num_masked_b = max(int(noise_schedule(t) * N_b), 1) (0 when N_b = 0) highest scores among its
  non-frozen positions (one topk per image), then the step of generate_ids: the forward, the sampling tail (ids = where(is_mask, pred, ids),
  so frozen ids are never replaced) and, with a critic, the critic's scores.  Frozen scores are ignored by the next re-mask."""
import torch

from oracle import muse_oracle as O


def image_schedules(regen, timesteps):
    """[b][timesteps] regenerated-token counts per image and step (O.mask_schedule with seq_len = N_b, all 0 when N_b = 0)."""
    return [O.mask_schedule(int(c), timesteps) if int(c) else [0] * timesteps for c in regen.sum(dim=1)]


def inpaint_ids(sd, cfg, text_embeds, known_ids, regen, mask_id, noise_fn, cond_ids=None, timesteps=18, cond_scale=3.0, temperature=1.0,
                topk_thres=0.9, trace=None, critic=None, critic_noise_scale=1.0, can_remask_prev_masked=False):
    """known_ids (b, n) int64: the encoded image tokens; regen (b, n) bool: True = regenerate.  noise_fn and critic as in
    O.generate_ids (the same draws in the same order).  trace (list) receives one dict per step, with num_masked the per-image list."""
    b, n = known_ids.shape
    regen = regen.reshape(b, n).bool()
    frozen = ~regen
    ids = torch.where(regen, torch.full_like(known_ids, mask_id), known_ids)
    scores = torch.zeros((b, n), dtype=torch.float32)
    scheds = image_schedules(regen, timesteps)
    self_cond_embed = None
    for step, steps_until_x0 in enumerate(reversed(range(timesteps))):
        counts = [s[step] for s in scheds]
        ids = ids.clone()                                       # the re-mask below writes in place; the trace keeps the previous step's ids
        for i, c in enumerate(counts):
            if c:
                free = (~frozen[i]).nonzero().flatten()
                sel = free[scores[i, free].topk(c).indices]
                ids[i, sel] = mask_id
        logits, embed = O.forward_with_cond_scale(sd, cfg, ids, text_embeds, cond_ids, cond_scale, self_cond_embed)
        if cfg.get("self_cond", False):
            self_cond_embed = embed
        temp = temperature * (steps_until_x0 / timesteps)
        u = noise_fn(step, logits.shape)
        masked_in = ids
        ids, scores, pred = O.sample_step(logits, ids, mask_id, temp, u, topk_thres, can_remask_prev_masked)
        if critic is not None:
            uc = noise_fn(step, scores.shape)
            scores = O.critic_scores(critic, ids, text_embeds, cond_ids, cond_scale, uc, critic_noise_scale * (steps_until_x0 / timesteps))
        if trace is not None:
            trace.append(dict(ids_in=masked_in, logits=logits, u=u, temperature=temp, pred=pred, ids_out=ids, scores=scores,
                              num_masked=counts, embed=embed))
    return ids

"""CPU restatement of MaskGit.forward, the training loss (ref: muse_maskgit_pytorch.py:623-741), on oracle/muse_oracle.py's
transformer_forward.  TEST INFRASTRUCTURE ONLY.

draw(shape) stands in for every torch uniform draw of the reference, in its order:
  uniform((b,)) mask ratio -> rand((b, n)) permutation -> rand((b, n)) of get_mask_subset_prob (no_mask_token_prob > 0) ->
  uniform((b, 1)) conditioning drop (0 < cond_drop_prob < 1) -> critic branch: gumbel noise (b, n, V), the critic's own drop mask;
py_random() for python's random(): self-conditioning (transformer self_cond only) and the critic's sampling temperature.
"""
import math

import torch
import torch.nn.functional as F

from oracle import muse_oracle as O


def cosine_schedule(t):
    return torch.cos(t * math.pi * 0.5)


def mask_subset_prob(mask, prob, draw, min_mask=0):
    """ref: muse_maskgit_pytorch.py:46-60."""
    num_to_mask = (mask.sum(dim=-1, keepdim=True) * prob).clamp(min=min_mask)
    logits = draw(mask.shape).masked_fill(~mask, -1)
    randperm = logits.argsort(dim=-1).argsort(dim=-1).float()
    randperm -= (~mask).sum(dim=-1, keepdim=True)
    return (randperm < num_to_mask).masked_fill_(~mask, False)


def drop_text(text_embeds, cond_drop_prob, draw):
    """prob_mask_like((b, 1), 1 - cond_drop_prob) of Transformer.forward (ref :306-310, 393-399) as zeroed text rows (= masked keys);
    cond_drop_prob == 1 is transformer_forward's drop_text flag."""
    if not 0. < cond_drop_prob < 1.:
        return text_embeds
    keep = draw((text_embeds.shape[0], 1)) < (1. - cond_drop_prob)
    return text_embeds * keep[:, :, None]


def maskgit_loss(sd, cfg, ids, text_embeds, mask_id, draw, py_random, cond_ids=None, ignore_index=-1, cond_drop_prob=0.5,
                 no_mask_token_prob=0., self_cond_prob=0.9, noise_schedule=cosine_schedule,
                 critic=None, critic_loss_weight=1., train_only_generator=False, sample_temperature=None):
    """ids (b, ...) int64 token ids (already tokenised); cfg = dict(heads, depth, self_cond).  critic: None, dict(kind="token", sd, cfg) or
    dict(kind="self", w_pred, b_pred) (the generator's own stack).  Returns the 0-d loss."""
    ids = ids.reshape(ids.shape[0], -1)
    b, n = ids.shape
    num_token_masked = (n * noise_schedule(draw((b,)))).round().clamp(min=1)
    mask = draw((b, n)).argsort(dim=-1) < num_token_masked[:, None]
    labels = torch.where(mask, ids, ignore_index)
    if no_mask_token_prob > 0.:
        mask &= ~mask_subset_prob(mask, no_mask_token_prob, draw)
    x = torch.where(mask, mask_id, ids)
    self_cond_embed = None
    if cfg.get("self_cond", False) and py_random() < self_cond_prob:
        _, self_cond_embed = O.transformer_forward(sd, cfg, x, text_embeds, cond_ids, False, None, True)
    te = drop_text(text_embeds, cond_drop_prob, draw)
    logits = O.transformer_forward(sd, cfg, x, te, cond_ids, cond_drop_prob == 1, self_cond_embed)
    ce_loss = F.cross_entropy(logits.transpose(1, 2), labels, ignore_index=ignore_index)
    if critic is None or train_only_generator:
        return ce_loss
    temperature = py_random()
    if sample_temperature is not None:
        temperature = sample_temperature
    sampled = (logits / max(temperature, 1e-10) + O.gumbel_from_uniform(draw(logits.shape))).argmax(dim=-1)
    critic_input = torch.where(mask, sampled, x)
    critic_labels = (ids != critic_input).float()
    te_c = drop_text(text_embeds, cond_drop_prob, draw)
    if critic["kind"] == "token":
        s = O.transformer_forward(critic["sd"], critic["cfg"], critic_input, te_c, cond_ids, cond_drop_prob == 1)[..., 0]
    else:
        _, embed = O.transformer_forward(sd, cfg, critic_input, te_c, cond_ids, cond_drop_prob == 1, None, True)
        s = (embed @ critic["w_pred"].t() + critic["b_pred"])[..., 0]
    return ce_loss + critic_loss_weight * F.binary_cross_entropy_with_logits(s, critic_labels)


# ------------------------------------------------------------------ the cases of tests/golden/loss_small.npz (make_loss_golden.py)
def golden_cases():
    """{name: dict(model, model_kw, kw, input, cond_images, seed, py_seed, loss)} from tests/golden/loss_small.npz."""
    import json
    import numpy as np
    from tests import util
    z = np.load(f"{util.GOLDEN}/loss_small.npz")
    cases = {}
    for key in z.files:
        name, field = key.split(".")
        c = cases.setdefault(name, {})
        if field == "meta":
            c.update(json.loads(bytes(z[key]).decode()))
        elif field == "seeds":
            c["seed"], c["py_seed"] = (int(v) for v in z[key])
        elif field == "loss":
            c["loss"] = float(z[key][0])
        elif field == "py_draws":
            c["py_draws"] = [float(v) for v in z[key]]
        else:
            c[field] = torch.from_numpy(z[key])
    for c in cases.values():
        c.setdefault("cond_images", None)
    return cases


def model_weights(model):
    """State dicts of the G4-G8 models (tests/golden/make_golden.py): (transformer sd, cfg, critic, vae sd, seq_len)."""
    from tests import util
    vae = util.vae_sd(16, 2, 1024, seed=12)
    seq_len, seed, self_cond = dict(g4=(16, 13, False), g5=(64, 15, False), g6=(16, 21, True), g7=(16, 13, False), g8=(16, 21, True))[model]
    sd = util.transformer_sd(1024, 128, seq_len, 2, 2, seed=seed, text_dim=128)
    critic = None
    if model == "g7":
        critic = dict(kind="token", sd=util.critic_sd(1024, 128, 16, 1, 2, seed=22, text_dim=128), cfg=dict(heads=2, depth=1))
    elif model == "g8":
        w, b = util.self_critic_head()
        critic = dict(kind="self", w_pred=w, b_pred=b)
    return sd, dict(heads=2, depth=2, self_cond=self_cond), critic, vae, seq_len


def golden_case_loss(c, draw, py_random):
    """The oracle loss of one golden case with the given draws."""
    from tests import util
    sd, cfg, critic, vae, _ = model_weights(c["model"])
    inp = c["input"]
    ids = O.vae_encode(vae, inp)[1] if inp.dtype == torch.float32 else inp
    cond_ids = None if c["cond_images"] is None else O.vae_encode(vae, c["cond_images"])[1]
    te = util.text_embeds("g4.te", 3, 8, 128, 14)[:inp.shape[0]]
    kw = dict(c["kw"])
    mkw = dict(c["model_kw"])
    return maskgit_loss(sd, cfg, ids, te, 1024, draw, py_random, cond_ids=cond_ids, critic=critic,
                        cond_drop_prob=kw.pop("cond_drop_prob", 0.5), no_mask_token_prob=mkw.pop("no_mask_token_prob", 0.),
                        critic_loss_weight=mkw.pop("critic_loss_weight", 1.), **kw)

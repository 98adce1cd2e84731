"""Shared builders for the parity tests: hash-generated weights/inputs (same values as tests/golden/make_golden.py)."""
import os
import numpy as np
import torch

from oracle import synth, shapes, muse_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def sd_from_table(table, seed, overrides=None):
    return {k: torch.from_numpy(v) for k, v in synth.fill_state_dict(table, seed=seed, overrides=overrides).items()}


def transformer_sd(num_tokens, dim, seq_len, depth, heads, seed, text_dim=None, logit_gain=1.0):
    sd = sd_from_table(shapes.transformer_shapes(num_tokens, dim, seq_len, depth, heads=heads, text_dim=text_dim), seed)
    if logit_gain != 1.0:
        sd["to_logits.weight"] = sd["to_logits.weight"] * logit_gain
    return sd


def critic_sd(num_tokens, dim, seq_len, depth, heads, seed, text_dim=None):
    """TokenCritic: no mask row in token_emb, dim_out = 1 (ref: muse_maskgit_pytorch.py:383-386)."""
    return sd_from_table(shapes.transformer_shapes(num_tokens, dim, seq_len, depth, heads=heads, text_dim=text_dim,
                                                   add_mask_id=False, dim_out=1), seed)


def self_critic_head(seed=23, dim=128):
    w = torch.from_numpy(synth.normal("g8.to_pred.weight", (1, dim), seed)) * 0.2
    b = torch.from_numpy(synth.normal("g8.to_pred.bias", (1,), seed)) * 0.2
    return w, b


def vae_sd(dim, layers, codebook_size, seed):
    return sd_from_table(shapes.vae_shapes(dim, layers=layers, codebook_size=codebook_size), seed)


def text_embeds(name, b, m, d, seed):
    te = torch.from_numpy(synth.normal(name, (b, m, d), seed))
    te[1::2, (3 * m) // 4:] = 0.
    return te


def oracle_rows(logits, u_rows, temp, k):
    """per-row reference of the sampling tail: top-k filter (exactly k kept, ties by lowest index) + gumbel argmax + confidence, in the
    dtype of `logits` (float64 for the fused-tail tests).  Returns (token, 1 - softmax[token], top-2 margin of the perturbed values)."""
    R, V = logits.shape
    order = torch.argsort(-logits, dim=-1, stable=True)[:, :k]
    keep = torch.zeros((R, V), dtype=torch.bool).scatter_(1, order, True)
    filt = torch.where(keep, logits, torch.tensor(float("-inf"), dtype=logits.dtype))
    pert = filt / max(temp, 1e-10) + muse_oracle.gumbel_from_uniform(u_rows)
    pred = pert.argmax(-1)
    top2 = pert.topk(2, dim=-1).values
    p = logits.softmax(-1).gather(1, pred[:, None])[:, 0]
    return pred, 1 - p, top2[:, 0] - top2[:, 1]


def torch_noise_fn(seed):
    """Replays the reference's RNG consumption: torch.manual_seed(seed) once, then one
    zeros(shape).uniform_(0,1) per decode step (ref: muse_maskgit_pytorch.py:407)."""
    gen_state = {"started": False}

    def fn(step, shape):
        if not gen_state["started"]:
            torch.manual_seed(seed)
            gen_state["started"] = True
        return torch.zeros(shape).uniform_(0, 1)
    return fn

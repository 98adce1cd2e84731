"""Shared by the T5 encoder tests: configurations, seeded HF-keyed random weights (no transformers needed), the pinned error bounds."""
import types

import torch

# relative L2 error of the bf16 T5Encoder against the fp64 oracle.  Pinned to HF's own `T5EncoderModel.bfloat16()` error against fp64 at
# PIN_CFG (re-derived by tests/test_t5_oracle.py::test_bf16_bound_is_pinned_to_hf_bf16_error, which asserts this is <= 1.5x that error)
BF16_REL_L2_BOUND = 2.0e-2        # HF bf16 at PIN_CFG: 1.83e-2 (CPU, torch 2.11 / transformers 5.5)
# max-abs error on live rows of HF's fp32 T5EncoderModel against the fp64 oracle at the GPU test configurations (the largest over them,
# measured on the CPU with torch 2.11 / transformers 5.5); the fp32 T5Encoder must stay within 4x the error HF makes, and this stands in for
# HF's error when transformers is not installed
HF_FP32_MAX_ABS = 7.0e-6

SMALL_RELU = dict(vocab_size=512, d_model=128, d_kv=64, d_ff=192, num_layers=2, num_heads=2, feed_forward_proj="relu")
SMALL_GATED = dict(vocab_size=512, d_model=192, d_kv=64, d_ff=320, num_layers=3, num_heads=3, feed_forward_proj="gated-gelu")
V11_BASE = dict(vocab_size=1024, d_model=768, d_kv=64, d_ff=2048, num_layers=12, num_heads=12, feed_forward_proj="gated-gelu")
PIN_CFG, PIN_B, PIN_T = V11_BASE, 8, 32


def config(c):
    """A T5Config-like object (the fields T5Encoder and the oracle read), with HF's defaults for the rest."""
    full = dict(relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6)
    full.update(c)
    return types.SimpleNamespace(**full)


def hf_config(c):
    from transformers import T5Config
    return T5Config(**c, dropout_rate=0.0)


def random_sd(c, seed):
    """HF T5EncoderModel state_dict with HF's init scales (T5PreTrainedModel._init_weights, factor 1), fp32, seeded."""
    g = torch.Generator().manual_seed(seed)
    d, dkv, h, ff, V = c["d_model"], c["d_kv"], c["num_heads"], c["d_ff"], c["vocab_size"]
    n = lambda shape, std: torch.randn(shape, generator=g) * std
    one = lambda k: 1.0 + 0.1 * torch.randn(k, generator=g)
    sd = {"shared.weight": n((V, d), 1.0)}
    sd["encoder.embed_tokens.weight"] = sd["shared.weight"]
    for i in range(c["num_layers"]):
        p = f"encoder.block.{i}.layer."
        sd[p + "0.SelfAttention.q.weight"] = n((h * dkv, d), (d * dkv) ** -0.5)
        sd[p + "0.SelfAttention.k.weight"] = n((h * dkv, d), d ** -0.5)
        sd[p + "0.SelfAttention.v.weight"] = n((h * dkv, d), d ** -0.5)
        sd[p + "0.SelfAttention.o.weight"] = n((d, h * dkv), (h * dkv) ** -0.5)
        if i == 0:
            sd[p + "0.SelfAttention.relative_attention_bias.weight"] = n((32, h), d ** -0.5)
        sd[p + "0.layer_norm.weight"] = one(d)
        if c["feed_forward_proj"] == "gated-gelu":
            sd[p + "1.DenseReluDense.wi_0.weight"] = n((ff, d), d ** -0.5)
            sd[p + "1.DenseReluDense.wi_1.weight"] = n((ff, d), d ** -0.5)
        else:
            sd[p + "1.DenseReluDense.wi.weight"] = n((ff, d), d ** -0.5)
        sd[p + "1.DenseReluDense.wo.weight"] = n((d, ff), ff ** -0.5)
        sd[p + "1.layer_norm.weight"] = one(d)
    sd["encoder.final_layer_norm.weight"] = one(d)
    return sd


def random_batch(B, T, V, seed, pad=True):
    """ids [B, T] and a ragged right-padded mask (row 0 full length; with pad, the others random lengths >= 1)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (B, T), generator=g)
    lens = torch.randint(1, T + 1, (B,), generator=g) if pad else torch.full((B,), T)
    lens[0] = T
    mask = (torch.arange(T)[None, :] < lens[:, None]).long()
    return ids, mask


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())

"""fp64 CPU restatement of HF's T5 encoder (modeling_t5, T5EncoderModel in eval mode) from a state_dict under HF's keys.

No transformers import: the GPU tests of libmmg's T5Encoder compare against this.  Semantics restated literally:
  x = shared[ids]; per block: x += o(Attn(RMS(x))), x += wo(act(RMS(x))); out = RMS(x) with final_layer_norm, padding rows zeroed
  (t5_encode_text); RMS(x) = w * (x * rsqrt(mean(x^2) + eps)) with fp32 statistics;
  scores = q k^T (no scaling) + bias[h, bucket(key - query)] + mask, a masked key adding
  finfo(float32).min, softmax in fp32; block 0's relative_attention_bias serves every block; act = relu(wi x) or gelu_new(wi_0 x) * wi_1 x."""
import math

import torch

F64_MIN = float(torch.finfo(torch.float32).min)        # HF builds the mask in the model dtype; the fp32 model is the reference


def relative_position_bucket(relative_position, bidirectional=True, num_buckets=32, max_distance=128):
    """HF T5Attention._relative_position_bucket."""
    relative_buckets = 0
    if bidirectional:
        num_buckets //= 2
        relative_buckets += (relative_position > 0).to(torch.long) * num_buckets
        relative_position = torch.abs(relative_position)
    else:
        relative_position = -torch.min(relative_position, torch.zeros_like(relative_position))
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    relative_position_if_large = max_exact + (
        torch.log(relative_position.float() / max_exact) / math.log(max_distance / max_exact) * (num_buckets - max_exact)).to(torch.long)
    relative_position_if_large = torch.min(relative_position_if_large, torch.full_like(relative_position_if_large, num_buckets - 1))
    relative_buckets += torch.where(is_small, relative_position, relative_position_if_large)
    return relative_buckets


def _rms(x, w, eps):
    # T5LayerNorm: the variance, and so the rsqrt factor, are fp32 whatever the model's dtype
    variance = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    return w * (x * torch.rsqrt(variance + eps))


def _gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def encode(sd, cfg, input_ids, attention_mask=None):
    """sd: HF T5EncoderModel state_dict; cfg: dict(num_layers, num_heads, feed_forward_proj, relative_attention_num_buckets,
    relative_attention_max_distance, layer_norm_epsilon).  Returns fp64 [B, T, d_model] with padding rows zero."""
    W = lambda k: sd[k].detach().double().cpu()
    eps, heads = cfg.get("layer_norm_epsilon", 1e-6), cfg["num_heads"]
    gated = cfg.get("feed_forward_proj", "relu") == "gated-gelu"
    ids = input_ids.cpu()
    B, T = ids.shape
    mask = torch.ones((B, T), dtype=torch.long) if attention_mask is None else attention_mask.cpu().long()
    x = W("shared.weight")[ids]
    ctx = torch.arange(T)[:, None]
    mem = torch.arange(T)[None, :]
    buckets = relative_position_bucket(mem - ctx, True, cfg.get("relative_attention_num_buckets", 32), cfg.get("relative_attention_max_distance", 128))
    rel = W("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight")
    position_bias = rel[buckets].permute(2, 0, 1)[None]                                 # [1, H, T, T]
    position_bias = position_bias + (1.0 - mask[:, None, None, :].double()) * F64_MIN   # extended attention mask
    for i in range(cfg["num_layers"]):
        p = f"encoder.block.{i}.layer."
        h = _rms(x, W(p + "0.layer_norm.weight"), eps)
        split = lambda t: t.view(B, T, heads, -1).transpose(1, 2)
        q, k, v = (split(h @ W(p + f"0.SelfAttention.{n}.weight").t()) for n in "qkv")
        scores = q @ k.transpose(-1, -2) + position_bias
        attn = torch.softmax(scores.float(), dim=-1).type_as(scores) @ v          # HF: softmax in fp32 whatever the dtype
        x = x + attn.transpose(1, 2).reshape(B, T, -1) @ W(p + "0.SelfAttention.o.weight").t()
        h = _rms(x, W(p + "1.layer_norm.weight"), eps)
        if gated:
            a = _gelu_new(h @ W(p + "1.DenseReluDense.wi_0.weight").t()) * (h @ W(p + "1.DenseReluDense.wi_1.weight").t())
        else:
            a = torch.relu(h @ W(p + "1.DenseReluDense.wi.weight").t())
        x = x + a @ W(p + "1.DenseReluDense.wo.weight").t()
    out = _rms(x, W("encoder.final_layer_norm.weight"), eps)
    return out.masked_fill(~mask.bool()[..., None], 0.0)

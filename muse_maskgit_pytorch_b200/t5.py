"""Text encoder: dimension lookup, `t5_encode_text` (ref: t5.py:35-99), and `T5Encoder`, the T5 encoder on libmmg kernels.

`get_encoded_dim` / `T5_CONFIGS` are what constructing a Transformer needs (ref: t5.py:44-55, muse_maskgit_pytorch.py:229-233).
`t5_encode_text` runs HuggingFace's `T5EncoderModel` unless `T5_CONFIGS[name]` holds a `"native"` entry, a `T5Encoder`: then the text is
tokenized on the host and encoded by sm_90a kernels (RMSNorm, the fused q|k|v / feed-forward GEMMs, relative-position-bias attention),
and no HF model is built or called:

    t5.T5_CONFIGS[name] = {"native": T5Encoder.from_hf(T5EncoderModel.from_pretrained(name)).cuda(), "tokenizer": tok}
"""
import math

import torch
from torch import nn

DEFAULT_T5_NAME = "google/t5-v1_1-base"
MAX_LENGTH = 256

# name -> {"config": object with .d_model} ; pre-seed to stay offline, e.g. T5_CONFIGS["t5-small"] = {"d_model": 512};
# {"native": T5Encoder, "tokenizer": ...} routes t5_encode_text through libmmg
T5_CONFIGS = {}

_KNOWN_DIMS = {"t5-small": 512, "t5-base": 768, "t5-large": 1024, "t5-3b": 1024, "t5-11b": 1024,
               "google/t5-v1_1-small": 512, "google/t5-v1_1-base": 768, "google/t5-v1_1-large": 1024,
               "google/t5-v1_1-xl": 2048, "google/t5-v1_1-xxl": 4096}


def get_encoded_dim(name):
    entry = T5_CONFIGS.get(name)
    if entry is not None:
        if "native" in entry:
            return entry["native"].d_model
        if "d_model" in entry:
            return entry["d_model"]
        if "config" in entry:
            return entry["config"].d_model
        if "model" in entry:
            return entry["model"].config.d_model
    if name in _KNOWN_DIMS:
        return _KNOWN_DIMS[name]
    from transformers import T5Config          # needs a local HF cache; same behaviour as the reference
    cfg = T5Config.from_pretrained(name)
    T5_CONFIGS[name] = dict(config=cfg)
    return cfg.d_model


def _tokenize(tok, texts, dev):
    enc = tok.batch_encode_plus(texts, return_tensors="pt", padding="longest", max_length=MAX_LENGTH, truncation=True)
    return enc.input_ids.to(dev), enc.attention_mask.to(dev)


def t5_encode_text(texts, name=DEFAULT_T5_NAME, output_device=None):
    """ref: t5.py:60-99 — tokenizer + encoder, padded positions zero-filled.  With a "native" entry the encoder is libmmg's T5Encoder."""
    entry = T5_CONFIGS.get(name)
    if entry is not None and "native" in entry:
        enc = entry["native"]
        if entry.get("tokenizer") is None:
            from transformers import T5Tokenizer
            entry["tokenizer"] = T5Tokenizer.from_pretrained(name)
        ids, attn = _tokenize(entry["tokenizer"], texts, enc.shared.weight.device)
        out = enc(ids, attn)                              # padding rows are written as zeros by the final RMSNorm
        return out if output_device is None else out.to(output_device)
    from transformers import T5Tokenizer, T5EncoderModel
    entry = T5_CONFIGS.setdefault(name, {})
    if "model" not in entry:
        entry["model"] = T5EncoderModel.from_pretrained(name)
        entry["tokenizer"] = T5Tokenizer.from_pretrained(name)
    model, tok = entry["model"], entry["tokenizer"]
    if torch.cuda.is_available():
        model = model.cuda()
    dev = next(model.parameters()).device
    ids, attn = _tokenize(tok, texts, dev)
    model.eval()
    with torch.no_grad():
        out = model(input_ids=ids, attention_mask=attn).last_hidden_state.detach()
    out = out.masked_fill(~attn.bool()[..., None], 0.)
    return out if output_device is None else out.to(output_device)


# ------------------------------------------------------------------------------------------------ native encoder
def relative_position_bucket(relative_position, num_buckets=32, max_distance=128):
    """T5's bidirectional relative-position bucket (HF T5Attention._relative_position_bucket, bidirectional=True), on the host:
    int64 buckets of an integer tensor of key - query offsets, with HF's fp32 log arithmetic."""
    rp = torch.as_tensor(relative_position, dtype=torch.long)
    nb = num_buckets // 2
    buckets = (rp > 0).to(torch.long) * nb
    rp = rp.abs()
    max_exact = nb // 2
    is_small = rp < max_exact
    large = max_exact + (torch.log(rp.float() / max_exact) / math.log(max_distance / max_exact) * (nb - max_exact)).to(torch.long)
    large = torch.minimum(large, torch.full_like(large, nb - 1))
    return buckets + torch.where(is_small, rp, large)


class _W(nn.Module):
    """One bias-free weight under HF's `<name>.weight` key (q / k / v / o, wi / wi_0 / wi_1 / wo, layer_norm, embeddings)."""
    def __init__(self, *shape, ones=False):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(shape) if ones else torch.empty(shape))


def _t5_config_error(field, value, why):
    from ._lib import MMGError
    return MMGError(f"T5Encoder: unsupported config {field}={value!r}: {why}")


class T5Encoder(nn.Module):
    """HF `T5EncoderModel` (eval mode) on libmmg: the same state_dict keys (`shared.weight` and `encoder.embed_tokens.weight` are one tensor),
    `forward(input_ids (B, T) int64, attention_mask (B, T)) -> (B, T, d_model)` fp32 with padding rows zero.

    precision "bf16" (default): bf16 GEMM operands on the wgmma path, fp32 residual stream and statistics; "fp32": the products as 3-way bf16
    splits with fp32 accumulation, fp32 attention on the CUDA cores.  Supported: d_kv == 64, d_model and d_ff multiples of 64,
    feed_forward_proj "relu" or "gated-gelu" (every t5 / t5-v1_1 checkpoint but t5-3b and t5-11b, whose d_kv is 128).
    forward() does no host synchronisation and can be captured in a CUDA graph once it has run eagerly at that sequence length (the packed
    weights and the per-length bucket map are built on the first call)."""

    def __init__(self, config, precision=None, init_weights=True):
        super().__init__()
        g = lambda k, default=None: getattr(config, k, default)
        d, d_kv, d_ff, heads, layers = g("d_model"), g("d_kv"), g("d_ff"), g("num_heads"), g("num_layers")
        ffp = g("feed_forward_proj", "relu")
        if d_kv != 64:
            raise _t5_config_error("d_kv", d_kv, "the attention kernel takes 64-wide heads only")
        for field, v in (("d_model", d), ("d_ff", d_ff)):
            if not isinstance(v, int) or v <= 0 or v % 64:
                raise _t5_config_error(field, v, "must be a positive multiple of 64 (wgmma GEMM tiles)")
        if not isinstance(heads, int) or heads <= 0:
            raise _t5_config_error("num_heads", heads, "must be positive")
        if ffp not in ("relu", "gated-gelu"):
            raise _t5_config_error("feed_forward_proj", ffp, 'only "relu" and "gated-gelu" are implemented')
        self.precision = precision or "bf16"
        if self.precision not in ("bf16", "fp32"):
            raise _t5_config_error("precision", self.precision, 'must be "bf16" or "fp32"')
        self.config = config
        self.d_model, self.d_ff, self.heads, self.num_layers = d, d_ff, heads, layers
        self.gated = ffp == "gated-gelu"
        self.num_buckets = g("relative_attention_num_buckets", 32)
        self.max_distance = g("relative_attention_max_distance", 128)
        self.eps = float(g("layer_norm_epsilon", 1e-6))
        inner = heads * 64

        self.shared = _W(g("vocab_size"), d)
        self.encoder = nn.Module()
        self.encoder.embed_tokens = self.shared               # tied: both keys name one tensor, as in HF
        self.encoder.block = nn.ModuleList()
        for i in range(layers):
            attn = nn.Module()
            attn.q, attn.k, attn.v, attn.o = _W(inner, d), _W(inner, d), _W(inner, d), _W(d, inner)
            if i == 0:
                attn.relative_attention_bias = _W(self.num_buckets, heads)
            ff = nn.Module()
            if self.gated:
                ff.wi_0, ff.wi_1 = _W(d_ff, d), _W(d_ff, d)
            else:
                ff.wi = _W(d_ff, d)
            ff.wo = _W(d, d_ff)
            l0, l1 = nn.Module(), nn.Module()
            l0.SelfAttention, l0.layer_norm = attn, _W(d, ones=True)
            l1.DenseReluDense, l1.layer_norm = ff, _W(d, ones=True)
            blk = nn.Module()
            blk.layer = nn.ModuleList([l0, l1])
            self.encoder.block.append(blk)
        self.encoder.final_layer_norm = _W(d, ones=True)
        if init_weights:
            with torch.no_grad():
                for name, p in self.named_parameters():
                    if "layer_norm" not in name:
                        p.normal_(0.0, d ** -0.5)
        self._pack = None
        self._buckets = {}
        self.register_load_state_dict_post_hook(lambda m, _inc: m._invalidate())

    @classmethod
    def from_hf(cls, model, precision=None):
        """A T5Encoder holding a copy of the weights of a loaded HF `T5EncoderModel`, on the model's device."""
        enc = cls(model.config, precision=precision, init_weights=False)
        enc.load_state_dict(model.state_dict(), strict=True)
        return enc.to(next(model.parameters()).device)

    # ----- packing (the pattern of Transformer: lazy, through pack_cache, dropped after load_state_dict / .to() / in-place edits) -------
    def _invalidate(self):
        self._pack = None
        self._buckets = {}

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def _weights_sig(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _packed(self):
        from . import pack_cache
        from ._lib import MMGError
        sig = self._weights_sig()
        if self._pack is not None and self._pack["sig"] == sig:
            return self._pack
        dev = self.shared.weight.device
        if dev.type != "cuda":
            raise MMGError("T5Encoder runs on CUDA only (libmmg.so); there is no CPU path: move it with .cuda()")
        P = pack_cache.load_or_build("t5_encoder", self, (self.precision, self.gated), self._build_pack, dev)
        P["sig"] = sig
        self._pack = P
        return P

    def _build_pack(self):
        dev = self.shared.weight.device
        adt = torch.bfloat16 if self.precision == "bf16" else torch.float32
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        wa = lambda t: t.detach().to(dev, adt).contiguous()
        layers = []
        for blk in self.encoder.block:
            sa, ff = blk.layer[0].SelfAttention, blk.layer[1].DenseReluDense
            if self.gated:
                # rows interleaved in blocks of 32, [wi_0 (gelu arm) | wi_1 (linear arm)], for the GEGLU_TANH epilogue
                w0, w1 = ff.wi_0.weight.detach(), ff.wi_1.weight.detach()
                wi = torch.stack((w0.reshape(-1, 32, w0.shape[1]), w1.reshape(-1, 32, w1.shape[1])), 1).reshape(-1, w0.shape[1])
            else:
                wi = ff.wi.weight
            layers.append(dict(ln0=f32(blk.layer[0].layer_norm.weight), ln1=f32(blk.layer[1].layer_norm.weight),
                               wqkv=wa(torch.cat((sa.q.weight, sa.k.weight, sa.v.weight), 0)), wo=wa(sa.o.weight), wi=wa(wi), wff=wa(ff.wo.weight)))
        rel = self.encoder.block[0].layer[0].SelfAttention.relative_attention_bias.weight
        return dict(adt=adt, layers=layers, emb=f32(self.shared.weight), rel_bias=f32(rel), lnf=f32(self.encoder.final_layer_norm.weight))

    def _bucket_map(self, T, dev):
        """int32 [2T-1] on the device: bucket of the offset key - query at index key - query + T - 1 (cached per T)."""
        b = self._buckets.get(T)
        if b is None:
            b = relative_position_bucket(torch.arange(-(T - 1), T), self.num_buckets, self.max_distance).to(torch.int32).to(dev)
            self._buckets[T] = b
        return b

    # ----- forward ------------------------------------------------------------------------------------------------------------------------
    def forward(self, input_ids, attention_mask=None):
        from . import ops
        from ._lib import MMGError
        P = self._packed()
        dev, adt = P["emb"].device, P["adt"]
        B, T = input_ids.shape
        if not 1 <= T <= 512:
            raise MMGError(f"T5Encoder: sequence length {T} not in [1, 512]")
        d, inner, R = self.d_model, self.heads * 64, B * T
        ids = input_ids.to(dev, torch.int64).contiguous().view(-1)
        mask = None if attention_mask is None else (attention_mask.to(dev) != 0).to(torch.uint8).contiguous()
        bucket = self._bucket_map(T, dev)
        x = torch.empty((R, d), device=dev, dtype=torch.float32)              # fp32 residual stream
        ops.embed(ids, P["emb"], None, x, n=T, use_pos=False)
        xn = torch.empty((R, d), device=dev, dtype=adt)
        qkv = torch.empty((R, 3 * inner), device=dev, dtype=adt)
        ao = torch.empty((R, inner), device=dev, dtype=adt)
        h = torch.empty((R, self.d_ff), device=dev, dtype=adt)
        for L in P["layers"]:
            ops.rmsnorm(x, L["ln0"], xn, self.eps)
            ops.linear(xn, L["wqkv"], qkv)
            ops.t5_attention(qkv, ao, B, T, self.heads, bucket, P["rel_bias"], mask)
            ops.linear(ao, L["wo"], x, ops.EPI_RESIDUAL, resid=x)
            ops.rmsnorm(x, L["ln1"], xn, self.eps)
            if self.gated:
                ops.linear(xn, L["wi"], h, ops.EPI_GEGLU_TANH)
            else:
                ops.linear(xn, L["wi"], h, ops.EPI_STORE, act=2)
            ops.linear(h, L["wff"], x, ops.EPI_RESIDUAL, resid=x)
        y = torch.empty((R, d), device=dev, dtype=torch.float32)
        ops.rmsnorm(x, P["lnf"], y, self.eps, row_mask=None if mask is None else mask.view(-1))
        return y.view(B, T, d)

"""Thin tensor-level wrappers over the C-ABI (one Python function per mmg_* entry point).  PyTorch supplies device
memory and the stream; every number is computed by libmmg.so."""
import os

import torch

from . import _lib as L
from ._lib import (F32, BF16, EPI_STORE, EPI_RESIDUAL, EPI_GEGLU, EPI_GLU, EPI_QKV, EPI_CONVT, EPI_CONVT_RGB,  # noqa: F401
                   EPI_LNFOLD_RESIDUAL, EPI_LFQ_IDS, EPI_ARGMIN)


def _chk(t, name="tensor"):
    assert t.is_cuda and t.is_contiguous(), f"{name} must be a contiguous CUDA tensor"
    return t


def _epi(out=None, ldo=0, bias=None, act=0, resid=None, ldr=0, row_stats=None, ln_width=0):
    e = L.EpilogueArgs()
    e.row_stats = L.ptr(row_stats); e.ln_width = ln_width
    if row_stats is not None:                     # [M, slots, 2] per-chunk partials (GEGLU writes, LNFOLD reads); [M, 2] = one slot of totals
        e.stats_slots = row_stats.shape[1] if row_stats.dim() == 3 else 1
    if out is not None:
        e.out = out.data_ptr(); e.ldo = ldo
        e.out_dtype = L.dt(out) if out.dtype in (torch.float32, torch.bfloat16) else L.F32     # int64 outputs (LFQ ids / argmin keys)
    e.act = act
    e.bias = L.ptr(bias)
    if resid is not None:
        e.resid = resid.data_ptr(); e.ldr = ldr
    return e


# ---- fp32 on the tensor cores ---------------------------------------------------------------------------------------------
# precision="fp32" (the token-identical parity mode) runs its matrix products and convolutions on the SAME wgmma kernels as the bf16 path:
# both operands are split into three bf16 terms (mmg_split3) and one bf16 product over 6K columns accumulates the six significant cross
# terms in fp32.  Shapes the TMA path cannot take (K or N not a multiple of 64) stay on the CUDA-core kernel.  MMG_FP32_TC=0 / fp32_tc(False)
# forces the CUDA-core kernel everywhere (the round-1 behaviour).
_FP32_TC = [os.environ.get("MMG_FP32_TC", "1") != "0"]


def fp32_tc(enabled=None):
    """Query / set whether fp32 matrix products run as 3-way bf16 splits on the tensor cores."""
    if enabled is not None:
        _FP32_TC[0] = bool(enabled)
    return _FP32_TC[0]


def split3(src2d, side, out=None):
    """src2d [rows, K] fp32 (row stride allowed) -> [rows, 6K] bf16 terms, ordered for `side` (0 left operand, 1 right operand)."""
    assert src2d.dtype == torch.float32 and src2d.dim() == 2 and src2d.stride(1) == 1
    rows, K = src2d.shape
    if out is None:
        out = torch.empty((rows, 6 * K), device=src2d.device, dtype=torch.bfloat16)
    a = L.Split3Args()
    a.src = src2d.data_ptr(); a.dst = out.data_ptr(); a.rows = rows; a.K = K; a.lds = src2d.stride(0) if rows > 1 else K; a.side = side
    L.call("mmg_split3", a)
    return out


def _split_weight(w, rows, K):
    """Right-operand split of a packed weight viewed as [rows, K], cached on the tensor (dropped with it; redone after in-place edits)."""
    c = getattr(w, "_mmg_split3", None)
    if c is not None and c[0] == (w.data_ptr(), w._version, rows, K):
        return c[1]
    s3 = split3(w.reshape(rows, K), 1)
    try:
        w._mmg_split3 = ((w.data_ptr(), w._version, rows, K), s3)
    except AttributeError:
        pass
    return s3


def linear(a, w, out, epilogue=EPI_STORE, bias=None, act=0, resid=None, M=None, N=None, epi=None, row_stats=None, ln_width=0):
    """out = a @ w.T (+ epilogue).  a [M, K], w [N, K] same dtype (bf16 -> wgmma, fp32 -> CUDA cores)."""
    _chk(a, "a"); _chk(w, "w")
    assert w.shape[1] == a.shape[1] and a.dtype == w.dtype
    if a.dtype == torch.float32 and _FP32_TC[0] and a.shape[1] % 64 == 0 and (w.shape[0] if N is None else N) % 64 == 0 and a.shape[0] > 0:
        a, w = split3(a, 0), _split_weight(w, w.shape[0], w.shape[1])          # same product, 6K bf16 columns, fp32 accumulation on the tensor cores
    args = L.LinearArgs()
    args.a = a.data_ptr(); args.w = w.data_ptr()
    args.M = a.shape[0] if M is None else M
    args.N = w.shape[0] if N is None else N
    args.K = a.shape[1]; args.lda = a.stride(0); args.ldw = w.stride(0)
    args.dtype = L.dt(a); args.epilogue = epilogue
    if epilogue in (EPI_GEGLU, EPI_GLU) and out is not None:
        assert out.shape[-1] * 2 >= args.N and out.stride(0) * 2 >= args.N, "GEGLU / GLU write N / 2 columns per row: `out` is too narrow"
    if epi is None:
        epi = _epi(out, out.stride(0), bias, act, resid, resid.stride(0) if resid is not None else 0, row_stats, ln_width)
    args.epi = epi
    L.call("mmg_linear", args)
    return out


def qkv_epilogue(dtype_t, heads, tokens, q=None, k=None, v=None, q_scale=None, k_scale=None, key_off=0, null_k=None, null_v=None):
    """Epilogue block for MMG_EPI_QKV.  q [BH, q_rows, 64]; k, v [BH, kv_rows, 64]."""
    e = L.EpilogueArgs()
    e.out_dtype = L.F32 if dtype_t == torch.float32 else L.BF16
    e.heads = heads; e.tokens = tokens; e.key_off = key_off
    if q is not None:
        e.q_out = q.data_ptr(); e.q_scale = q_scale.data_ptr(); e.q_rows = q.shape[1]; e.nq_heads = heads
    if k is not None:
        e.k_out = k.data_ptr(); e.k_scale = k_scale.data_ptr(); e.kv_rows = k.shape[1]; e.nk_heads = heads
        e.v_out = v.data_ptr(); e.nv_heads = heads
        e.null_k = L.ptr(null_k); e.null_v = L.ptr(null_v)
    return e


def conv2d(x, w, out, B, H, W, Cin, Cout, kind, epilogue=EPI_STORE, bias=None, act=0, resid=None):
    """x [B,H,W,Cin] NHWC, w packed [Cout, taps*Cin]; out rows = output pixels."""
    _chk(x); _chk(w)
    if x.dtype == torch.float32 and _FP32_TC[0] and Cin % 32 == 0 and Cout % 64 == 0 and kind != 3:
        # per-pixel / per-tap split: 6*Cin channels (a multiple of 64), the same implicit GEMM
        x, w, Cin = split3(x.reshape(-1, Cin), 0), _split_weight(w, w.numel() // Cin, Cin), 6 * Cin
    a = L.Conv2dArgs()
    a.x = x.data_ptr(); a.w = w.data_ptr(); a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.kind = kind
    a.dtype = L.dt(x); a.epilogue = epilogue
    ldo = out.shape[-1]
    a.epi = _epi(out, ldo, bias, act, resid, resid.shape[-1] if resid is not None else 0)
    L.call("mmg_conv2d", a)
    return out


def conv_transpose2d(x, w, out, B, H, W, Cin, Cout, bias=None, rgb_w=None, rgb_b=None):
    """ConvTranspose2d(4,2,1) + LeakyReLU(0.1); with rgb_w: fused trailing 1x1 conv, out fp32 [B, ch, 2H, 2W]."""
    _chk(x); _chk(w)
    if x.dtype == torch.float32 and _FP32_TC[0] and Cin % 32 == 0 and Cout % 64 == 0:
        x, w, Cin = split3(x.reshape(-1, Cin), 0), _split_weight(w, w.numel() // Cin, Cin), 6 * Cin
    a = L.ConvTranspose2dArgs()
    a.x = x.data_ptr(); a.w = w.data_ptr(); a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout
    a.dtype = L.dt(x)
    e = L.EpilogueArgs()
    e.out = out.data_ptr(); e.bias = L.ptr(bias)
    if rgb_w is not None:
        a.epilogue = EPI_CONVT_RGB
        e.out_dtype = L.F32; e.rgb_w = rgb_w.data_ptr(); e.rgb_b = rgb_b.data_ptr(); e.rgb_channels = rgb_w.shape[0]
    else:
        a.epilogue = EPI_CONVT
        e.out_dtype = L.dt(out); e.ldo = Cout
    a.epi = e
    L.call("mmg_conv_transpose2d", a)
    return out


def conv_in(img, w, bias, out, ksize=5):
    a = L.ConvInArgs()
    a.ksize = ksize
    assert tuple(w.shape[2:]) == (ksize, ksize)
    B, Cc, H, W = img.shape
    a.img = _chk(img).data_ptr(); a.w = _chk(w).data_ptr(); a.bias = L.ptr(bias); a.out = out.data_ptr()
    a.B = B; a.C = Cc; a.H = H; a.W = W; a.Cout = w.shape[0]; a.out_dtype = L.dt(out)
    L.call("mmg_conv_in", a)
    return out


def groupnorm_(x, gamma, beta, B, HW, Cch, groups=16, act=0):
    a = L.GroupNormArgs()
    a.x = _chk(x).data_ptr(); a.gamma = gamma.data_ptr(); a.beta = beta.data_ptr()
    a.B = B; a.HW = HW; a.C = Cch; a.groups = groups; a.dtype = L.dt(x); a.act = act
    L.call("mmg_groupnorm", a)
    return x


def layernorm(x, gamma, y, width=None, add=None, x_out=None, rows=None, zero_stats=None, add_from=0):
    a = L.LayerNormArgs()
    a.zero_stats = L.ptr(zero_stats); a.add_from = add_from
    a.x = _chk(x).data_ptr(); a.x_dtype = L.dt(x); a.y = _chk(y).data_ptr(); a.y_dtype = L.dt(y)
    a.gamma = gamma.data_ptr(); a.add = L.ptr(add); a.x_out = L.ptr(x_out)
    a.rows = x.shape[0] if rows is None else rows
    a.width = x.shape[1] if width is None else width
    a.ldx = x.stride(0); a.ldy = y.stride(0)
    L.call("mmg_layernorm", a)
    return y


def embed(ids, token_emb, pos_emb, x, n, copies=1, use_pos=True):
    a = L.EmbedArgs()
    a.ids = _chk(ids).data_ptr(); a.token_emb = token_emb.data_ptr(); a.pos_emb = L.ptr(pos_emb); a.x = x.data_ptr()
    a.rows = ids.numel(); a.n = n; a.dim = token_emb.shape[1]; a.copies = copies; a.use_pos = int(use_pos)
    L.call("mmg_embed", a)
    return x


def attention(q, k, v, out, B, heads, Tk, key_mask=None, kv_shared=False, scale=8.0, logit_bound=0.0):
    """q [B*heads, Tq, 64]; k, v [(B or 1)*heads, Tk_alloc, 64]; out [B*Tq, heads*64]."""
    a = L.AttentionArgs()
    _chk(q); _chk(k); _chk(v)
    Tq, Tk_alloc, dtype = q.shape[1], k.shape[1], L.dt(q)
    if q.dtype == torch.float32 and _FP32_TC[0] and 2 <= Tk <= 4096 and out.dtype == torch.float32 and out.stride(0) % 8 == 0:
        # fp32 parity on the tensor cores: three bf16 terms per operand, six cross terms per product (mmg_attention_split.cuh)
        q, k, v = split3(q.view(-1, 64), 0), split3(k.view(-1, 64), 1), split3(v.view(-1, 64), 1)
        dtype = L.BF16; a.split3 = 1
    a.q = q.data_ptr(); a.k = k.data_ptr(); a.v = v.data_ptr(); a.out = out.data_ptr()
    a.key_mask = L.ptr(key_mask)
    a.B = B; a.heads = heads; a.Tq = Tq; a.Tk = Tk; a.Tk_alloc = Tk_alloc; a.dtype = dtype
    a.ldo = out.stride(0); a.kv_batch_stride_zero = int(kv_shared); a.scale = scale; a.logit_bound = logit_bound
    L.call("mmg_attention", a)
    return out


def remask(ids, scores, masked_pos, num_masked, mask_id):
    a = L.RemaskArgs()
    a.ids = ids.data_ptr(); a.scores = scores.data_ptr(); a.masked_pos = masked_pos.data_ptr()
    a.B, a.n = ids.shape; a.num_masked = num_masked; a.mask_id = mask_id
    L.call("mmg_remask", a)


def final_embed(x_cond, x_null, gamma, masked_pos, e, B, n, num_masked, cond_scale):
    a = L.FinalEmbedArgs()
    a.x_cond = x_cond.data_ptr(); a.x_null = L.ptr(x_null); a.gamma = gamma.data_ptr(); a.masked_pos = masked_pos.data_ptr()
    a.e = e.data_ptr(); a.e_dtype = L.dt(e); a.B = B; a.n = n; a.num_masked = num_masked; a.dim = gamma.shape[0]
    a.cond_scale = cond_scale
    L.call("mmg_final_embed", a)
    return e


def logits_sample(logits, masked_pos, ids, scores, num_masked, k, temperature, u=None, seed=0, step=0, row_offset=0, seed_dev=None,
                  only_masked_id=None, aten=None):
    """aten = (offset, offset_dev, stride): draw the noise from ATen's CUDA uniform_ stream instead of libmmg's keying."""
    a = L.LogitsSampleArgs()
    a.logits = _chk(logits).data_ptr(); a.masked_pos = masked_pos.data_ptr(); a.ids = ids.data_ptr(); a.scores = scores.data_ptr()
    a.u = L.ptr(u)
    a.B, a.n = ids.shape; a.num_masked = num_masked; a.V = logits.shape[-1]; a.k = k; a.temperature = temperature
    a.seed = seed; a.step = step; a.row_offset = row_offset; a.seed_dev = L.ptr(seed_dev)
    if only_masked_id is not None:
        a.only_masked = 1; a.mask_id = only_masked_id
    if aten is not None:
        a.rng_mode = 1; a.aten_offset = aten[0]; a.aten_offset_dev = L.ptr(aten[1]); a.aten_stride = aten[2]
    L.call("mmg_logits_sample", a)


def logits_fused_workspace_bytes(rows_capacity, V, K, k):
    """Bytes of workspace mmg_logits_fused needs for up to `rows_capacity` sampled rows; 0 = shape not supported by the fused path."""
    return int(L.lib().mmg_logits_fused_workspace_bytes(int(rows_capacity), int(V), int(K), int(k)))


def logits_fused(e, w, masked_pos, ids, scores, num_masked, k, temperature, workspace, status, rows_capacity=0, u=None, seed=0, step=0,
                 row_offset=0, seed_dev=None, only_masked_id=None, aten=None):
    """to_logits + top-k / gumbel argmax / confidence on the rows listed in masked_pos without a [rows, V] logits buffer."""
    a = L.LogitsFusedArgs()
    a.e = _chk(e).data_ptr(); a.w = _chk(w).data_ptr(); a.K = e.shape[1]; a.rows_capacity = rows_capacity
    assert e.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and w.shape[1] == e.shape[1]
    a.workspace = workspace.data_ptr(); a.workspace_bytes = workspace.numel() * workspace.element_size(); a.status = status.data_ptr()
    s = a.s
    s.masked_pos = masked_pos.data_ptr(); s.ids = ids.data_ptr(); s.scores = scores.data_ptr(); s.u = L.ptr(u)
    s.B, s.n = ids.shape; s.num_masked = num_masked; s.V = w.shape[0]; s.k = k; s.temperature = temperature
    s.seed = seed; s.step = step; s.row_offset = row_offset; s.seed_dev = L.ptr(seed_dev)
    if only_masked_id is not None:
        s.only_masked = 1; s.mask_id = only_masked_id
    if aten is not None:
        s.rng_mode = 1; s.aten_offset = aten[0]; s.aten_offset_dev = L.ptr(aten[1]); s.aten_stride = aten[2]
    L.call("mmg_logits_fused", a)


def critic_score(x_cond, x_null, gamma, w, bias, cond_scale, noise_mul, scores, u=None, seed=0, step=0, row_offset=0, seed_dev=None,
                 aten=None):
    """scores[r] = CFG(dot(LN(x[r]) * gamma, w) + bias) + (u[r] - 0.5) * noise_mul   (ref: muse_maskgit_pytorch.py:590-600)"""
    a = L.CriticScoreArgs()
    a.x_cond = _chk(x_cond).data_ptr(); a.x_null = L.ptr(x_null); a.gamma = gamma.data_ptr(); a.w = _chk(w).data_ptr()
    a.bias = bias; a.cond_scale = cond_scale; a.noise_mul = noise_mul; a.dim = x_cond.shape[-1]
    a.u = L.ptr(u); a.scores = scores.data_ptr(); a.rows = scores.numel(); a.row_offset = row_offset
    a.seed = seed; a.seed_dev = L.ptr(seed_dev); a.step = step
    assert x_cond.dtype == torch.float32 and w.dtype == torch.float32 and x_cond.shape[0] >= a.rows
    if aten is not None:
        a.rng_mode = 1; a.aten_offset = aten[0]; a.aten_offset_dev = L.ptr(aten[1]); a.aten_stride = aten[2]
    L.call("mmg_critic_score", a)
    return scores


def ff_geglu(x, ln_gamma, w1, w2f, cvec, F, xn, h, stats, add=None, add_from=0):
    """x += FeedForward(x) in place (one C call = LayerNorm + GEGLU GEMM + LN-folded GEMM); bf16 operands, fp32 residual stream."""
    a = L.FfGegluArgs()
    a.x = _chk(x).data_ptr(); a.rows, a.dim = x.shape; a.F = F; a.Fp = w2f.shape[1]
    a.ln_gamma = ln_gamma.data_ptr(); a.w1 = _chk(w1).data_ptr(); a.w2f = _chk(w2f).data_ptr(); a.cvec = cvec.data_ptr()
    a.add = L.ptr(add); a.add_from = add_from
    assert stats.dtype == torch.float32 and stats.numel() >= a.rows * (a.Fp // 32) * 2, "stats: [rows, Fp / 32, 2] fp32 per-chunk partials"
    a.xn = _chk(xn).data_ptr(); a.h = _chk(h).data_ptr(); a.stats = stats.data_ptr()
    assert x.dtype == torch.float32 and w1.dtype == torch.bfloat16 and w1.shape[0] == 2 * a.Fp and tuple(h.shape) == (a.rows, a.Fp)
    L.call("mmg_ff_geglu", a)
    return x


def vq_lfq_encode(x, w_in, b_in, ids, bits, w_split=None):
    """w_split: [64, D] bf16 3-way split of w_in -> bf16 tokens take the wgmma route (one TMA stream over the tokens)."""
    a = L.LfqEncodeArgs()
    a.x = _chk(x).data_ptr(); a.dtype = L.dt(x); a.w_in = L.ptr(w_in); a.b_in = L.ptr(b_in); a.ids = ids.data_ptr()
    a.w_split = L.ptr(w_split)
    a.T = x.shape[0]; a.D = x.shape[1]; a.bits = bits
    L.call("mmg_vq_lfq_encode", a)
    return ids


def vq_l2_argmin(x, codebook, ids):
    a = L.L2ArgminArgs()
    a.x = _chk(x).data_ptr(); a.codebook = _chk(codebook).data_ptr(); a.ids = ids.data_ptr()
    a.T = x.shape[0]; a.K = codebook.shape[0]; a.D = x.shape[1]
    L.call("mmg_vq_l2_argmin", a)
    return ids


def vq_decode_codes(ids, w_out, b_out, out, bits):
    a = L.DecodeCodesArgs()
    a.ids = _chk(ids).data_ptr(); a.w_out = L.ptr(w_out); a.b_out = L.ptr(b_out); a.out = out.data_ptr()
    a.dtype = L.dt(out); a.T = ids.numel(); a.D = out.shape[-1]; a.bits = bits
    L.call("mmg_vq_decode_codes", a)
    return out

"""Transformer / MaskGitTransformer / TokenCritic / MaskGit / Muse — host-side mirror of the reference classes
(ref: muse_maskgit_pytorch.py:199-386, 427-791) over libmmg.so.

The nn.Modules here only HOLD parameters under the reference's state_dict keys (SURVEY.md 8b); the arithmetic of
`forward`, `forward_with_cond_scale` and `MaskGit.generate` is issued as sm_90a kernels through the C-ABI:
  wgmma GEMMs with fused epilogues (QKV split + l2norm/scale, residual, GEGLU), wgmma attention, LayerNorm,
  the masked-row final-LN + CFG combine, the logits GEMM on masked rows only, and the fused sampling tail.
Both CFG branches of a decode step run as one batch of 2B sequences; the null branch's cross-attention is the
constant to_out(null_v) (every text key masked -> softmax puts weight exactly 1 on the null key, SURVEY.md 8a T3).
"""
import ctypes
import dataclasses
import math
import numbers
import os
import random
from functools import partial
from pathlib import Path
from typing import Callable, List, NamedTuple, Optional

import torch
from torch import nn

from . import ops, _lib, pack_cache
from .t5 import t5_encode_text, get_encoded_dim, DEFAULT_T5_NAME
from .vqgan_vae import VQGanVAE


def _round_up(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ parameter holders
class LayerNorm(nn.Module):
    """gamma parameter + zero `beta` buffer (ref: muse_maskgit_pytorch.py:63-67)."""
    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.register_buffer("beta", torch.zeros(dim))


def _geglu_interleave(w1, Fp):
    """(2F, K) feed-forward weight (rows [0, F) gelu arm, [F, 2F) gate) -> (2 Fp, K) in the GEGLU epilogue's row order: arm unit u at row
    64 (u // 32) + u % 32, its gate 32 rows further; the padding rows past F are zero.  Works on a trailing-dim-free (2F,) vector too."""
    F_ = w1.shape[0] // 2
    out = torch.zeros((2 * Fp,) + tuple(w1.shape[1:]), device=w1.device, dtype=w1.dtype)
    xi = torch.arange(Fp, device=w1.device).view(-1, 32)
    dst_x = (xi // 32 * 64 + xi % 32).reshape(-1)                       # unit u -> row 64*(u//32) + u%32 ; gate -> +32
    valid = torch.arange(Fp, device=w1.device) < F_
    out[dst_x[valid]] = w1[:F_]
    out[dst_x[valid] + 32] = w1[F_:]
    return out


def quantize_rows_e4m3(w):
    """Per-row e4m3 quantisation of an fp32 matrix (precision="fp8" weights, and the rounding of mmg_layernorm_fp8):
    amax = max |w[r]|, q[r] = rne_satfinite_e4m3(w[r] * (448 / amax)) (0 where amax == 0), scale[r] = amax / 448, so q * scale ~= w.
    Returns (q float8_e4m3fn, scale fp32)."""
    w = w.float()
    amax = w.abs().amax(dim=1)
    inv = torch.where(amax > 0, 448.0 / torch.where(amax > 0, amax, torch.ones_like(amax)), torch.zeros_like(amax))
    q = (w * inv[:, None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)     # clamp first: the cast of a value past 448 is NaN
    return q.contiguous(), (amax / 448.0).contiguous()


def _ff_params(dim, mult=4):
    inner = int(dim * mult * 2 / 3)                       # ref: muse_maskgit_pytorch.py:82
    return nn.Sequential(LayerNorm(dim), nn.Linear(dim, inner * 2, bias=False), nn.Identity(), LayerNorm(inner),
                         nn.Linear(inner, dim, bias=False))


class Attention(nn.Module):
    def __init__(self, dim, dim_head=64, heads=8, cross_attend=False, scale=8):
        super().__init__()
        inner = dim_head * heads
        self.scale, self.heads, self.cross_attend = scale, heads, cross_attend
        self.norm = LayerNorm(dim)
        self.null_kv = nn.Parameter(torch.randn(2, heads, 1, dim_head))
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_kv = nn.Linear(dim, inner * 2, bias=False)
        self.q_scale = nn.Parameter(torch.ones(dim_head))
        self.k_scale = nn.Parameter(torch.ones(dim_head))
        self.to_out = nn.Linear(inner, dim, bias=False)


class TransformerBlocks(nn.Module):
    def __init__(self, *, dim, depth, dim_head=64, heads=8, ff_mult=4, flash=True):
        super().__init__()
        if dim_head not in (64, 128):
            raise ValueError(f"dim_head must be 64 or 128 here (got {dim_head}): the QKV epilogues and the attention kernels are written for "
                             "those two head sizes; the reference accepts any value (muse_maskgit_pytorch.py:95-110, 164-172)")
        if dim_head == 128 and dim % 64 != 0:
            raise ValueError(f"dim_head=128 needs dim % 64 == 0 (got dim = {dim}): the 128-wide QKV epilogue runs on the wgmma product only, "
                             "whose k-blocks are 64 wide")
        self.dim, self.depth, self.heads, self.dim_head, self.ff_mult = dim, depth, heads, dim_head, ff_mult
        self.layers = nn.ModuleList([nn.ModuleList([Attention(dim, dim_head, heads), Attention(dim, dim_head, heads, True),
                                                    _ff_params(dim, ff_mult)]) for _ in range(depth)])
        self.norm = LayerNorm(dim)


# ------------------------------------------------------------------------------------------------ transformer
class Transformer(nn.Module):
    def __init__(self, *, num_tokens, dim, seq_len, dim_out=None, t5_name=DEFAULT_T5_NAME, self_cond=False,
                 add_mask_id=False, precision=None, **kwargs):
        super().__init__()
        self.dim = dim
        self.mask_id = num_tokens if add_mask_id else None
        self.num_tokens, self.seq_len = num_tokens, seq_len
        self.token_emb = nn.Embedding(num_tokens + int(add_mask_id), dim)
        self.pos_emb = nn.Embedding(seq_len, dim)
        self.transformer_blocks = TransformerBlocks(dim=dim, **kwargs)
        self.norm = LayerNorm(dim)                       # present in checkpoints, never applied (reference defect B4)
        self.dim_out = dim_out if dim_out is not None else num_tokens
        self.to_logits = nn.Linear(dim, self.dim_out, bias=False)
        self.encode_text = partial(t5_encode_text, name=t5_name)
        text_dim = get_encoded_dim(t5_name)
        self.text_embed_proj = nn.Linear(text_dim, dim, bias=False) if text_dim != dim else nn.Identity()
        self.self_cond = self_cond
        self.self_cond_to_init_embed = _ff_params(dim)
        self.precision = precision or "bf16"
        if self.precision == "fp8" and dim % 128 != 0:
            raise ValueError(f'precision="fp8" needs dim % 128 == 0 (one 128-element e4m3 k-block per wgmma step); got dim = {dim}')
        self._pack = None
        # nn.Module.load_state_dict on a PARENT never calls a child's load_state_dict override, but it does run the child's
        # post hooks: the packed weights are dropped whichever module the load was started from
        self.register_load_state_dict_post_hook(lambda m, _inc: m._invalidate())

    # ----- packing ------------------------------------------------------------------------------------------------
    def _invalidate(self):
        self._pack = None
        self.__dict__.pop("_ws", None)

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def _weights_sig(self):
        """(storage, version) of every parameter: catches in-place edits (`p.data.copy_`, optimizer steps) between calls."""
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _check_weights(self):
        sig = self._weights_sig()
        if self._pack is not None and self._pack.get("sig") != sig:
            self._invalidate()
        return sig

    def _adt(self):
        """operand dtype of every product that is not e4m3: bf16 for "bf16" and "fp8", fp32 (3-way bf16 splits) otherwise"""
        return torch.bfloat16 if self.precision in ("bf16", "fp8") else torch.float32

    def _packed(self):
        if self._pack is not None and self._pack["adt"] == self._adt() and self._pack.get("fp8", False) == (self.precision == "fp8"):
            return self._pack
        dev = self.token_emb.weight.device
        assert dev.type == "cuda", "Transformer runs on CUDA only (libmmg.so); there is no CPU path"
        P = pack_cache.load_or_build("transformer", self, (self.precision, self.dim_out, self.self_cond), self._build_pack, dev)
        P["sig"] = self._weights_sig()
        self._pack = P
        return P

    def _build_pack(self):
        dev = self.token_emb.weight.device
        adt = self._adt()
        tb = self.transformer_blocks
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        wa = lambda t: t.detach().to(dev, adt).contiguous()
        fp8 = self.precision == "fp8"
        P = dict(adt=adt, fp8=fp8, layers=[])

        def ff_pack(ff):
            F_ = ff[3].gamma.shape[0]
            Fp = _round_up(F_, 64)
            w1p = _geglu_interleave(ff[1].weight.detach().to(dev, torch.float32), Fp)   # (2F, dim): rows [0,F) -> gelu arm, [F,2F) -> gate
            g3 = torch.zeros(Fp, device=dev); g3[:F_] = ff[3].gamma.detach().float()
            w2 = torch.zeros((ff[4].weight.shape[0], Fp), device=dev); w2[:, :F_] = ff[4].weight.detach().float()
            out = dict(F=F_, Fp=Fp, g0=f32(ff[0].gamma), w1=w1p.to(adt).contiguous(), g3=g3.contiguous(), w2=w2.to(adt).contiguous())
            if adt == torch.bfloat16:
                # LayerNorm(inner) folded through the second linear: LN(h) W2^T = rstd * (h (W2*gamma)^T - mean * cvec), cvec = rowsum(W2*gamma)
                w2f = (w2 * g3[None, :]).to(adt).contiguous()
                out["w2f"], out["cvec"] = w2f, w2f.float().sum(dim=1).contiguous()
            if fp8:      # FF1 on e4m3: rows quantised after the interleave, so the scales follow it
                out["w1_8"], out["s1"] = quantize_rows_e4m3(w1p)
                del out["w1"]
            return out

        for attn, cross, ff in tb.layers:
            h = attn.heads
            lay = dict(
                sa=dict(g=f32(attn.norm.gamma), wqkv=wa(torch.cat((attn.to_q.weight, attn.to_kv.weight), 0)), wo=wa(attn.to_out.weight),
                        qs=f32(attn.q_scale), ks=f32(attn.k_scale),
                        bound=1.02 * float((attn.q_scale.detach().abs() * attn.k_scale.detach().abs()).max()),   # |q.k| <= max_i|qs_i ks_i| for unit q, k (+ bf16 slack)
                        nk=(torch.nn.functional.normalize(attn.null_kv[0].detach().float(), dim=-1) * attn.k_scale.detach().float()).to(dev, adt).contiguous(),
                        nv=attn.null_kv[1].detach().to(dev, adt).contiguous()),
                ca=dict(g=f32(cross.norm.gamma), wq=wa(cross.to_q.weight), wkv=wa(cross.to_kv.weight), wo=wa(cross.to_out.weight),
                        qs=f32(cross.q_scale), ks=f32(cross.k_scale),
                        bound=1.02 * float((cross.q_scale.detach().abs() * cross.k_scale.detach().abs()).max()),
                        nk=(torch.nn.functional.normalize(cross.null_kv[0].detach().float(), dim=-1) * cross.k_scale.detach().float()).to(dev, adt).contiguous(),
                        nv=cross.null_kv[1].detach().to(dev, adt).contiguous(),
                        # cross-attention output when every context key is masked: to_out(null_v)  (weight 1.0 on the null key)
                        null_out=f32(cross.null_kv[1].detach().float().reshape(1, -1) @ cross.to_out.weight.detach().float().t()).reshape(-1)),
                ff=ff_pack(ff))
            if fp8:      # self QKV and cross q on e4m3, one scale per output row
                lay["sa"]["wqkv_8"], lay["sa"]["s_qkv"] = quantize_rows_e4m3(lay["sa"].pop("wqkv"))
                lay["ca"]["wq_8"], lay["ca"]["s_q"] = quantize_rows_e4m3(lay["ca"].pop("wq"))
            P["layers"].append(lay)
        P["gf"] = f32(tb.norm.gamma)
        P["tok"], P["pos"] = f32(self.token_emb.weight), f32(self.pos_emb.weight)
        P["wlog"] = wa(self.to_logits.weight)
        P["whead"] = f32(self.to_logits.weight).reshape(-1) if self.dim_out == 1 else None     # TokenCritic head, applied in mmg_critic_score
        P["wproj"] = wa(self.text_embed_proj.weight) if isinstance(self.text_embed_proj, nn.Linear) else None
        P["sc"] = ff_pack(self.self_cond_to_init_embed) if self.self_cond else None
        return P

    # ----- context (text / conditioning tokens): computed once per generate() ----------------------------------------
    def _prepare_context(self, text_embeds, cond_ids, branches):
        """Returns per-layer cross K/V buffers and the key mask for `branches` = list of drop flags (False = cond, True = text
        dropped).  ref: muse_maskgit_pytorch.py:302-318."""
        P = self._packed()
        adt, dev = P["adt"], text_embeds.device
        tb = self.transformer_blocks
        b, m_text, _ = text_embeds.shape
        te = text_embeds.to(torch.float32)
        text_mask = (te != 0).any(dim=-1)                                           # muse_maskgit_pytorch.py:304
        te_a = te.reshape(b * m_text, -1).to(adt).contiguous()
        if P["wproj"] is not None:
            ctx = torch.empty((b * m_text, self.dim), device=dev, dtype=adt)
            ops.linear(te_a, P["wproj"], ctx)
        else:
            ctx = te_a
        m = m_text
        if cond_ids is not None:
            cond_ids = cond_ids.reshape(b, -1).contiguous()
            mc = cond_ids.shape[1]
            cemb = torch.empty((b * mc, self.dim), device=dev, dtype=torch.float32)
            ops.embed(cond_ids, P["tok"], None, cemb, n=mc, use_pos=False)             # token_emb only, no pos-emb (muse_maskgit_pytorch.py:316)
            ctx = torch.cat((ctx.view(b, m_text, -1), cemb.to(adt).view(b, mc, -1)), dim=1).reshape(b * (m_text + mc), -1).contiguous()
            m = m_text + mc
        masks = []
        for drop in branches:
            tm = text_mask & (not drop)
            if cond_ids is not None:
                tm = torch.cat((tm, torch.ones((b, m - m_text), dtype=torch.bool, device=dev)), dim=1)
            masks.append(tm)
        key_mask = torch.cat(masks, 0).to(torch.uint8).contiguous()                # [len(branches)*b, m]
        # a branch whose keys are all masked has the constant cross-attention output to_out(null_v): _run_blocks attends over the others
        all_masked = [bool(d) and cond_ids is None for d in branches]
        live = all_masked.count(False)
        assert all_masked == [False] * live + [True] * (len(branches) - live), "live CFG branches must come first"
        heads = tb.heads
        tk_alloc = _round_up(m + 1, 8)
        kvs = []
        for lay in P["layers"]:
            ca = lay["ca"]
            k = torch.zeros((b * heads, tk_alloc, tb.dim_head), device=dev, dtype=adt)
            v = torch.zeros((b * heads, tk_alloc, tb.dim_head), device=dev, dtype=adt)
            epi = ops.qkv_epilogue(adt, heads, m, k=k, v=v, k_scale=ca["ks"], key_off=1, null_k=ca["nk"], null_v=ca["nv"])
            ops.linear(ctx, ca["wkv"], None, epilogue=ops.qkv_kind(k), epi=epi)
            if len(branches) > 1:
                k, v = k.repeat(len(branches), 1, 1), v.repeat(len(branches), 1, 1)
            kvs.append((k, v))
        return dict(kv=kvs, key_mask=key_mask, m=m, live=live)

    # ----- the block stack over R = nb*b*n rows -------------------------------------------------------------------------
    def _workspace(self, nb, b, n, dev):
        key = (nb, b, n, str(dev), self._adt(), self.precision == "fp8")
        cache = self.__dict__.setdefault("_ws", {})        # a few shapes stay resident (e.g. 2-branch decode + 1-branch self-critic)
        if key in cache:
            return cache[key]
        P = self._packed()
        adt, tb = P["adt"], self.transformer_blocks
        heads, dim, dh = tb.heads, self.dim, tb.dim_head
        inner = heads * dh
        R = nb * b * n
        Fp = max([l["ff"]["Fp"] for l in P["layers"]] + ([P["sc"]["Fp"]] if P["sc"] is not None else []))
        tk_alloc = _round_up(n + 1, 8)
        ws = dict(key=key,
                  x=torch.empty((R, dim), device=dev, dtype=torch.float32),
                  xn=torch.empty((R, dim), device=dev, dtype=adt),
                  q=torch.empty((nb * b * heads, n, dh), device=dev, dtype=adt),
                  k=torch.zeros((nb * b * heads, tk_alloc, dh), device=dev, dtype=adt),
                  v=torch.zeros((nb * b * heads, tk_alloc, dh), device=dev, dtype=adt),
                  ao=torch.empty((R, inner), device=dev, dtype=adt),
                  h=torch.empty((R, Fp), device=dev, dtype=adt),
                  hn=torch.empty((R, Fp), device=dev, dtype=adt),
                  stats=torch.zeros((R, Fp // 32, 2), device=dev, dtype=torch.float32))   # per-chunk (sum, sumsq) of the GEGLU output
        if P["fp8"]:     # the quantising LayerNorm's output: e4m3 rows and one scale per row (the A operand of the fp8 products)
            ws["xq"] = torch.empty((R, dim), device=dev, dtype=torch.float8_e4m3fn)
            ws["xs"] = torch.empty((R,), device=dev, dtype=torch.float32)
        if len(cache) >= 4:
            cache.pop(next(iter(cache)))
        cache[key] = ws
        return ws

    def _run_blocks(self, ids, ctx, nb, self_cond_embed=None):
        """ids (b, n) int64 -> residual stream x [nb*b*n, dim] fp32 after all blocks (before the final LayerNorm).
        Branch j occupies rows [j*b*n, (j+1)*b*n).  ref: muse_maskgit_pytorch.py:322-330, 187-193"""
        P = self._packed()
        adt, tb = P["adt"], self.transformer_blocks
        b, n = ids.shape
        assert n <= self.seq_len
        heads = tb.heads
        dev = ids.device
        ws = self._workspace(nb, b, n, dev)
        x, xn, q, k, v, ao = ws["x"], ws["xn"], ws["q"], ws["k"], ws["v"], ws["ao"]
        qkv = ops.qkv_kind(q)
        R, bn = nb * b * n, b * n
        if self.self_cond and self_cond_embed is not None:
            # x += self_cond_to_init_embed(embed of the previous step), identical for every CFG branch (muse_maskgit_pytorch.py:325-328);
            # a missing embed is zeros in the reference and FeedForward(0) == 0 exactly, so that case adds nothing
            ops.embed(ids.contiguous(), P["tok"], P["pos"], x[:bn], n=n, copies=1)
            self._ff(self_cond_embed.reshape(bn, -1).float().contiguous(), P["sc"], x[:bn], ws, bn)
            for j in range(1, nb):
                x[j * bn:(j + 1) * bn].copy_(x[:bn])
        else:
            ops.embed(ids.contiguous(), P["tok"], P["pos"], x, n=n, copies=nb)
        live = min(ctx["live"], nb)
        Rl, ql = live * bn, live * b * heads          # rows and attention batches of the live branches

        def norm(rows, g, fp8, **kw):
            """LayerNorm of x[rows] into the A operand of the next product (xn; fp8: e4m3 rows + row scales)"""
            if fp8:
                ops.layernorm_fp8(x[rows], g, ws["xq"][rows], ws["xs"][rows], **kw)
            else:
                ops.layernorm(x[rows], g, xn[rows], **kw)

        for li, lay in enumerate(P["layers"]):
            sa, ca, ff = lay["sa"], lay["ca"], lay["ff"]
            # --- self attention (all branches) ---
            norm(slice(None), sa["g"], "wqkv_8" in sa)
            epi = ops.qkv_epilogue(adt, heads, n, q=q, k=k, v=v, q_scale=sa["qs"], k_scale=sa["ks"], key_off=1,
                                   null_k=sa["nk"], null_v=sa["nv"])
            if "wqkv_8" in sa:
                ops.linear_fp8(ws["xq"], ws["xs"], sa["wqkv_8"], sa["s_qkv"], None, epilogue=qkv, epi=epi)
            else:
                ops.linear(xn, sa["wqkv"], None, epilogue=qkv, epi=epi)
            ops.attention(q, k, v, ao, nb * b, heads, n + 1, logit_bound=sa["bound"])
            ops.linear(ao, sa["wo"], x, epilogue=ops.EPI_RESIDUAL, resid=x)
            # --- cross attention ---
            kc, vc = ctx["kv"][li]
            if live:
                norm(slice(0, Rl), ca["g"], "wq_8" in ca)
                epi = ops.qkv_epilogue(adt, heads, n, q=q[:ql], q_scale=ca["qs"])
                if "wq_8" in ca:
                    ops.linear_fp8(ws["xq"][:Rl], ws["xs"][:Rl], ca["wq_8"], ca["s_q"], None, epilogue=qkv, epi=epi)
                else:
                    ops.linear(xn[:Rl], ca["wq"], None, epilogue=qkv, epi=epi)
                ops.attention(q[:ql], kc[:ql], vc[:ql], ao[:Rl], live * b, heads, ctx["m"] + 1, key_mask=ctx["key_mask"][:live * b],
                              logit_bound=ca["bound"])
                ops.linear(ao[:Rl], ca["wo"], x[:Rl], epilogue=ops.EPI_RESIDUAL, resid=x[:Rl])
            # --- feed forward: one LayerNorm over every branch, which first adds to_out(null_v) to the rows of the masked branches ---
            null_add = dict(add=ca["null_out"], x_out=x, add_from=Rl) if live < nb else {}
            norm(slice(None), ff["g0"], "w1_8" in ff, **null_add)
            self._ff_tail(xn, ff, x, ws, R)
        return x

    def _ff_tail(self, xn, ff, x, ws, R):
        h, hn = ws["h"][:R, :ff["Fp"]], ws["hn"][:R, :ff["Fp"]]
        if ff["Fp"] != ws["h"].shape[1]:
            h, hn = h.contiguous(), hn.contiguous()
        if "w2f" in ff:      # bf16: inner LayerNorm folded into the two GEMM epilogues (no pass over h between them)
            stats = ws["stats"][:R, :ff["Fp"] // 32]     # per-chunk (sum, sumsq) partials written by FF1's epilogue, added in order by FF2's
            if stats.shape[1] != ws["stats"].shape[1]:
                stats = stats.contiguous()
            if "w1_8" in ff:     # fp8: the quantising LayerNorm left e4m3 rows [0, R) and their scales in the workspace
                ops.linear_fp8(ws["xq"][:R], ws["xs"][:R], ff["w1_8"], ff["s1"], h, epilogue=ops.EPI_GEGLU, row_stats=stats)
            else:
                ops.linear(xn[:R], ff["w1"], h, epilogue=ops.EPI_GEGLU, row_stats=stats)
            ops.linear(h, ff["w2f"], x[:R], epilogue=ops.EPI_LNFOLD_RESIDUAL, bias=ff["cvec"], resid=x[:R], row_stats=stats, ln_width=ff["F"])
            return
        ops.linear(xn[:R], ff["w1"], h, epilogue=ops.EPI_GEGLU)
        ops.layernorm(h, ff["g3"], hn, width=ff["F"])
        ops.linear(hn, ff["w2"], x[:R], epilogue=ops.EPI_RESIDUAL, resid=x[:R])

    def _ff(self, inp, ff, x_acc, ws, R):
        """x_acc += FeedForward(inp)   (self-conditioning embed, muse_maskgit_pytorch.py:325-328)"""
        xn = ws["xn"][:R]
        if "w1_8" in ff:
            ops.layernorm_fp8(inp, ff["g0"], ws["xq"][:R], ws["xs"][:R])
        else:
            ops.layernorm(inp, ff["g0"], xn)
        self._ff_tail(xn, ff, x_acc, ws, R)

    # ----- public API ---------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x, return_embed=False, return_logits=False, labels=None, ignore_index=0, self_cond_embed=None,
                cond_drop_prob=0., conditioning_token_ids: Optional[torch.Tensor] = None, texts: Optional[List[str]] = None,
                text_embeds: Optional[torch.Tensor] = None):
        """ref: muse_maskgit_pytorch.py:279-348.  cond_drop_prob in {0, 1} is deterministic; other values draw one
        Bernoulli per batch row like prob_mask_like."""
        ids = x
        b, n = ids.shape
        assert (texts is not None) ^ (text_embeds is not None)
        if texts is not None:
            text_embeds = self.encode_text(texts)
        text_embeds = text_embeds.to(ids.device)
        if 0. < cond_drop_prob < 1.:
            keep = torch.zeros((b, 1, 1), device=ids.device).uniform_(0, 1) < (1. - cond_drop_prob)
            text_embeds = text_embeds * keep           # zero rows == masked keys (muse_maskgit_pytorch.py:304)
        ctx = self._prepare_context(text_embeds, conditioning_token_ids, [cond_drop_prob == 1])
        xres = self._run_blocks(ids, ctx, 1, self_cond_embed)
        P = self._packed()
        embed = torch.empty((b * n, self.dim), device=ids.device, dtype=torch.float32)
        ops.layernorm(xres, P["gf"], embed)
        logits = torch.empty((b * n, self.dim_out), device=ids.device, dtype=torch.float32)
        ops.linear(embed.to(P["adt"]) if P["adt"] != torch.float32 else embed, P["wlog"], logits)
        logits, embed = logits.view(b, n, -1), embed.view(b, n, -1)
        if return_embed:
            return logits, embed
        if labels is None:
            return logits
        F = torch.nn.functional
        if self.dim_out == 1:
            loss = F.binary_cross_entropy_with_logits(logits[..., 0], labels)
        else:
            loss = F.cross_entropy(logits.transpose(1, 2), labels, ignore_index=ignore_index)
        return (loss, logits) if return_logits else loss

    @torch.no_grad()
    def forward_with_cond_scale(self, *args, cond_scale=3., return_embed=False, **kwargs):
        """ref: muse_maskgit_pytorch.py:240-259."""
        if cond_scale == 1:
            return self.forward(*args, return_embed=return_embed, cond_drop_prob=0., **kwargs)
        logits, embed = self.forward(*args, return_embed=True, cond_drop_prob=0., **kwargs)
        null_logits = self.forward(*args, cond_drop_prob=1., **kwargs)
        scaled = null_logits + (logits - null_logits) * cond_scale
        return (scaled, embed) if return_embed else scaled

    def forward_with_neg_prompt(self, text_embed, neg_text_embed, cond_scale=3., return_embed=False, **kwargs):
        raise NotImplementedError("negative prompting is broken in the reference (muse_maskgit_pytorch.py:261-277 references "
                                  "undefined names); not part of the accelerated path")


class MaskGitTransformer(Transformer):
    def __init__(self, *args, **kwargs):
        assert "add_mask_id" not in kwargs
        super().__init__(*args, add_mask_id=True, **kwargs)


class TokenCritic(Transformer):
    def __init__(self, *args, **kwargs):
        assert "dim_out" not in kwargs
        super().__init__(*args, dim_out=1, **kwargs)


class SelfCritic(nn.Module):
    """ref: muse_maskgit_pytorch.py:352-375 — the generator itself as critic: to_pred(embed of the conditional forward)."""
    def __init__(self, net):
        super().__init__()
        self.net = net
        self.to_pred = nn.Linear(net.dim, 1)
        self._head_cache = None
        self.register_load_state_dict_post_hook(lambda m, _inc: setattr(m, "_head_cache", None))

    def _apply(self, fn, *a, **k):
        self._head_cache = None
        return super()._apply(fn, *a, **k)

    def _head(self):
        sig = (self.to_pred.weight._version, self.to_pred.bias._version, self.to_pred.weight.data_ptr())
        if self._head_cache is None or self._head_cache[2] != sig:      # one host read of the bias per weight load, not per generate()
            self._head_cache = (self.to_pred.weight.detach().float().reshape(-1).contiguous(), float(self.to_pred.bias.detach().float().item()), sig)
        return self._head_cache[:2]

    @torch.no_grad()
    def forward_with_cond_scale(self, x, *args, **kwargs):
        _, embeds = self.net.forward_with_cond_scale(x, *args, return_embed=True, **kwargs)
        return embeds @ self.to_pred.weight.float().t() + self.to_pred.bias.float()

    @torch.no_grad()
    def forward(self, x, *args, labels=None, **kwargs):
        _, embeds = self.net(x, *args, return_embed=True, **kwargs)
        logits = embeds @ self.to_pred.weight.float().t() + self.to_pred.bias.float()
        if labels is None:
            return logits
        return torch.nn.functional.binary_cross_entropy_with_logits(logits[..., 0], labels)

    def forward_with_neg_prompt(self, x, *args, **kwargs):
        return self.net.forward_with_neg_prompt(x, *args, **kwargs)


def cosine_schedule(t):
    return torch.cos(t * math.pi * 0.5)


def _aten_uniform_geometry(device, numel):
    """(stride, Philox offset increment) of one ATen CUDA `uniform_` call over `numel` values.  Launch geometry as ATen's
    calc_execution_policy: block 256, grid = min(SMs * maxThreadsPerSM / 256, ceil(numel / 256)), 4 values per thread and round."""
    props = torch.cuda.get_device_properties(device)
    cap = props.multi_processor_count * (props.max_threads_per_multi_processor // 256)
    stride = 256 * min(cap, (numel + 255) // 256)
    return stride, ((numel - 1) // (stride * 4) + 1) * 4


def _cuda_generator(device):
    return torch.cuda.default_generators[device.index if device.index is not None else torch.cuda.current_device()]


def _reserve_aten_offsets(device, increment):
    """Takes `increment` Philox offsets of torch's CUDA generator on `device` for uniforms our kernels draw in place of ATen uniform_
    calls: returns (seed, first offset) and advances the generator past them, as those calls would have."""
    gen = _cuda_generator(device)
    seed, off = gen.initial_seed(), gen.get_offset()
    gen.set_offset(off + increment)
    return seed, off


def _mask_subset_prob(mask, prob, draw, min_mask=0):
    """ref: muse_maskgit_pytorch.py:46-60 (get_mask_subset_prob) with its torch.rand drawn through `draw`."""
    num_to_mask = (mask.sum(dim=-1, keepdim=True) * prob).clamp(min=min_mask)
    logits = draw(mask.shape).masked_fill(~mask, -1)
    randperm = logits.argsort(dim=-1).argsort(dim=-1).float()
    randperm -= (~mask).sum(dim=-1, keepdim=True)
    return (randperm < num_to_mask).masked_fill_(~mask, False)


def regen_tokens(mask, b, image_size, fmap_size):
    """Inpainting mask -> (b, fmap_size, fmap_size) bool, True = regenerate the token.  `mask` is bool or {0, 1}, True = regenerate, at pixel
    resolution ((b, H, W) or (b, 1, H, W), H = W = image_size) or at token resolution ((b, fmap_size, fmap_size)).  A token is regenerated when
    any pixel of its patch is masked."""
    if not isinstance(mask, torch.Tensor):
        raise TypeError(f"mask must be a torch.Tensor, got {type(mask).__name__}")
    if mask.dtype != torch.bool:
        if mask.is_complex() or not ((mask == 0) | (mask == 1)).all():
            raise ValueError("mask must be bool or hold only the values 0 and 1")
        mask = mask != 0
    if mask.dim() == 4:
        if mask.shape[1] != 1:
            raise ValueError(f"a 4-d mask must be (b, 1, H, W), got {tuple(mask.shape)}")
        mask = mask[:, 0]
    f = fmap_size
    if mask.dim() != 3 or mask.shape[0] != b or mask.shape[1:] not in ((image_size, image_size), (f, f)):
        raise ValueError(f"mask must be (b, H, W), (b, 1, H, W) with H = W = image_size = {image_size}, or (b, f, f) with f = fmap_size = {f}, "
                         f"for b = {b}; got {tuple(mask.shape)}")
    if mask.shape[1] == f:
        return mask
    p = image_size // f
    if p * f != image_size:
        raise ValueError(f"image_size {image_size} is not a multiple of fmap_size {f}: pass the mask at token resolution")
    return mask.reshape(b, f, p, f, p).any(dim=4).any(dim=2)


@dataclasses.dataclass(frozen=True)
class _Region:
    """The tokens inpaint() regenerates or edit() resamples.  n_max: the most an image regenerates per round (its schedule gives the rows
    sampled per step); iterations: None for inpaint(), else edit()'s rounds, each opened by an mmg_edit_select that writes its frozen map;
    tensors: images, counts int32 [timesteps, b], and frozen uint8 [b, n] or keep uint8 [b, n] (1 = not editable) + num_select int32 [b]."""
    n_max: int
    iterations: Optional[int]
    tensors: dict


def _per_image(name, value, b):
    """A sampling setting of generate() / inpaint() / edit() as a tuple of b Python floats: `value` is a number (every image), or a
    length-b sequence of numbers or 1-D tensor (image by image).  Raises ValueError on a wrong length or a value that is not finite."""
    if isinstance(value, torch.Tensor):
        if value.dim() > 1:
            raise ValueError(f"{name} must be a number or 1-D, got a tensor of shape {tuple(value.shape)}")
        value = value.item() if value.dim() == 0 else value.detach().cpu().double().tolist()
    if isinstance(value, numbers.Real):
        vals = (float(value),) * b
    else:
        try:
            vals = tuple(float(v) for v in value)
        except (TypeError, ValueError):
            raise ValueError(f"{name} must be a number, a sequence of numbers or a 1-D tensor, got {value!r}") from None
        if len(vals) != b:
            raise ValueError(f"{name} has {len(vals)} values for {b} texts")
    if not all(math.isfinite(v) for v in vals):
        raise ValueError(f"{name} must be finite, got {vals}")
    return vals


def _fill_on_device(t, device):
    """Host tensor `t` rebuilt on `device` with one fill kernel per run of equal values.  Used when a caller captures the whole call into
    their own CUDA graph, where a host-to-device copy cannot be recorded; the values are then fixed in that graph, as scalar arguments are."""
    flat = t.reshape(-1).tolist()
    out = torch.empty((len(flat),), dtype=t.dtype, device=device)
    start = 0
    for i in range(1, len(flat) + 1):
        if i == len(flat) or flat[i] != flat[start]:
            out[start:i].fill_(flat[start])
            start = i
    return out.view(t.shape)


@dataclasses.dataclass(frozen=True)
class _DecodeRequest:
    """One validated generate() / inpaint() / edit() call.  temperature, cond_scale, critic_noise_scale: one float per image.
    seed: the libmmg sampling seed (None: sampler_seed or a draw when it runs)."""
    texts: List[str]
    cond_images: Optional[torch.Tensor]
    fmap_size: int
    temperature: tuple
    topk_filter_thres: float
    timesteps: int
    cond_scale: tuple
    critic_noise_scale: tuple
    can_remask_prev_masked: bool
    use_critic: bool
    return_ids: bool
    region: Optional[_Region] = None
    seed: Optional[int] = None

    @property
    def branches(self):
        """CFG branches of the call: 1 when every image's cond_scale is 1 (no null forward, as the reference), else 2."""
        return 1 if all(c == 1 for c in self.cond_scale) else 2

    def settings(self, n):
        """The host fp32 tables the sampling kernels read, each value the float64 expression of a scalar call rounded once: temps and
        crit_noise [timesteps, b] (step s anneals by steps_until_x0 / timesteps, muse_maskgit_pytorch.py:578, 600), cond_scale [b]; with a
        critic, its per-row copies over the n positions of each image (crit_cond_scale [b*n], crit_noise [timesteps, b*n])."""
        anneal = [until / self.timesteps for until in reversed(range(self.timesteps))]
        f32 = lambda v: torch.tensor(v, dtype=torch.float32)
        out = dict(temps=f32([[t * a for t in self.temperature] for a in anneal]), cond_scale=f32(self.cond_scale))
        if self.use_critic:
            out["crit_cond_scale"] = out["cond_scale"].repeat_interleave(n)
            out["crit_noise"] = f32([[c * a for c in self.critic_noise_scale] for a in anneal]).repeat_interleave(n, dim=1)
        return out


class _CapturedCall(NamedTuple):
    """A whole-call CUDA graph of MaskGit._generate_body and the static tensors it reads and writes."""
    graph: "torch.cuda.CUDAGraph"
    inputs: tuple               # (text_embeds, cond_images or None, region tensors or None, settings tables), copied in before each replay
    outputs: tuple              # (images, ids, fused-tail status or None)
    pack_ids: tuple             # identities of the packed weights at capture: a re-pack re-captures
    keep_alive: tuple           # packed weights and workspaces the captured kernels point at


# ------------------------------------------------------------------------------------------------ MaskGit
class MaskGit(nn.Module):
    def __init__(self, image_size, transformer: MaskGitTransformer, noise_schedule: Callable = cosine_schedule,
                 token_critic: Optional[TokenCritic] = None, self_token_critic=False, vae: Optional[VQGanVAE] = None,
                 cond_vae: Optional[VQGanVAE] = None, cond_image_size=None, cond_drop_prob=0.5, self_cond_prob=0.9,
                 no_mask_token_prob=0., critic_loss_weight=1.):
        super().__init__()
        assert isinstance(transformer, MaskGitTransformer), "transformer must be a MaskGitTransformer"
        assert vae is None or isinstance(vae, VQGanVAE)
        assert vae is not None, "a VQGanVAE is required (the reference dereferences it unconditionally, muse_maskgit_pytorch.py:462)"
        self.vae = vae.copy_for_eval()
        self.cond_vae = cond_vae.eval() if cond_vae is not None else self.vae
        assert not (cond_vae is not None and cond_image_size is None), "cond_image_size must be specified if conditioning"
        self.image_size, self.cond_image_size = image_size, cond_image_size
        self.resize_image_for_cond_image = cond_image_size is not None
        self.cond_drop_prob = cond_drop_prob
        self.transformer = transformer
        self.self_cond = transformer.self_cond
        assert self.vae.codebook_size == self.cond_vae.codebook_size == transformer.num_tokens, \
            "transformer num_tokens must be set to be equal to the vae codebook size"
        self.mask_id = transformer.mask_id
        self.noise_schedule = noise_schedule
        assert not (self_token_critic and token_critic is not None)
        self.token_critic = token_critic
        if self_token_critic:
            self.token_critic = SelfCritic(transformer)
        self.critic_loss_weight, self.self_cond_prob, self.no_mask_token_prob = critic_loss_weight, self_cond_prob, no_mask_token_prob
        # sampler noise: None -> in-kernel Philox keyed on (seed, global row, vocab index); or a callable
        # noise_fn(step, shape) -> U[0,1) tensor (parity mode: the tensors the reference would draw, in its order:
        # shape (b, n, V) for the gumbel noise, then shape (b, n) for the token-critic noise when a critic scores the step)
        self.sampler_seed = None            # None: one draw from torch's global generator per call (reproducible under manual_seed)
        self.sampler_noise_fn = None
        # "mmg": libmmg's Philox keying (invariant to the GPU count).  "aten": the exact stream the reference's
        # `zeros_like(t).uniform_(0, 1)` / `uniform(scores.shape)` calls draw from torch's CUDA generator on this device, consumed
        # from (and advanced on) torch.cuda's default generator, with the reference's accurate log / division arithmetic
        self.sampler_rng = "mmg"
        self.global_batch = None            # "aten" + batch sharding: size of the whole batch the reference would have drawn noise for
        self.use_cuda_graph = True
        self.use_native_step = False        # True: one mmg_decode_step call per step (the same launch sequence issued from C++)
        self.check_fused_tail = True        # read the fused path's overflow word after every call (4 bytes, one host sync)
        self.last_fused_fallback_rows = 0   # rows of the last generate() that were redone through materialised logits (diagnostic)
        self.use_fused_tail = True          # bf16: to_logits + sampling tail without materialised logits (mmg_logits_fused); False: mmg_linear + mmg_logits_sample
        self._graphs = {}
        self.row_offset = 0                 # global index of this shard's first sequence (multi-GPU batch sharding)
        self.register_load_state_dict_post_hook(lambda m, _inc: m._graphs.clear())

    def _apply(self, fn, *a, **k):
        self.__dict__.get("_graphs", {}).clear()
        return super()._apply(fn, *a, **k)

    def save(self, path):
        torch.save(self.state_dict(), path)

    def load(self, path):
        path = Path(path)
        assert path.exists()
        self.load_state_dict(torch.load(str(path)))

    def mask_schedule(self, seq_len, timesteps):
        """Data-independent, so evaluated on the host once (the reference syncs with .item() every step,
        muse_maskgit_pytorch.py:558-559); same fp32 arithmetic."""
        return [max(int((self.noise_schedule(t) * seq_len).item()), 1) for t in torch.linspace(0, 1, timesteps)]

    @torch.no_grad()
    def generate(self, texts: List[str], negative_texts: Optional[List[str]] = None, cond_images: Optional[torch.Tensor] = None,
                 fmap_size=None, temperature=1., topk_filter_thres=0.9, can_remask_prev_masked=False,
                 force_not_use_token_critic=False, timesteps=18, cond_scale=3, critic_noise_scale=1, return_ids=False):
        """ref: muse_maskgit_pytorch.py:491-621.  Returns fp32 NCHW images (b, 3, H, W), unclamped.

        temperature, cond_scale and critic_noise_scale are each a number (every image) or per image, a length-b sequence of numbers or a
        1-D tensor on any device: image i is decoded as if the whole call had been made with its own values (values must be finite,
        temperature >= 0).  The settings reach the kernels as device data, so one captured CUDA graph replays for any of them; only
        whether every image has cond_scale == 1 (no null-CFG forward) selects a different graph.  inpaint() and edit() take them alike."""
        if self.use_native_step and self.transformer.precision == "fp8":
            raise ValueError('use_native_step=True runs mmg_decode_step, whose weights carry no fp8 scales: it cannot run precision="fp8"; '
                             "set use_native_step = False")
        if self.use_native_step and self.transformer.transformer_blocks.dim_head != 64:
            raise ValueError("use_native_step=True runs mmg_decode_step, which is written for 64-wide heads: it cannot run dim_head="
                             f"{self.transformer.transformer_blocks.dim_head}; set use_native_step = False")
        if negative_texts is not None:
            raise NotImplementedError("negative_texts raises TypeError in the reference (defect B2); not supported")
        return self._decode(self._request(texts, cond_images=cond_images, fmap_size=fmap_size, temperature=temperature, timesteps=timesteps,
                                          topk_filter_thres=topk_filter_thres, can_remask_prev_masked=can_remask_prev_masked, cond_scale=cond_scale,
                                          force_not_use_token_critic=force_not_use_token_critic, critic_noise_scale=critic_noise_scale, return_ids=return_ids))

    @torch.no_grad()
    def inpaint(self, texts: List[str], images: torch.Tensor, mask: torch.Tensor, cond_images: Optional[torch.Tensor] = None, temperature=1.,
                topk_filter_thres=0.9, can_remask_prev_masked=False, force_not_use_token_critic=False, timesteps=18, cond_scale=3,
                critic_noise_scale=1, return_ids=False):
        """Regenerates the masked region of `images` and keeps the rest (an extension: the reference has no inpainting).

        images: fp32 NCHW (b, C, image_size, image_size), as `vae.encode` takes them.  mask: bool or {0, 1}, True = regenerate, either
        (b, H, W) / (b, 1, H, W) at pixel resolution or (b, f, f) at token resolution (f = fmap_size); a token is regenerated when any pixel
        of its patch is masked.  Outpainting is the same call on a canvas whose border is masked.

        The tokens start as vae.encode_ids(images) with mask_id at the regenerated positions, which decode as in generate() except that
        each image re-masks only among its own regenerated tokens, on its own schedule max(int(noise_schedule(t) * N_b), 1) (N_b = its
        number of regenerated tokens, 0 when it has none).  Every other token id equals the encoded one bit for bit.  The pixels are
        vae.decode_from_ids(ids): the unmasked region is the VAE reconstruction, not the input pixels; pasting the input back is the
        caller's job.  With every token masked the result equals generate() under the same seed or injected noise.
        Returns what generate() returns.  `use_native_step` does not apply here (mmg_decode_step has no frozen positions)."""
        b = len(texts)
        fmap_size = self.vae.get_encoded_fmap_size(self.image_size)
        self._check_images(images, b)
        regen = regen_tokens(mask, b, self.image_size, fmap_size).reshape(b, -1)
        counts = [int(c) for c in regen.sum(dim=1).tolist()]                      # N_b: the call's one device-to-host read for a GPU mask
        region = self._region(images, counts, timesteps, frozen=(~regen).to(torch.uint8))
        return self._decode(self._request(texts, cond_images=cond_images, temperature=temperature, timesteps=timesteps, region=region,
                                          topk_filter_thres=topk_filter_thres, can_remask_prev_masked=can_remask_prev_masked, cond_scale=cond_scale,
                                          force_not_use_token_critic=force_not_use_token_critic, critic_noise_scale=critic_noise_scale, return_ids=return_ids))

    @torch.no_grad()
    def edit(self, texts: List[str], images: torch.Tensor, mask: Optional[torch.Tensor] = None, iterations=8, fraction=0.1, timesteps=4,
             cond_images: Optional[torch.Tensor] = None, temperature=1., topk_filter_thres=0.9, can_remask_prev_masked=False,
             force_not_use_token_critic=False, cond_scale=3, critic_noise_scale=1, return_ids=False):
        """Mask-free editing (an extension, as inpaint() is; the Muse paper's third editing mode): moves `images` towards the prompts while
        keeping their layout, by repeatedly re-masking a random subset of their tokens and resampling it.

        images: fp32 NCHW (b, C, image_size, image_size), encoded once as ids0 = vae.encode_ids(images).  mask: the editable region in any
        form inpaint() takes (True = editable); None = the whole image.  E_b is image b's editable tokens, N_b = |E_b|, and
        r_b = max(int(fraction * N_b), 1) when N_b > 0, else 0 (host Python floats, the same in every iteration).
        Iteration i (0 <= i < iterations):
          1. image b draws one key per position and selects the r_b editable positions with the largest keys (ties: lowest position);
          2. exactly inpaint()'s token loop with the selection as the regenerated region: `timesteps` decode steps, image b on the schedule
             max(int(noise_schedule(t) * r_b), 1), the temperature annealed over the iteration's steps, scores and the self-conditioning
             embedding reset at the start of the iteration.  Decode step s has the global step index i * timesteps + s, which keys the
             sampler's Philox stream and is the step passed to `sampler_noise_fn`.
        Keys: libmmg's Philox with counter (0xFFFFFFFE, i, global position) and the call's seed (disjoint from the gumbel and critic noise,
        independent of how the batch is sharded over `row_offset`); with `sampler_noise_fn` set, sampler_noise_fn(i * timesteps, (b, n)),
        drawn before that iteration's first gumbel draw.  sampler_rng = "aten" has no reference stream for the keys and raises ValueError.
        Tokens outside the selections keep their ids bit for bit; the token grid stays on the device for the whole call (one encode, one
        decode).  iterations = 1, fraction = 1 is inpaint(mask) (generate() for mask=None) under the same seed; iterations = 0 returns
        ids0 and its decode.  The defaults (8 iterations of 4 steps on 10 % of the tokens) are this project's provisional choice, not
        settings from the paper.  Returns what generate() returns.  `use_native_step` does not apply here, as for inpaint()."""
        if isinstance(iterations, bool) or not isinstance(iterations, int) or iterations < 0:
            raise ValueError(f"iterations must be an int >= 0, got {iterations!r}")
        if not 0 < fraction <= 1:
            raise ValueError(f"fraction must lie in (0, 1], got {fraction!r}")
        if isinstance(timesteps, bool) or not isinstance(timesteps, int) or timesteps < 1:
            raise ValueError(f"timesteps must be an int >= 1, got {timesteps!r}")
        if self.sampler_rng == "aten":
            raise ValueError('edit() has no "aten" noise stream (the reference has no editing): use sampler_rng = "mmg" or sampler_noise_fn')
        b = len(texts)
        fmap_size = self.vae.get_encoded_fmap_size(self.image_size)
        self._check_images(images, b)
        editable = (torch.ones((b, fmap_size ** 2), dtype=torch.bool) if mask is None
                    else regen_tokens(mask, b, self.image_size, fmap_size).reshape(b, -1))
        counts = [int(c) for c in editable.sum(dim=1).tolist()]                   # N_b
        select = [max(int(fraction * c), 1) if c else 0 for c in counts]          # r_b
        region = self._region(images, select, timesteps, iterations, keep=(~editable).to(torch.uint8), num_select=torch.tensor(select, dtype=torch.int32))
        return self._decode(self._request(texts, cond_images=cond_images, temperature=temperature, timesteps=timesteps, region=region,
                                          topk_filter_thres=topk_filter_thres, can_remask_prev_masked=can_remask_prev_masked, cond_scale=cond_scale,
                                          force_not_use_token_critic=force_not_use_token_critic, critic_noise_scale=critic_noise_scale, return_ids=return_ids))

    def _check_images(self, images, b):
        if not isinstance(images, torch.Tensor) or tuple(images.shape) != (b, self.vae.channels, self.image_size, self.image_size):
            raise ValueError(f"images must be a (b, {self.vae.channels}, {self.image_size}, {self.image_size}) tensor for b = {b} texts, got "
                             f"{tuple(images.shape) if isinstance(images, torch.Tensor) else type(images).__name__}")

    def _region(self, images, counts, timesteps, iterations=None, **tensors):
        """The _Region of a call whose image b regenerates counts[b] tokens per round, on the schedule of that count (none: 0 throughout)."""
        table = [self.mask_schedule(c, timesteps) if c else [0] * timesteps for c in counts]
        tensors.update(images=images.to(torch.float32), counts=torch.tensor(table, dtype=torch.int32).t())        # counts: [timesteps, b]
        device = next(self.parameters()).device
        return _Region(max(counts, default=0), iterations, {k: v.to(device).contiguous() for k, v in tensors.items()})

    def _request(self, texts, *, force_not_use_token_critic, fmap_size=None, **settings):
        use_critic = self.token_critic is not None and not force_not_use_token_critic
        if settings["can_remask_prev_masked"] and not use_critic:      # the reference only reaches this assert in the no-critic branch (:611-612)
            assert self.no_mask_token_prob > 0., "without training with some of the non-masked tokens forced to predict, not sure if the logits will be meaningful for these token"
        fmap_size = fmap_size if fmap_size is not None else self.vae.get_encoded_fmap_size(self.image_size)
        for name in ("temperature", "cond_scale", "critic_noise_scale"):
            settings[name] = _per_image(name, settings[name], len(texts))
        if any(t < 0 for t in settings["temperature"]):
            raise ValueError(f"temperature must be >= 0, got {settings['temperature']}")
        return _DecodeRequest(texts=texts, fmap_size=fmap_size, use_critic=use_critic, **settings)

    def _check_weights(self):          # in-place parameter edits since the last call drop the packed copies (and the captured graphs)
        for net in (self.transformer, self.vae, self.cond_vae, self.token_critic if isinstance(self.token_critic, Transformer) else None):
            if net is not None:
                net._check_weights()

    def _injected_noise(self, step, shape, device):
        """sampler_noise_fn's U[0, 1) tensor for (step, shape) as contiguous fp32 on `device`; None when no noise is injected."""
        if self.sampler_noise_fn is None:
            return None
        return self.sampler_noise_fn(step, shape).to(device=device, dtype=torch.float32).contiguous()

    def _resolve_critic(self, text_embeds, cond_ids, branches, ctx=None):
        """(net, CFG branches, context, head weight, head bias, final LayerNorm gamma) of the token critic.  A SelfCritic is the generator's
        conditional branch (muse_maskgit_pytorch.py:352-361), over `ctx` when given; a TokenCritic runs `branches` over its own context."""
        if isinstance(self.token_critic, SelfCritic):
            net, nb = self.transformer, 1
            whead, bhead = self.token_critic._head()
            whead = whead.to(text_embeds.device)
            ctx = ctx if ctx is not None else net._prepare_context(text_embeds, cond_ids, branches)
        else:
            net, nb = self.token_critic, len(branches)
            ctx = net._prepare_context(text_embeds, cond_ids, branches)
            whead, bhead = net._packed()["whead"], 0.
            assert whead is not None, "token_critic must have dim_out == 1"
        return net, nb, ctx, whead, bhead, net._packed()["gf"]

    def _decode(self, req):
        """Runs a generate() / inpaint() / edit() request in eval mode.  A call whose fused tail overflowed is repeated on the materialised
        path with the same noise: the same libmmg seed, or the ATen generator position the failed attempt started from."""
        was_training, saved = self.training, self.use_fused_tail
        self.eval()
        try:
            images, ids, status, seed = self._decode_once(req)
            if not self._fused_tail_overflowed(status):
                return (images, ids) if req.return_ids else images
            self.use_fused_tail = False
            if self.sampler_rng == "aten" and self.sampler_noise_fn is None:       # re-read the generator position the failed attempt consumed
                _cuda_generator(next(self.parameters()).device).set_offset(self._aten_start_offset)
            return self._decode(dataclasses.replace(req, seed=seed))
        finally:
            self.train(was_training)
            self.use_fused_tail = saved

    def _decode_once(self, req):
        """One attempt at a request: (images, ids, the fused tail's status word or None, the libmmg seed it sampled with)."""
        tr = self.transformer
        device = next(self.parameters()).device
        b = len(req.texts)
        self._check_weights()
        text_embeds = tr.encode_text(req.texts).to(device, non_blocking=True)
        if self.use_cuda_graph and text_embeds.shape[1] % 32:
            # T5 pads to the longest prompt of the batch: bucket the length (multiples of 32) so that prompt lengths share captured
            # graphs; all-zero rows are padding to the reference too (masked keys, muse_maskgit_pytorch.py:304)
            text_embeds = torch.nn.functional.pad(text_embeds, (0, 0, 0, 32 - text_embeds.shape[1] % 32))
        if self.resize_image_for_cond_image:
            assert req.cond_images is not None, "conditioning image must be passed in to generate for super res maskgit"
            cond_images = req.cond_images.to(device, torch.float32)
        else:
            cond_images = None
        # per-call seed: explicit sampler_seed, else one draw from torch's global generator (reproducible under manual_seed)
        assert self.sampler_rng in ("mmg", "aten"), self.sampler_rng
        if getattr(self, "_seed_dev", None) is None or self._seed_dev.device != device:
            self._seed_dev = torch.zeros((1,), dtype=torch.int64, device=device)
        aten, seed = None, req.seed
        if self.sampler_rng == "aten" and self.sampler_noise_fn is None:
            aten = self._aten_plan(device, b, req.fmap_size ** 2, tr.num_tokens, req.timesteps, req.use_critic)
        elif self.sampler_noise_fn is None:      # (injected noise: the host generator is the caller's stream — nothing is drawn from it here)
            if seed is None:                     # (a rerun on the materialised path keeps the seed of the attempt it repeats)
                seed = self.sampler_seed if self.sampler_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
            self._seed_dev.fill_(seed)
        region = None if req.region is None else req.region.tensors
        # per-image sampling settings as device data: a captured graph copies them in like the region, so they are not in its key
        upload = _fill_on_device if torch.cuda.is_current_stream_capturing() else (lambda t, dev: t.to(dev))
        settings = {k: upload(v, device) for k, v in req.settings(req.fmap_size ** 2).items()}
        if not self.use_cuda_graph or self.sampler_noise_fn is not None:
            return self._generate_body(req, text_embeds, cond_images, region, settings, aten) + (seed,)
        # ---- whole-call CUDA graph: 18 decode steps + VAE decode replayed as one launch (no per-kernel host work) ----
        key = (b, tuple(text_embeds.shape), text_embeds.dtype, None if cond_images is None else tuple(cond_images.shape), req.fmap_size,
               float(req.topk_filter_thres), int(req.timesteps), req.branches, int(self.row_offset),
               tr.precision, self.vae.precision, req.use_critic, bool(req.can_remask_prev_masked),
               None if aten is None else aten["key"], bool(self.use_native_step), id(self.noise_schedule), bool(self.use_fused_tail))
        if req.region is not None:
            key += (("inpaint", req.region.n_max) if req.region.iterations is None else ("edit", req.region.iterations, req.region.n_max),)
        critic_net = self.token_critic if isinstance(self.token_critic, Transformer) and req.use_critic else None
        pack_ids = lambda: (id(tr._pack), id(self.vae._pack), id(self.cond_vae._pack), id(critic_net._pack) if critic_net is not None else 0,
                            id(self.token_critic._head_cache) if isinstance(self.token_critic, SelfCritic) else 0)
        entry = self._graphs.get(key)
        if entry is not None and entry.pack_ids != pack_ids():
            entry = None                                       # weights were re-packed (load_state_dict / .to()): re-capture
        if entry is None:
            te_s = text_embeds.clone()
            ci_s = None if cond_images is None else cond_images.clone()
            region_s = None if region is None else {k: v.clone() for k, v in region.items()}
            settings_s = {k: v.clone() for k, v in settings.items()}
            self._generate_body(req, te_s, ci_s, region_s, settings_s, aten)        # eager warm-up: lazy packing, workspaces, function attributes
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                outputs = self._generate_body(req, te_s, ci_s, region_s, settings_s, aten)
            entry = _CapturedCall(graph, (te_s, ci_s, region_s, settings_s), outputs, pack_ids(),
                                  keep_alive=(tr._pack, self.vae._pack, self.cond_vae._pack, dict(getattr(tr, "_ws", {})),
                                              None if critic_net is None else (critic_net._pack, dict(getattr(critic_net, "_ws", {}))),
                                              self.token_critic._head_cache if isinstance(self.token_critic, SelfCritic) else None))
            if len(self._graphs) >= 4:
                self._graphs.pop(next(iter(self._graphs)))       # least recently used (hits are moved to the end below)
        self._graphs.pop(key, None)
        self._graphs[key] = entry
        te_s, ci_s, region_s, settings_s = entry.inputs
        te_s.copy_(text_embeds, non_blocking=True)
        if ci_s is not None:
            ci_s.copy_(cond_images, non_blocking=True)
        for k, v in (region_s or {}).items():
            v.copy_(region[k], non_blocking=True)
        for k, v in settings_s.items():
            v.copy_(settings[k], non_blocking=True)
        entry.graph.replay()
        images, ids, status = entry.outputs
        return images.clone(), ids.clone(), status, seed

    def _fused_tail_overflowed(self, status):
        """status[1] != 0: some decode step had more rows whose sampled top-k threshold missed than the fused path's fallback holds (e.g. constant
        logits rows).  One 4-byte read per call; `check_fused_tail = False` skips it (and the host synchronisation it implies)."""
        if status is None or not self.check_fused_tail:
            return False
        self.last_fused_fallback_rows, overflow = (int(v) for v in status.tolist())
        return overflow != 0

    def _native_step_setup(self, ctx, P, b, n, nb, max_masked, V, device):
        """Argument block of mmg_decode_step for this generate(): the packed weights and the per-call context as raw pointers, plus the
        zero-initialised workspace.  Everything referenced is kept alive by the returned dict (and by `P` / `ctx`)."""
        tr = self.transformer
        tb = tr.transformer_blocks
        depth = len(P["layers"])
        layers = (_lib.LayerWeights * depth)()
        for li, lay in enumerate(P["layers"]):
            sa, ca, ff, lw = lay["sa"], lay["ca"], lay["ff"], layers[li]
            lw.self_attn.ln_gamma = sa["g"].data_ptr(); lw.self_attn.w_qkv = sa["wqkv"].data_ptr(); lw.self_attn.w_out = sa["wo"].data_ptr()
            lw.self_attn.q_scale = sa["qs"].data_ptr(); lw.self_attn.k_scale = sa["ks"].data_ptr()
            lw.self_attn.null_k = sa["nk"].data_ptr(); lw.self_attn.null_v = sa["nv"].data_ptr(); lw.self_attn.logit_bound = sa["bound"]
            lw.cross_attn.ln_gamma = ca["g"].data_ptr(); lw.cross_attn.w_qkv = ca["wq"].data_ptr(); lw.cross_attn.w_out = ca["wo"].data_ptr()
            lw.cross_attn.q_scale = ca["qs"].data_ptr(); lw.cross_attn.logit_bound = ca["bound"]
            kc, vc = ctx["kv"][li]
            lw.ctx_k = kc.data_ptr(); lw.ctx_v = vc.data_ptr(); lw.cross_null_out = ca["null_out"].data_ptr()
            lw.ff_ln_gamma = ff["g0"].data_ptr(); lw.ff_w1 = ff["w1"].data_ptr(); lw.ff_w2f = ff["w2f"].data_ptr(); lw.ff_cvec = ff["cvec"].data_ptr()
        ff0 = P["layers"][0]["ff"]
        assert all(l["ff"]["Fp"] == ff0["Fp"] and l["ff"]["F"] == ff0["F"] for l in P["layers"])
        nbytes = int(_lib.lib().mmg_decode_step_workspace_bytes(b, nb, n, tr.dim, tb.heads, ff0["Fp"], V, max_masked))
        ws = torch.zeros((nbytes,), dtype=torch.uint8, device=device)
        a = _lib.DecodeStepArgs()
        a.depth = depth; a.dim = tr.dim; a.heads = tb.heads; a.n = n; a.V = V; a.F = ff0["F"]; a.Fp = ff0["Fp"]; a.b = b
        a.branches = nb; a.live_branches = min(ctx["live"], nb)
        a.layers = ctypes.cast(layers, ctypes.POINTER(_lib.LayerWeights))
        a.tok_emb = P["tok"].data_ptr(); a.pos_emb = P["pos"].data_ptr(); a.final_gamma = P["gf"].data_ptr(); a.w_logits = P["wlog"].data_ptr()
        a.ctx_key_mask = ctx["key_mask"].data_ptr(); a.ctx_keys = ctx["m"]; a.ctx_alloc = ctx["kv"][0][0].shape[1]
        a.mask_id = self.mask_id
        a.workspace = ws.data_ptr(); a.workspace_bytes = nbytes
        return dict(args=a, layers=layers, ws=ws, ctx=ctx, P=P)

    def _aten_plan(self, device, b, n, V, timesteps, use_critic):
        """Offsets of the reference's uniform_ calls in torch's CUDA Philox stream (one (b, n, V) gumbel draw, then one (b, n) critic
        draw per step, muse_maskgit_pytorch.py:407, 598) in ATen's launch geometry.  The generator is read here and advanced by what the
        reference would have consumed; seed / offset reach the kernels through device words (graph replay)."""
        B = self.global_batch if self.global_batch is not None else b
        (stride_g, inc_g), (stride_c, inc_c) = _aten_uniform_geometry(device, B * n * V), _aten_uniform_geometry(device, B * n)
        per_step = inc_g + (inc_c if use_critic else 0)
        seed, off = _reserve_aten_offsets(device, timesteps * per_step)
        self._aten_start_offset = off
        if getattr(self, "_aten_dev", None) is None or self._aten_dev.device != device:
            self._aten_dev = torch.zeros((2,), dtype=torch.int64, device=device)
        wrap = lambda v: v - (1 << 64) if v >= (1 << 63) else v
        self._aten_dev.copy_(torch.tensor([wrap(seed), off], dtype=torch.int64), non_blocking=False)
        return dict(key=(B, stride_g, stride_c, per_step), stride_g=stride_g, stride_c=stride_c, inc_g=inc_g, per_step=per_step)

    def _tail_buffers(self, b, n, rows_max, V, device, k_keep=None):
        """Scratch of the per-step sampling tail for at most `rows_max` sampled rows per sequence.  bf16 + a supported shape: the workspace of
        the fused logits / sampling path (candidate lists, no [rows, V] logits); otherwise the materialised fp32 logits."""
        tr = self.transformer
        adt = tr._packed()["adt"]
        bufs = dict(e=torch.empty((b * n, tr.dim), device=device, dtype=adt), rows_max=rows_max)
        nbytes = 0
        if self.use_fused_tail and adt == torch.bfloat16 and k_keep is not None:
            nbytes = ops.logits_fused_workspace_bytes(b * rows_max, V, tr.dim, k_keep)
        if nbytes:
            bufs["fused_ws"] = torch.empty((nbytes,), dtype=torch.uint8, device=device)
            bufs["status"] = torch.zeros((2,), dtype=torch.int32, device=device)
        else:
            bufs["logits"] = torch.empty((b * rows_max, V), device=device, dtype=torch.float32)
        return bufs

    def _sample_tail(self, x, nb, pos, rows_b, ids, scores, temp, step, u, cond_scale, k_keep, tail, seed_dev=None, only_masked_id=None, aten=None,
                     temp_dev=None, cond_scale_dev=None):
        """The sampling tail of one decode step (muse_maskgit_pytorch.py:576-609) on the rows listed in `pos` (b, rows_b): final LayerNorm +
        CFG combine in embedding space, to_logits, top-k filter, gumbel argmax, confidence score; ids / scores are updated in place.
        x: residual stream [nb*b*n, dim] after the blocks (cond rows first, then the null-CFG rows).  temp_dev / cond_scale_dev: fp32 [b]
        per-image values the kernels read in place of the scalars `temp` / `cond_scale`."""
        tr = self.transformer
        P = tr._packed()
        b, n = ids.shape
        bn = b * n
        R = b * rows_b
        e = tail["e"]
        ops.final_embed(x[:bn], x[bn:2 * bn] if nb == 2 else None, P["gf"], pos, e, b, n, rows_b, cond_scale, cond_scale_dev=cond_scale_dev)
        kw = dict(u=u, seed=0, seed_dev=seed_dev, step=step, row_offset=self.row_offset * n, only_masked_id=only_masked_id, aten=aten,
                  temperature_dev=temp_dev)
        if "fused_ws" in tail:      # logits never reach HBM: candidate lists out of the GEMM epilogue, sampled by the finishing kernel
            ops.logits_fused(e[:R], P["wlog"], pos, ids, scores, rows_b, k_keep, temp, tail["fused_ws"], tail["status"],
                             rows_capacity=b * tail["rows_max"], **kw)
            return
        lg = tail["logits"][:R]
        ops.linear(e[:R], P["wlog"], lg)
        ops.logits_sample(lg, pos, ids, scores, rows_b, k_keep, temp, **kw)

    def _generate_body(self, req, text_embeds, cond_images, region, settings, aten):
        """The device-side work of a request: no host synchronisation, no data-dependent host control flow.  region, settings: the device
        tensors of req.region and req.settings() (or a captured graph's static copies of them)."""
        tr = self.transformer
        device = text_embeds.device
        b, n, V, timesteps = len(req.texts), req.fmap_size ** 2, tr.num_tokens, req.timesteps
        cond_ids = self.cond_vae.encode_ids(cond_images) if cond_images is not None else None
        nb = req.branches
        # the kernels read the settings from the device tables; the scalar argument fields carry image 0's values, which are what a call
        # with one setting for every image passes (so its launch records are those of a scalar call)
        lead = lambda v: v[0] if v else 0.
        ctx = tr._prepare_context(text_embeds, cond_ids, [False, True][:nb])
        P = tr._packed()
        adt = P["adt"]
        edit = req.region is not None and req.region.iterations is not None
        if req.region is None:
            ids = torch.full((b, n), self.mask_id, dtype=torch.long, device=device)
        elif edit:
            ids = self.vae.encode_ids(region["images"]).reshape(b, n)
            frozen = torch.empty((b, n), dtype=torch.uint8, device=device)          # written by each round's mmg_edit_select
        else:
            frozen = region["frozen"]
            ids = self.vae.encode_ids(region["images"]).reshape(b, n).masked_fill(frozen == 0, self.mask_id)
        scores = torch.zeros((b, n), dtype=torch.float32, device=device)
        masked_pos = torch.empty((b, n), dtype=torch.int32, device=device)
        k_keep = math.ceil((1 - req.topk_filter_thres) * V)                    # muse_maskgit_pytorch.py:414
        sched = self.mask_schedule(n if req.region is None else req.region.n_max, timesteps)
        score_all = bool(req.can_remask_prev_masked) and not req.use_critic
        bn = b * n
        native = None
        if (self.use_native_step and adt == torch.bfloat16 and not self.self_cond and not req.use_critic and not score_all and aten is None
                and req.region is None and all("w2f" in l["ff"] for l in P["layers"])):
            native = self._native_step_setup(ctx, P, b, n, nb, max(sched), V, device)
        rows_max = n if score_all else max(sched)
        tail = self._tail_buffers(b, n, rows_max, V, device, k_keep) if native is None else None
        all_pos = torch.arange(n, dtype=torch.int32, device=device).repeat(b, 1).contiguous() if score_all else None
        sc_embed = torch.empty((bn, tr.dim), device=device, dtype=torch.float32) if self.self_cond else None
        # token critic (muse_maskgit_pytorch.py:535-538, 590-600): a second stack over the freshly filled ids scores EVERY position
        if req.use_critic:
            cnet, cnb, cctx, whead, bhead, gcrit = self._resolve_critic(text_embeds, cond_ids, [False, True][:nb], ctx)
        seed_dev = self._seed_dev if aten is None else self._aten_dev[0:1]

        def aten_draw(step, critic=False):      # (Philox offset, device offset word, stride) of the step's gumbel or critic draw
            return None if aten is None else (step * aten["per_step"] + (aten["inc_g"] if critic else 0), self._aten_dev[1:2],
                                              aten["stride_c" if critic else "stride_g"])

        nvtx = os.environ.get("MMG_NVTX", "0") == "1"            # host-side NVTX ranges per decode step / stage (visible in nsys / ncu --nvtx)
        iterations = req.region.iterations if edit else 1
        # edit(): `iterations` rounds of the token loop, step = the global step index (iteration * timesteps + s); one round otherwise
        for step, (num_masked, steps_until_x0) in enumerate(zip(sched * iterations, list(reversed(range(timesteps))) * iterations)):
            s = step % timesteps
            if edit and s == 0:
                ops.edit_select(ids, scores, frozen, region["keep"], region["num_select"], self.mask_id, step // timesteps,
                                u=self._injected_noise(step, (b, n), device), seed_dev=self._seed_dev, row_offset=self.row_offset * n)
            if nvtx:
                if step:
                    torch.cuda.nvtx.range_pop()
                torch.cuda.nvtx.range_push(f"mmg.decode_step[{step}] masked={num_masked}")
            temp = lead(req.temperature) * (steps_until_x0 / timesteps)        # annealed, muse_maskgit_pytorch.py:578
            temp_dev = settings["temps"][s]
            u = self._injected_noise(step, (b, n, V), device)
            if native is not None:
                a = native["args"]
                a.ids = ids.data_ptr(); a.scores = scores.data_ptr(); a.masked_pos = masked_pos.data_ptr()
                a.num_masked = num_masked; a.k_keep = k_keep; a.step = step
                a.temperature = float(temp); a.cond_scale = float(lead(req.cond_scale))
                a.temperature_dev = temp_dev.data_ptr(); a.cond_scale_dev = settings["cond_scale"].data_ptr()
                a.u = None if u is None else u.data_ptr(); a.seed = 0; a.seed_dev = self._seed_dev.data_ptr(); a.row_offset = self.row_offset * n
                _lib.call("mmg_decode_step", a)
                continue
            if req.region is None:
                ops.remask(ids, scores, masked_pos, num_masked, self.mask_id)
            else:      # each image re-masks among its own regenerated tokens; num_masked rows per image, the surplus padded
                ops.remask_frozen(ids, scores, masked_pos, frozen, region["counts"][s], num_masked, self.mask_id)
            x = tr._run_blocks(ids, ctx, nb, sc_embed if (self.self_cond and s > 0) else None)
            if self.self_cond:                                                 # embed of the conditional forward, fed back next step (:574)
                ops.layernorm(x[:bn], P["gf"], sc_embed)
            # rows that are sampled: the masked ones; every position when already-decoded tokens may be re-masked by confidence
            pos, rows_b = (all_pos, n) if score_all else (masked_pos, num_masked)
            self._sample_tail(x, nb, pos, rows_b, ids, scores, float(temp), step, u, float(lead(req.cond_scale)), k_keep, tail, seed_dev=seed_dev,
                              only_masked_id=self.mask_id if score_all or req.region is not None else None, aten=aten_draw(step),
                              temp_dev=temp_dev, cond_scale_dev=settings["cond_scale"])
            if req.use_critic:
                xc = cnet._run_blocks(ids, cctx, cnb)
                ops.critic_score(xc[:bn], xc[bn:2 * bn] if cnb == 2 else None, gcrit, whead, float(bhead), float(lead(req.cond_scale)),
                                 float(lead(req.critic_noise_scale) * (steps_until_x0 / timesteps)), scores, u=self._injected_noise(step, (b, n), device),
                                 seed=0, seed_dev=seed_dev, step=step, row_offset=self.row_offset * n, aten=aten_draw(step, critic=True),
                                 cond_scale_dev=settings["crit_cond_scale"], noise_mul_dev=settings["crit_noise"][s])
        ids = ids.view(b, req.fmap_size, req.fmap_size)
        if nvtx:
            torch.cuda.nvtx.range_pop()
            torch.cuda.nvtx.range_push("mmg.vae_decode")
        images = self.vae.decode_from_ids(ids)
        if nvtx:
            torch.cuda.nvtx.range_pop()
        return images, ids, (tail.get("status") if tail is not None else None)

    def forward(self, images_or_ids, ignore_index=-1, cond_images: Optional[torch.Tensor] = None, cond_token_ids: Optional[torch.Tensor] = None,
                texts: Optional[List[str]] = None, text_embeds: Optional[torch.Tensor] = None, cond_drop_prob=None, train_only_generator=False,
                sample_temperature=None):
        """The training objective of the reference (muse_maskgit_pytorch.py:623-741), evaluated without gradients: the mean cross-entropy of
        the masked tokens, plus critic_loss_weight * the token critic's BCE when a critic is present and train_only_generator is False.
        Returns a 0-d fp32 tensor on the model's device (NaN when no position is labelled, as F.cross_entropy).

        The random draws are the reference's, in its order, from torch on the model's device (python's `random` for the self-conditioning
        and sampling-temperature draws): with `sampler_noise_fn` set, every torch uniform draw is noise_fn(0, shape) instead.  The gumbel
        noise of the critic branch follows `sampler_rng` as in generate().  Must run under torch.no_grad() / torch.inference_mode()."""
        if torch.is_grad_enabled():
            raise RuntimeError("MaskGit.forward evaluates the loss without gradients (there are no backward kernels): call it under "
                               "torch.no_grad() or torch.inference_mode()")
        tr = self.transformer
        V, mask_id = tr.num_tokens, self.mask_id
        device = next(self.parameters()).device
        if images_or_ids.dtype == torch.float:
            assert all(s == self.image_size for s in images_or_ids.shape[-2:]), "the image you passed in is not of the correct dimensions"
        else:
            assert not self.resize_image_for_cond_image, ("you cannot pass in raw image token ids if you want the framework to autoresize image "
                                                          "for conditioning super res transformer")
            self._check_ids(images_or_ids, "images_or_ids")
        assert not (cond_images is not None and cond_token_ids is not None), \
            "if conditioning on low resolution, cannot pass in both images and token ids"
        if cond_token_ids is not None:
            self._check_ids(cond_token_ids, "cond_token_ids")
        assert (texts is None) != (text_embeds is None), "pass exactly one of texts / text_embeds"
        self._check_weights()
        if images_or_ids.dtype == torch.float:
            ids = self.vae.encode_ids(images_or_ids.to(device, torch.float32).contiguous())
        else:
            ids = images_or_ids.to(device, torch.long)
        ids = ids.reshape(ids.shape[0], -1)
        b, n = ids.shape
        cond_drop_prob = self.cond_drop_prob if cond_drop_prob is None else cond_drop_prob
        if cond_images is not None:
            assert all(s == self.cond_image_size for s in cond_images.shape[-2:])
            cond_token_ids = self.cond_vae.encode_ids(cond_images.to(device, torch.float32).contiguous())
        cond_ids = None if cond_token_ids is None else cond_token_ids.to(device, torch.long).reshape(b, -1).contiguous()
        if self.sampler_noise_fn is not None:
            draw = lambda shape: self._injected_noise(0, shape, device)
        else:
            draw = lambda shape: torch.zeros(shape, device=device).uniform_(0, 1)
        # ---- masks and labels (:670-686): labels use the mask before the no-mask subset is removed, the input x the mask after it
        num_token_masked = (n * self.noise_schedule(draw((b,)))).round().clamp(min=1)
        mask = draw((b, n)).argsort(dim=-1) < num_token_masked[:, None]
        labels = torch.where(mask, ids, ignore_index)
        if self.no_mask_token_prob > 0.:
            mask &= ~_mask_subset_prob(mask, self.no_mask_token_prob, draw)
        x = torch.where(mask, mask_id, ids).contiguous()
        flat = (labels != ignore_index).reshape(-1)
        R = int(flat.sum().item())
        if R == 0:
            return torch.full((), float("nan"), device=device)
        pos = flat.nonzero()[:, 0].to(torch.int32).contiguous()                   # labelled flat positions, ascending
        lab = labels.reshape(-1)[pos.long()].to(torch.int32).contiguous()
        if texts is not None:
            text_embeds = tr.encode_text(texts)
        text_embeds = text_embeds.to(device, torch.float32)
        P = tr._packed()
        # ---- self-conditioning (:696-708): one stack without drop, its final-LayerNorm embed fed to the loss pass
        sc_embed = None
        if tr.self_cond and random.random() < self.self_cond_prob:
            xs = tr._run_blocks(x, tr._prepare_context(text_embeds, cond_ids, [False]), 1)
            sc_embed = torch.empty((b * n, tr.dim), device=device, dtype=torch.float32)
            ops.layernorm(xs, P["gf"], sc_embed)
        # ---- the loss pass (:712-720): final LayerNorm of the labelled rows only, then to_logits + cross-entropy
        te = self._drop_text(text_embeds, cond_drop_prob, draw)
        xres = tr._run_blocks(x, tr._prepare_context(te, cond_ids, [cond_drop_prob == 1]), 1, sc_embed)
        e = torch.empty((R, tr.dim), device=device, dtype=P["adt"])
        ops.final_embed(xres, None, P["gf"], pos, e, 1, b * n, R, 1.)
        nll = torch.empty((R,), device=device, dtype=torch.float32)
        use_critic = self.token_critic is not None and not train_only_generator
        nbytes = 0
        if self.use_fused_tail and P["adt"] == torch.bfloat16 and not use_critic:
            nbytes = ops.logits_xent_workspace_bytes(R, V, tr.dim)
        if nbytes:
            ops.logits_xent(e, P["wlog"], lab, nll, torch.empty((nbytes,), dtype=torch.uint8, device=device))
        else:
            logits = torch.empty((R, V), device=device, dtype=torch.float32)
            ops.linear(e, P["wlog"], logits)
            ops.logits_xent_rows(logits, lab, nll)
        ce_loss = nll.mean()
        if not use_critic:
            return ce_loss
        # ---- token critic (:728-741): gumbel sample over the full vocabulary at the masked rows, then the critic's BCE over all b * n
        temperature = random.random()                                          # drawn even when given: default(...) evaluates it
        if sample_temperature is not None:
            temperature = sample_temperature
        critic_input = x.clone()
        kw = dict(seed=0, step=0, row_offset=0, only_masked_id=mask_id)
        if self.sampler_noise_fn is not None:
            kw["u"] = draw((b, n, V))
        elif self.sampler_rng == "aten":
            stride, inc = _aten_uniform_geometry(device, b * n * V)
            seed, off = _reserve_aten_offsets(device, inc)
            kw.update(seed=seed, aten=(off, None, stride))
        else:
            assert self.sampler_rng == "mmg", self.sampler_rng
            kw["seed"] = self.sampler_seed if self.sampler_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
        # one sequence of b * n positions: the noise of flat position p is that of (p // n, p % n) in the (b, n, V) draw
        ops.logits_sample(logits, pos.view(1, R), critic_input.view(1, b * n), torch.empty((1, b * n), device=device), R, V,
                          float(temperature), **kw)
        critic_labels = (ids != critic_input).float()
        te_c = self._drop_text(text_embeds, cond_drop_prob, draw)
        cnet, _, cctx, whead, bhead, gcrit = self._resolve_critic(te_c, cond_ids, [cond_drop_prob == 1])
        xc = cnet._run_blocks(critic_input, cctx, 1)
        critic_logits = torch.empty((b * n,), device=device, dtype=torch.float32)
        ops.critic_score(xc, None, gcrit, whead, float(bhead), 1., 0., critic_logits)
        bce_loss = torch.nn.functional.binary_cross_entropy_with_logits(critic_logits.view(b, n), critic_labels)
        return ce_loss + self.critic_loss_weight * bce_loss

    def _check_ids(self, t, name):
        """Token ids must lie in [0, num_tokens): checked on the host side before any kernel reads them (the reference would hit a
        device-side assert in the embedding)."""
        V = self.transformer.num_tokens
        if t.numel() and (int(t.min()) < 0 or int(t.max()) >= V):
            raise ValueError(f"{name} must lie in [0, num_tokens = {V}); got values in [{int(t.min())}, {int(t.max())}]")

    @staticmethod
    def _drop_text(text_embeds, cond_drop_prob, draw):
        """The conditioning drop of Transformer.forward (muse_maskgit_pytorch.py:306-310, prob_mask_like :393-399): a dropped sequence's text
        embeddings are zeroed, which masks its text keys.  Draws only when 0 < cond_drop_prob < 1; 1 drops every text key through the
        branch flag of _prepare_context."""
        if not 0. < cond_drop_prob < 1.:
            return text_embeds
        keep = draw((text_embeds.shape[0], 1)) < (1. - cond_drop_prob)
        return text_embeds * keep[:, :, None]


# ------------------------------------------------------------------------------------------------ Muse
class Muse(nn.Module):
    """ref: muse_maskgit_pytorch.py:745-791 — base -> super-resolution cascade; the low-res images stay on the device."""
    def __init__(self, base: MaskGit, superres: MaskGit):
        super().__init__()
        assert isinstance(base, MaskGit) and isinstance(superres, MaskGit)
        self.base_maskgit = base.eval()
        assert superres.resize_image_for_cond_image
        self.superres_maskgit = superres.eval()

    @torch.no_grad()
    def forward(self, texts: List[str], cond_scale=3., temperature=1., timesteps=18, superres_timesteps=None,
                return_lowres=False, return_pil_images=True):
        """cond_scale / temperature: a number or per image (see MaskGit.generate), used by both stages."""
        lowres = self.base_maskgit.generate(texts=texts, cond_scale=cond_scale, temperature=temperature, timesteps=timesteps)
        superres = self.superres_maskgit.generate(texts=texts, cond_scale=cond_scale, cond_images=lowres, temperature=temperature,
                                                  timesteps=superres_timesteps if superres_timesteps is not None else timesteps)
        if return_pil_images:
            import torchvision.transforms as T
            lowres = list(map(T.ToPILImage(), lowres))
            superres = list(map(T.ToPILImage(), superres))
        return (superres, lowres) if return_lowres else superres

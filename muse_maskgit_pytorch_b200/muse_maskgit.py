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
import math
import os
from functools import partial
from pathlib import Path
from typing import Callable, List, Optional

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
        assert dim_head == 64, ("dim_head must be 64 here: the wgmma attention kernel (one 128-byte swizzled row per head "
                                "vector) and the QKV epilogue are specialised for the head size every Muse config uses; the reference accepts "
                                "any value (muse_maskgit_pytorch.py:95-110, 164-172)")
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
        return torch.bfloat16 if self.precision == "bf16" else torch.float32

    def _packed(self):
        if self._pack is not None and self._pack["adt"] == self._adt():
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
        P = dict(adt=adt, layers=[])

        def ff_pack(ff):
            F_ = ff[3].gamma.shape[0]
            Fp = _round_up(F_, 64)
            w1 = ff[1].weight.detach().to(dev, torch.float32)                  # (2F, dim): rows [0,F) -> gelu arm, [F,2F) -> gate
            w1p = torch.zeros((2 * Fp, w1.shape[1]), device=dev)
            xi = torch.arange(Fp, device=dev).view(-1, 32)
            dst_x = (xi // 32 * 64 + xi % 32).reshape(-1)                       # unit u -> row 64*(u//32) + u%32 ; gate -> +32
            valid = torch.arange(Fp, device=dev) < F_
            w1p[dst_x[valid]] = w1[:F_]
            w1p[dst_x[valid] + 32] = w1[F_:]
            g3 = torch.zeros(Fp, device=dev); g3[:F_] = ff[3].gamma.detach().float()
            w2 = torch.zeros((ff[4].weight.shape[0], Fp), device=dev); w2[:, :F_] = ff[4].weight.detach().float()
            out = dict(F=F_, Fp=Fp, g0=f32(ff[0].gamma), w1=w1p.to(adt).contiguous(), g3=g3.contiguous(), w2=w2.to(adt).contiguous())
            if adt == torch.bfloat16:
                # LayerNorm(inner) folded through the second linear: LN(h) W2^T = rstd * (h (W2*gamma)^T - mean * cvec), cvec = rowsum(W2*gamma)
                w2f = (w2 * g3[None, :]).to(adt).contiguous()
                out["w2f"], out["cvec"] = w2f, w2f.float().sum(dim=1).contiguous()
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
        heads = tb.heads
        tk_alloc = _round_up(m + 1, 8)
        kvs = []
        for lay in P["layers"]:
            ca = lay["ca"]
            k = torch.zeros((b * heads, tk_alloc, 64), device=dev, dtype=adt)
            v = torch.zeros((b * heads, tk_alloc, 64), device=dev, dtype=adt)
            epi = ops.qkv_epilogue(adt, heads, m, k=k, v=v, k_scale=ca["ks"], key_off=1, null_k=ca["nk"], null_v=ca["nv"])
            ops.linear(ctx, ca["wkv"], None, epilogue=ops.EPI_QKV, epi=epi)
            if len(branches) > 1:
                k, v = k.repeat(len(branches), 1, 1), v.repeat(len(branches), 1, 1)
            kvs.append((k, v))
        return dict(kv=kvs, key_mask=key_mask, m=m, all_masked=[bool(d) and cond_ids is None for d in branches])

    # ----- the block stack over R = nb*b*n rows -------------------------------------------------------------------------
    def _workspace(self, nb, b, n, dev):
        key = (nb, b, n, str(dev), self._adt())
        cache = self.__dict__.setdefault("_ws", {})        # a few shapes stay resident (e.g. 2-branch decode + 1-branch self-critic)
        if key in cache:
            return cache[key]
        P = self._packed()
        adt, tb = P["adt"], self.transformer_blocks
        heads, dim, inner = tb.heads, self.dim, tb.heads * 64
        R = nb * b * n
        Fp = max([l["ff"]["Fp"] for l in P["layers"]] + ([P["sc"]["Fp"]] if P["sc"] is not None else []))
        tk_alloc = _round_up(n + 1, 8)
        ws = dict(key=key,
                  x=torch.empty((R, dim), device=dev, dtype=torch.float32),
                  xn=torch.empty((R, dim), device=dev, dtype=adt),
                  q=torch.empty((nb * b * heads, n, 64), device=dev, dtype=adt),
                  k=torch.zeros((nb * b * heads, tk_alloc, 64), device=dev, dtype=adt),
                  v=torch.zeros((nb * b * heads, tk_alloc, 64), device=dev, dtype=adt),
                  ao=torch.empty((R, inner), device=dev, dtype=adt),
                  h=torch.empty((R, Fp), device=dev, dtype=adt),
                  hn=torch.empty((R, Fp), device=dev, dtype=adt),
                  stats=torch.zeros((R, Fp // 32, 2), device=dev, dtype=torch.float32))   # per-chunk (sum, sumsq) of the GEGLU output
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
        live = [j for j in range(nb) if not ctx["all_masked"][j]]
        for li, lay in enumerate(P["layers"]):
            sa, ca, ff = lay["sa"], lay["ca"], lay["ff"]
            # --- self attention (all branches) ---
            ops.layernorm(x, sa["g"], xn)
            epi = ops.qkv_epilogue(adt, heads, n, q=q, k=k, v=v, q_scale=sa["qs"], k_scale=sa["ks"], key_off=1,
                                   null_k=sa["nk"], null_v=sa["nv"])
            ops.linear(xn, sa["wqkv"], None, epilogue=ops.EPI_QKV, epi=epi)
            ops.attention(q, k, v, ao, nb * b, heads, n + 1, logit_bound=sa["bound"])
            ops.linear(ao, sa["wo"], x, epilogue=ops.EPI_RESIDUAL, resid=x)
            # --- cross attention ---
            kc, vc = ctx["kv"][li]
            pending_add = {j: ca["null_out"] for j in range(nb) if ctx["all_masked"][j]}
            if live:
                assert live == list(range(len(live))), "live branches must come first"
                Rl = len(live) * bn
                ops.layernorm(x[:Rl], ca["g"], xn[:Rl])
                epi = ops.qkv_epilogue(adt, heads, n, q=q[:len(live) * b * heads], q_scale=ca["qs"])
                ops.linear(xn[:Rl], ca["wq"], None, epilogue=ops.EPI_QKV, epi=epi)
                ops.attention(q[:len(live) * b * heads], kc[:len(live) * b * heads], vc[:len(live) * b * heads], ao[:Rl], len(live) * b, heads,
                              ctx["m"] + 1, key_mask=ctx["key_mask"][:len(live) * b], logit_bound=ca["bound"])
                ops.linear(ao[:Rl], ca["wo"], x[:Rl], epilogue=ops.EPI_RESIDUAL, resid=x[:Rl])
            # --- feed forward (the constant null-branch cross-attention term is folded into this LayerNorm) ---
            if pending_add and sorted(pending_add) == list(range(min(pending_add), nb)):
                # one launch for all branches: rows of the all-masked (null) branches get += to_out(null_v) before the norm
                ops.layernorm(x, ff["g0"], xn, add=ca["null_out"], x_out=x, add_from=min(pending_add) * bn)
            elif not pending_add:
                ops.layernorm(x, ff["g0"], xn)
            else:
                for j in range(nb):
                    xs = x[j * bn:(j + 1) * bn]
                    if j in pending_add:
                        ops.layernorm(xs, ff["g0"], xn[j * bn:(j + 1) * bn], add=pending_add[j], x_out=xs)
                    else:
                        ops.layernorm(xs, ff["g0"], xn[j * bn:(j + 1) * bn])
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
            ops.linear(xn[:R], ff["w1"], h, epilogue=ops.EPI_GEGLU, row_stats=stats)
            ops.linear(h, ff["w2f"], x[:R], epilogue=ops.EPI_LNFOLD_RESIDUAL, bias=ff["cvec"], resid=x[:R], row_stats=stats, ln_width=ff["F"])
            return
        ops.linear(xn[:R], ff["w1"], h, epilogue=ops.EPI_GEGLU)
        ops.layernorm(h, ff["g3"], hn, width=ff["F"])
        ops.linear(hn, ff["w2"], x[:R], epilogue=ops.EPI_RESIDUAL, resid=x[:R])

    def _ff(self, inp, ff, x_acc, ws, R):
        """x_acc += FeedForward(inp)   (self-conditioning embed, muse_maskgit_pytorch.py:325-328)"""
        xn = ws["xn"][:R]
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
        """ref: muse_maskgit_pytorch.py:491-621.  Returns fp32 NCHW images (b, 3, H, W), unclamped."""
        was_training = self.training
        self.eval()
        try:
            return self._generate(texts, negative_texts, cond_images, fmap_size, temperature, topk_filter_thres,
                                  can_remask_prev_masked, force_not_use_token_critic, timesteps, cond_scale, critic_noise_scale, return_ids)
        finally:
            self.train(was_training)

    def _generate(self, texts, negative_texts, cond_images, fmap_size, temperature, topk_filter_thres, can_remask_prev_masked,
                  force_not_use_token_critic, timesteps, cond_scale, critic_noise_scale, return_ids, seed=None):
        tr = self.transformer
        if negative_texts is not None:
            raise NotImplementedError("negative_texts raises TypeError in the reference (defect B2); not supported")
        use_critic = self.token_critic is not None and not force_not_use_token_critic
        if can_remask_prev_masked and not use_critic:      # the reference only reaches this assert in the no-critic branch (:611-612)
            assert self.no_mask_token_prob > 0., "without training with some of the non-masked tokens forced to predict, not sure if the logits will be meaningful for these token"
        fmap_size = fmap_size if fmap_size is not None else self.vae.get_encoded_fmap_size(self.image_size)
        device = next(self.parameters()).device
        b = len(texts)
        for net in (tr, self.vae, self.cond_vae, self.token_critic if isinstance(self.token_critic, Transformer) else None):
            if net is not None:
                net._check_weights()          # in-place parameter edits since the last call drop the packed copies (and the graphs below)
        text_embeds = tr.encode_text(texts).to(device, non_blocking=True)
        if self.use_cuda_graph and text_embeds.shape[1] % 32:
            # T5 pads to the longest prompt of the batch: bucket the length (multiples of 32) so that prompt lengths share captured
            # graphs; all-zero rows are padding to the reference too (masked keys, muse_maskgit_pytorch.py:304)
            text_embeds = torch.nn.functional.pad(text_embeds, (0, 0, 0, 32 - text_embeds.shape[1] % 32))
        if self.resize_image_for_cond_image:
            assert cond_images is not None, "conditioning image must be passed in to generate for super res maskgit"
            cond_images = cond_images.to(device, torch.float32)
        else:
            cond_images = None
        # per-call seed: explicit sampler_seed, else one draw from torch's global generator (reproducible under manual_seed)
        assert self.sampler_rng in ("mmg", "aten"), self.sampler_rng
        if getattr(self, "_seed_dev", None) is None or self._seed_dev.device != device:
            self._seed_dev = torch.zeros((1,), dtype=torch.int64, device=device)
        aten = None
        if self.sampler_rng == "aten" and self.sampler_noise_fn is None:
            aten = self._aten_plan(device, b, fmap_size ** 2, tr.num_tokens, timesteps, use_critic)
        elif self.sampler_noise_fn is None:      # (injected noise: the host generator is the caller's stream — nothing is drawn from it here)
            if seed is None:                     # (a rerun on the materialised path keeps the seed of the attempt it repeats)
                seed = self.sampler_seed if self.sampler_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
            self._seed_dev.fill_(seed)
        body = partial(self._generate_body, fmap_size=fmap_size, temperature=temperature, topk_filter_thres=topk_filter_thres,
                       timesteps=timesteps, cond_scale=cond_scale, b=b, use_critic=use_critic, critic_noise_scale=critic_noise_scale,
                       score_all=bool(can_remask_prev_masked) and not use_critic, aten=aten)
        critic_net = self.token_critic if isinstance(self.token_critic, Transformer) and use_critic else None
        if not self.use_cuda_graph or self.sampler_noise_fn is not None:
            images, ids, status = body(text_embeds, cond_images)
            if self._fused_tail_overflowed(status):
                return self._generate_unfused(seed, texts, negative_texts, cond_images, fmap_size, temperature, topk_filter_thres, can_remask_prev_masked,
                                              force_not_use_token_critic, timesteps, cond_scale, critic_noise_scale, return_ids)
            return (images, ids) if return_ids else images
        # ---- whole-call CUDA graph: 18 decode steps + VAE decode replayed as one launch (no per-kernel host work) ----
        key = (b, tuple(text_embeds.shape), text_embeds.dtype, None if cond_images is None else tuple(cond_images.shape), fmap_size,
               float(temperature), float(topk_filter_thres), int(timesteps), float(cond_scale), int(self.row_offset), tr.precision, self.vae.precision,
               use_critic, float(critic_noise_scale), bool(can_remask_prev_masked), None if aten is None else aten["key"], bool(self.use_native_step),
               id(self.noise_schedule), bool(self.use_fused_tail))
        pack_ids = lambda: (id(tr._pack), id(self.vae._pack), id(self.cond_vae._pack), id(critic_net._pack) if critic_net is not None else 0,
                            id(self.token_critic._head_cache) if isinstance(self.token_critic, SelfCritic) else 0)
        entry = self._graphs.get(key)
        if entry is not None and entry[5] != pack_ids():
            entry = None                                       # weights were re-packed (load_state_dict / .to()): re-capture
        if entry is None:
            te_s = text_embeds.clone()
            ci_s = None if cond_images is None else cond_images.clone()
            body(te_s, ci_s)                                   # eager warm-up: lazy packing, workspaces, function attributes
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out_images, out_ids, out_status = body(te_s, ci_s)
            # the entry keeps alive everything the captured kernels point at (packed weights, workspaces)
            entry = (graph, te_s, ci_s, out_images, (out_ids, out_status), pack_ids(),
                     (tr._pack, self.vae._pack, self.cond_vae._pack, dict(getattr(tr, "_ws", {})),
                      None if critic_net is None else (critic_net._pack, dict(getattr(critic_net, "_ws", {}))),
                      self.token_critic._head_cache if isinstance(self.token_critic, SelfCritic) else None))
            if len(self._graphs) >= 4:
                self._graphs.pop(next(iter(self._graphs)))       # least recently used (hits are moved to the end below)
        self._graphs.pop(key, None)
        self._graphs[key] = entry
        graph, te_s, ci_s, out_images, (out_ids, out_status) = entry[:5]
        te_s.copy_(text_embeds, non_blocking=True)
        if ci_s is not None:
            ci_s.copy_(cond_images, non_blocking=True)
        graph.replay()
        images, ids = out_images.clone(), out_ids.clone()
        if self._fused_tail_overflowed(out_status):
            return self._generate_unfused(seed, texts, negative_texts, cond_images, fmap_size, temperature, topk_filter_thres, can_remask_prev_masked,
                                          force_not_use_token_critic, timesteps, cond_scale, critic_noise_scale, return_ids)
        return (images, ids) if return_ids else images

    def _fused_tail_overflowed(self, status):
        """status[1] != 0: some decode step had more rows whose sampled top-k threshold missed than the fused path's fallback holds (e.g. constant
        logits rows).  One 4-byte read per call; `check_fused_tail = False` skips it (and the host synchronisation it implies)."""
        if status is None or not self.check_fused_tail:
            return False
        self.last_fused_fallback_rows, overflow = (int(v) for v in status.tolist())
        return overflow != 0

    def _generate_unfused(self, seed, *args):
        """Repeats a generate() call whose fused tail overflowed on the materialised path, with the same noise: the same libmmg seed, or the
        ATen generator position the failed attempt started from."""
        saved = self.use_fused_tail
        self.use_fused_tail = False
        try:
            if self.sampler_rng == "aten" and self.sampler_noise_fn is None:       # re-read the generator position the failed attempt consumed
                gen = torch.cuda.default_generators[next(self.parameters()).device.index or 0]
                gen.set_offset(self._aten_start_offset)
            return self._generate(*args, seed=seed)
        finally:
            self.use_fused_tail = saved

    def _native_step_setup(self, ctx, P, b, n, nb, max_masked, V, device):
        """Argument block of mmg_decode_step for this generate(): the packed weights and the per-call context as raw pointers, plus the
        zero-initialised workspace.  Everything referenced is kept alive by the returned dict (and by `P` / `ctx`)."""
        tr = self.transformer
        tb = tr.transformer_blocks
        depth = len(P["layers"])
        live = sum(1 for m in ctx["all_masked"][:nb] if not m)
        assert ctx["all_masked"][:nb] == [False] * live + [True] * (nb - live), "live CFG branches must come first"
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
        a.branches = nb; a.live_branches = live
        a.layers = ctypes.cast(layers, ctypes.POINTER(_lib.LayerWeights))
        a.tok_emb = P["tok"].data_ptr(); a.pos_emb = P["pos"].data_ptr(); a.final_gamma = P["gf"].data_ptr(); a.w_logits = P["wlog"].data_ptr()
        a.ctx_key_mask = ctx["key_mask"].data_ptr(); a.ctx_keys = ctx["m"]; a.ctx_alloc = ctx["kv"][0][0].shape[1]
        a.mask_id = self.mask_id
        a.workspace = ws.data_ptr(); a.workspace_bytes = nbytes
        return dict(args=a, layers=layers, ws=ws, ctx=ctx, P=P)

    def _aten_plan(self, device, b, n, V, timesteps, use_critic):
        """Offsets of the reference's uniform_ calls in torch's CUDA Philox stream (one (b, n, V) gumbel draw, then one (b, n) critic
        draw per step, muse_maskgit_pytorch.py:407, 598).  Launch geometry as ATen's calc_execution_policy: block 256,
        grid = min(SMs * maxThreadsPerSM / 256, ceil(numel / 256)), 4 values per thread and round.  The generator is read here and
        advanced by what the reference would have consumed; seed / offset reach the kernels through device words (graph replay)."""
        gen = torch.cuda.default_generators[device.index if device.index is not None else torch.cuda.current_device()]
        props = torch.cuda.get_device_properties(device)
        cap = props.multi_processor_count * (props.max_threads_per_multi_processor // 256)
        B = self.global_batch if self.global_batch is not None else b
        stride = lambda numel: 256 * min(cap, (numel + 255) // 256)
        inc = lambda numel: ((numel - 1) // (stride(numel) * 4) + 1) * 4
        ng, nc = B * n * V, B * n
        per_step = inc(ng) + (inc(nc) if use_critic else 0)
        seed, off = gen.initial_seed(), gen.get_offset()
        self._aten_start_offset = off
        gen.set_offset(off + timesteps * per_step)
        if getattr(self, "_aten_dev", None) is None or self._aten_dev.device != device:
            self._aten_dev = torch.zeros((2,), dtype=torch.int64, device=device)
        wrap = lambda v: v - (1 << 64) if v >= (1 << 63) else v
        self._aten_dev.copy_(torch.tensor([wrap(seed), off], dtype=torch.int64), non_blocking=False)
        return dict(key=(B, stride(ng), stride(nc), per_step), stride_g=stride(ng), stride_c=stride(nc), inc_g=inc(ng), per_step=per_step)

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

    def _sample_tail(self, x, nb, pos, rows_b, ids, scores, temp, step, u, cond_scale, k_keep, tail, seed_dev=None, only_masked_id=None, aten=None):
        """The sampling tail of one decode step (muse_maskgit_pytorch.py:576-609) on the rows listed in `pos` (b, rows_b): final LayerNorm +
        CFG combine in embedding space, to_logits, top-k filter, gumbel argmax, confidence score; ids / scores are updated in place.
        x: residual stream [nb*b*n, dim] after the blocks (cond rows first, then the null-CFG rows)."""
        tr = self.transformer
        P = tr._packed()
        b, n = ids.shape
        bn = b * n
        R = b * rows_b
        e = tail["e"]
        ops.final_embed(x[:bn], x[bn:2 * bn] if nb == 2 else None, P["gf"], pos, e, b, n, rows_b, cond_scale)
        kw = dict(u=u, seed=0, seed_dev=seed_dev, step=step, row_offset=self.row_offset * n, only_masked_id=only_masked_id, aten=aten)
        if "fused_ws" in tail:      # logits never reach HBM: candidate lists out of the GEMM epilogue, sampled by the finishing kernel
            ops.logits_fused(e[:R], P["wlog"], pos, ids, scores, rows_b, k_keep, temp, tail["fused_ws"], tail["status"],
                             rows_capacity=b * tail["rows_max"], **kw)
            return
        lg = tail["logits"][:R]
        ops.linear(e[:R], P["wlog"], lg)
        ops.logits_sample(lg, pos, ids, scores, rows_b, k_keep, temp, **kw)

    def _generate_body(self, text_embeds, cond_images, *, fmap_size, temperature, topk_filter_thres, timesteps, cond_scale, b,
                       use_critic=False, critic_noise_scale=1., score_all=False, aten=None):
        """The device-side work of generate(): no host synchronisation, no data-dependent host control flow."""
        tr = self.transformer
        device = text_embeds.device
        n = fmap_size ** 2
        V = tr.num_tokens
        cond_ids = self.cond_vae.encode_ids(cond_images) if cond_images is not None else None
        nb = 1 if cond_scale == 1 else 2
        ctx = tr._prepare_context(text_embeds, cond_ids, [False, True][:nb])
        P = tr._packed()
        adt = P["adt"]
        ids = torch.full((b, n), self.mask_id, dtype=torch.long, device=device)
        scores = torch.zeros((b, n), dtype=torch.float32, device=device)
        masked_pos = torch.empty((b, n), dtype=torch.int32, device=device)
        k_keep = math.ceil((1 - topk_filter_thres) * V)                        # muse_maskgit_pytorch.py:414
        sched = self.mask_schedule(n, timesteps)
        bn = b * n
        native = None
        if (self.use_native_step and adt == torch.bfloat16 and not self.self_cond and not use_critic and not score_all and aten is None
                and all("w2f" in l["ff"] for l in P["layers"])):
            native = self._native_step_setup(ctx, P, b, n, nb, max(sched), V, device)
        rows_max = n if score_all else max(sched)
        tail = self._tail_buffers(b, n, rows_max, V, device, k_keep) if native is None else None
        all_pos = torch.arange(n, dtype=torch.int32, device=device).repeat(b, 1).contiguous() if score_all else None
        sc_embed = torch.empty((bn, tr.dim), device=device, dtype=torch.float32) if self.self_cond else None
        # token critic (muse_maskgit_pytorch.py:535-538, 590-600): a second stack over the freshly filled ids scores EVERY position
        if use_critic:
            if isinstance(self.token_critic, SelfCritic):      # the generator itself; only its conditional embed is used (:352-361)
                cnet, cnb, cctx = tr, 1, ctx
                whead, bhead = self.token_critic._head()
                whead = whead.to(device)
            else:
                cnet, cnb = self.token_critic, nb
                cctx = cnet._prepare_context(text_embeds, cond_ids, [False, True][:nb])
                whead, bhead = cnet._packed()["whead"], 0.
                assert whead is not None, "token_critic must have dim_out == 1"
            gcrit = cnet._packed()["gf"]
        nvtx = os.environ.get("MMG_NVTX", "0") == "1"            # host-side NVTX ranges per decode step / stage (visible in nsys / ncu --nvtx)
        for step, (num_masked, steps_until_x0) in enumerate(zip(sched, reversed(range(timesteps)))):
            if nvtx:
                if step:
                    torch.cuda.nvtx.range_pop()
                torch.cuda.nvtx.range_push(f"mmg.decode_step[{step}] masked={num_masked}")
            if native is not None:
                u = None
                if self.sampler_noise_fn is not None:
                    u = self.sampler_noise_fn(step, (b, n, V)).to(device=device, dtype=torch.float32).contiguous()
                a = native["args"]
                a.ids = ids.data_ptr(); a.scores = scores.data_ptr(); a.masked_pos = masked_pos.data_ptr()
                a.num_masked = num_masked; a.k_keep = k_keep; a.step = step
                a.temperature = float(temperature * (steps_until_x0 / timesteps)); a.cond_scale = float(cond_scale)
                a.u = None if u is None else u.data_ptr(); a.seed = 0; a.seed_dev = self._seed_dev.data_ptr(); a.row_offset = self.row_offset * n
                _lib.call("mmg_decode_step", a)
                continue
            ops.remask(ids, scores, masked_pos, num_masked, self.mask_id)
            x = tr._run_blocks(ids, ctx, nb, sc_embed if (self.self_cond and step > 0) else None)
            if self.self_cond:                                                 # embed of the conditional forward, fed back next step (:574)
                ops.layernorm(x[:bn], P["gf"], sc_embed)
            # rows that are sampled: the masked ones; every position when already-decoded tokens may be re-masked by confidence
            pos, rows_b = (all_pos, n) if score_all else (masked_pos, num_masked)
            temp = temperature * (steps_until_x0 / timesteps)                  # annealed, muse_maskgit_pytorch.py:578
            u = None
            if self.sampler_noise_fn is not None:
                u = self.sampler_noise_fn(step, (b, n, V)).to(device=device, dtype=torch.float32).contiguous()
            seed_dev = self._seed_dev if aten is None else self._aten_dev[0:1]
            self._sample_tail(x, nb, pos, rows_b, ids, scores, float(temp), step, u, float(cond_scale), k_keep, tail, seed_dev=seed_dev,
                              only_masked_id=self.mask_id if score_all else None,
                              aten=None if aten is None else (step * aten["per_step"], self._aten_dev[1:2], aten["stride_g"]))
            if use_critic:
                xc = cnet._run_blocks(ids, cctx, cnb)
                uc = None
                if self.sampler_noise_fn is not None:
                    uc = self.sampler_noise_fn(step, (b, n)).to(device=device, dtype=torch.float32).contiguous()
                ops.critic_score(xc[:bn], xc[bn:2 * bn] if cnb == 2 else None, gcrit, whead, float(bhead), float(cond_scale),
                                 float(critic_noise_scale * (steps_until_x0 / timesteps)), scores, u=uc, seed=0, seed_dev=seed_dev,
                                 step=step, row_offset=self.row_offset * n,
                                 aten=None if aten is None else (step * aten["per_step"] + aten["inc_g"], self._aten_dev[1:2], aten["stride_c"]))
        ids = ids.view(b, fmap_size, fmap_size)
        if nvtx:
            torch.cuda.nvtx.range_pop()
            torch.cuda.nvtx.range_push("mmg.vae_decode")
        images = self.vae.decode_from_ids(ids)
        if nvtx:
            torch.cuda.nvtx.range_pop()
        return images, ids, (tail.get("status") if tail is not None else None)

    def forward(self, *args, **kwargs):
        raise NotImplementedError("MaskGit.forward is the training loss (muse_maskgit_pytorch.py:623-741); training is out of scope")


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
        lowres = self.base_maskgit.generate(texts=texts, cond_scale=cond_scale, temperature=temperature, timesteps=timesteps)
        superres = self.superres_maskgit.generate(texts=texts, cond_scale=cond_scale, cond_images=lowres, temperature=temperature,
                                                  timesteps=superres_timesteps if superres_timesteps is not None else timesteps)
        if return_pil_images:
            import torchvision.transforms as T
            lowres = list(map(T.ToPILImage(), lowres))
            superres = list(map(T.ToPILImage(), superres))
        return (superres, lowres) if return_lowres else superres

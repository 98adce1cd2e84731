"""GPU parity tests ON THE BENCHMARKED PATH at the BASELINE configs (bf16 / wgmma, the kernels bench.py times):

  C2  MaskGitTransformer dim 512, depth 8, seq 256, V = 65536: full forward with CFG vs the fp32 CPU oracle;
  C3  MaskGit.generate() decode steps, teacher forced with the oracle's ids and noise, at the full model config: sampled-token flip rate;
  C4  super-resolution transformer (seq 1024, depth 2, 32 text + 256 conditioning tokens): forward vs the oracle (1025 / 289-key attention);
  C5  VQGanVAE dim 256 at 512 x 512: encode -> LFQ ids -> decode vs the oracle;
  every tc_gemm_kernel instantiation at the shapes generate() launches, against an fp32 torch matmul / conv of the same bf16 inputs.

Weights: the modules' own default init under torch.manual_seed (as bench.py); the oracle receives the same state_dict.
Tolerances (bf16 operands, fp32 accumulation; SURVEY.md section 7): logits rel-L2 <= 2e-2, pixels max-abs <= 5e-2 of the output range,
teacher-forced flip rate <= 8 % (the reference's own bf16-vs-fp32 argmax disagreement is 3-5 %, BASELINE.md section 2).
"""
import math
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import muse_oracle as O

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
bf = torch.bfloat16
TR_BASE = dict(num_tokens=65536, seq_len=256, dim=512, depth=8, dim_head=64, heads=8, ff_mult=4)
TR_SR = dict(num_tokens=65536, seq_len=1024, dim=512, depth=2, dim_head=64, heads=8, ff_mult=4)


def M():
    import muse_maskgit_pytorch_b200 as m
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-512"] = {"d_model": 512}
    return m


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm())


def cpu_sd(module):
    return {k: v.detach().float().cpu() for k, v in module.state_dict().items()}


def text_embeds(b, seed=1):
    te = torch.randn((b, 32, 512), generator=torch.Generator().manual_seed(seed))
    te[1::2, 24:] = 0.
    return te


def set_threads():
    import os
    torch.set_num_threads(min(os.cpu_count() or 1, 32))


_cache = {}


def base_transformer():
    if "base" not in _cache:
        torch.manual_seed(0)
        tr = M().MaskGitTransformer(t5_name="synth-512", precision="bf16", **TR_BASE)
        _cache["base"] = (tr.cuda(), cpu_sd(tr))
    return _cache["base"]


# ------------------------------------------------------------------------------------------------ C2
def test_c2_full_config_forward_bf16_vs_oracle():
    set_threads()
    tr, sd = base_transformer()
    te = text_embeds(2)
    ids = torch.randint(0, 65537, (2, 256), generator=torch.Generator().manual_seed(5))
    ref, ref_embed = O.forward_with_cond_scale(sd, dict(heads=8, depth=8), ids, te, cond_scale=3.)
    got, embed = tr.forward_with_cond_scale(ids.cuda(), text_embeds=te.cuda(), cond_scale=3., return_embed=True)
    r, re_ = rel_l2(got, ref), rel_l2(embed, ref_embed)
    agree = float((got.cpu().argmax(-1) == ref.argmax(-1)).float().mean())
    top2 = ref.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > 4 * float((got.cpu() - ref).abs().max())
    agree_clear = float((got.cpu().argmax(-1) == ref.argmax(-1))[clear].float().mean()) if bool(clear.any()) else 1.0
    print(f"C2 full config (depth 8, V 65536, B 2) bf16 vs fp32 oracle: logits rel-L2 {r:.3e}, embed rel-L2 {re_:.3e}, argmax agreement {agree:.4f} "
          f"(clear-margin rows {int(clear.sum())}: {agree_clear:.4f})")
    assert r < 2e-2 and re_ < 1.5e-2
    assert agree_clear == 1.0          # an argmax may only move where the fp32 top-2 margin is within the bf16 error
    assert agree > 0.80


# ------------------------------------------------------------------------------------------------ C3 teacher forced
class _Trace(list):
    """keeps the per-step tensors the teacher-forced comparison needs and drops the [b, n, V] logits"""
    def append(self, st):
        st = dict(st); st.pop("logits", None); st.pop("embed", None)
        super().append(st)


def _c3_trace():
    """The fp32 oracle's 18-step trace at the C3 model config (ids in / out, noise, scores per step), computed once per test session."""
    if "c3_trace" not in _cache:
        set_threads()
        _, sd = base_transformer()
        te = text_embeds(2)
        g = torch.Generator().manual_seed(2)
        noise = lambda step, shape: torch.rand(shape, generator=g)
        trace = _Trace()
        O.generate_ids(sd, dict(heads=8, depth=8), te, 256, 65536, noise, timesteps=18, cond_scale=3., trace=trace)
        _cache["c3_trace"] = (te, trace)
    return _cache["c3_trace"]


def _c3_teacher_forced(tr):
    """Runs the decode step the bench times (block stack -> final LayerNorm + CFG -> logits -> top-k / gumbel / confidence) on `tr`, fed with
    the fp32 oracle's ids and the oracle's noise on every one of the 18 steps.  Returns (flips, masked tokens, per-step flips, worst score diff)."""
    m = M()
    torch.manual_seed(0)
    vae = m.VQGanVAE(dim=16, layers=4, codebook_size=65536, precision=tr.precision)   # the token loop does not touch the VAE
    mg = m.MaskGit(image_size=256, transformer=tr, vae=vae.cuda()).cuda()
    b, n, V = 2, 256, 65536
    te, trace = _c3_trace()
    ctx = tr._prepare_context(te.cuda(), None, [False, True])
    tail = mg._tail_buffers(b, n, n, V, torch.device("cuda"), math.ceil(0.1 * V))
    k_keep = math.ceil(0.1 * V)
    flips = total = 0
    worst_score = 0.
    per_step = []
    for step, st in enumerate(trace):
        ids_in = st["ids_in"].cuda()
        nm = st["num_masked"]
        mp = torch.stack([torch.nonzero(ids_in[i] == V).flatten() for i in range(b)]).int().contiguous()
        assert mp.shape == (b, nm)
        x = tr._run_blocks(ids_in, ctx, 2)
        ids = ids_in.clone(); sc = torch.full((b, n), -1e5, device="cuda")
        mg._sample_tail(x, 2, mp, nm, ids, sc, float(st["temperature"]), step, st["u"].cuda().contiguous(), 3.0, k_keep, tail)
        is_mask = st["ids_in"] == V
        same = ids.cpu() == st["ids_out"]
        f = int((~same & is_mask).sum())
        flips += f; total += int(is_mask.sum())
        per_step.append(f)
        ok = same & is_mask
        if bool(ok.any()):
            worst_score = max(worst_score, float((sc.cpu() - st["scores"])[ok].abs().max()))
        assert bool((ids.cpu()[~is_mask] == st["ids_in"][~is_mask]).all())                      # unmasked positions are never touched
    return flips, total, per_step, worst_score


def test_c3_teacher_forced_flip_rate_full_config():
    """bf16 operands (the timed path): a sampled token may differ from the fp32 oracle's only through the bf16 rounding of the logits.  Also
    checks the confidence scores on the agreeing positions."""
    tr, _ = base_transformer()
    flips, total, per_step, worst_score = _c3_teacher_forced(tr)
    rate = flips / total
    print(f"C3 full-config teacher-forced flip rate {flips}/{total} = {rate:.4f} (per step {per_step}); max |score diff| on agreeing tokens {worst_score:.2e}")
    assert rate < 0.08
    assert worst_score < 2e-3


def test_c3_teacher_forced_token_identical_fp32_on_tensor_cores():
    """precision='fp32' at the SAME full C3 config, on the SAME wgmma GEMM / attention kernels (operands as 3-way bf16 splits, six cross terms
    per product, fp32 accumulation; no CUDA-core GEMM or attention launch): every one of the 5 782 sampled tokens of the 18 teacher-forced
    steps equals the fp32 oracle's token.  (A token could still differ where the oracle's own top-2 margin is below fp32 summation noise.)"""
    from muse_maskgit_pytorch_b200 import _lib
    bf_tr, _ = base_transformer()
    torch.manual_seed(0)
    tr = M().MaskGitTransformer(t5_name="synth-512", precision="fp32", **TR_BASE)
    tr.load_state_dict(bf_tr.state_dict())
    tr = tr.cuda()
    assert ops().fp32_tc()
    fb0 = _lib.simt_launch_count()
    flips, total, per_step, worst_score = _c3_teacher_forced(tr)
    print(f"C3 full-config teacher-forced, fp32 on wgmma (3-way bf16 split): {flips}/{total} tokens differ (per step {per_step}); "
          f"max |score diff| {worst_score:.2e}; CUDA-core GEMM / attention launches {_lib.simt_launch_count() - fb0}")
    assert flips <= 1 and worst_score < 5e-5
    assert _lib.simt_launch_count() == fb0


# ------------------------------------------------------------------------------------------------ C4
def test_c4_superres_forward_bf16_vs_oracle():
    """Super-resolution transformer at the C4 geometry: 1024 tokens (1025-key self-attention), context = 32 text + 256 conditioning tokens
    (289-key masked cross-attention in the cond branch; the null branch still attends the conditioning tokens)."""
    set_threads()
    torch.manual_seed(1)
    tr = M().MaskGitTransformer(t5_name="synth-512", precision="bf16", **TR_SR).cuda()
    sd = cpu_sd(tr)
    te = text_embeds(2, seed=3)
    gen = torch.Generator().manual_seed(6)
    ids = torch.randint(0, 65537, (2, 1024), generator=gen)
    cond_ids = torch.randint(0, 65536, (2, 256), generator=gen)
    ref, _ = O.forward_with_cond_scale(sd, dict(heads=8, depth=2), ids, te, cond_ids, 3.)
    got = tr.forward_with_cond_scale(ids.cuda(), text_embeds=te.cuda(), conditioning_token_ids=cond_ids.cuda(), cond_scale=3.)
    r = rel_l2(got, ref)
    agree = float((got.cpu().argmax(-1) == ref.argmax(-1)).float().mean())
    print(f"C4 super-res forward (n 1024, depth 2, ctx 32+256) bf16 vs fp32 oracle: logits rel-L2 {r:.3e}, argmax agreement {agree:.4f}")
    assert r < 2e-2 and agree > 0.80


# ------------------------------------------------------------------------------------------------ C5
def test_c5_vae_512_bf16_vs_oracle():
    """VQGanVAE dim 256, codebook 65536 at 512 x 512 (b = 1): LFQ bits may flip only where the fp32 projection is within bf16 noise of
    zero; the decoder is compared from the ORACLE's ids (pixels), and vae(x) == decode_from_ids(encode(x).ids)."""
    set_threads()
    torch.manual_seed(0)
    vae = M().VQGanVAE(dim=256, codebook_size=65536, precision="bf16").cuda()
    sd = cpu_sd(vae)
    img = torch.rand((1, 3, 512, 512), generator=torch.Generator().manual_seed(7))
    fmap = O.vae_encode_fmap(sd, img)
    proj = fmap.permute(0, 2, 3, 1).reshape(-1, fmap.shape[1]) @ sd["quantizer.project_in.weight"].t() + sd["quantizer.project_in.bias"]
    _, ref_ids = O.lfq_quantize(sd, fmap)
    ref_img = O.vae_decode_from_ids(sd, ref_ids, 16)
    fq, ids, _ = vae.encode(img.cuda())
    assert ids.shape == (1, 32, 32)
    flips = ((ids.cpu().reshape(-1, 1) >> torch.arange(15, -1, -1)) & 1) != (proj > 0).long()
    nflip = int(flips.sum())
    scale = float(proj.abs().mean())
    print(f"C5 VAE 512x512: {nflip} of {flips.numel()} LFQ bits differ; |proj| at flipped bits <= {float(proj.abs()[flips].max()) if nflip else 0.:.3e} (mean |proj| {scale:.3e})")
    assert nflip == 0 or float(proj.abs()[flips].max()) < 0.05 * max(scale, 1e-6) + 2e-2
    rec = vae.decode_from_ids(ref_ids.cuda())
    err = float((rec.cpu() - ref_img).abs().max())
    rng = float(ref_img.abs().max())
    print(f"C5 decode from the oracle's ids: max |pixel diff| {err:.3e} (output range {rng:.3e}), rel-L2 {rel_l2(rec, ref_img):.3e}")
    assert err < 5e-2 * max(rng, 1.0) and rel_l2(rec, ref_img) < 2e-2
    assert torch.equal(vae(img.cuda()), vae.decode_from_ids(ids))


# ------------------------------------------------------------------------------------------------ GEMM instantiations at generate() shapes
def grand(shape, seed, std=1.0, dtype=bf):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * std).to(dtype)


def close(a, b, atol, rtol):
    err = (a.float() - b.float()).abs()
    ok = bool((err <= atol + rtol * b.float().abs()).all())
    return ok, f"max abs err {float(err.max()):.3e}, mean {float(err.mean()):.3e} (ref max {float(b.float().abs().max()):.3e})"


@pytest.fixture(autouse=True)
def _fp32_reference_math():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("q_only", [False, True], ids=["self_qkv_32768x1536x512", "cross_q_16384x512x512"])
def test_gemm_generate_shape_qkv(q_only):
    """The QKV tile epilogue: the self-attention QKV product of a batch-64 CFG step (128 sequences x 256 tokens; tc_gemm_kernel<256, 4>)
    and the cross-attention q product of its 64 conditional sequences (tc_gemm_kernel<128, 4>)."""
    o = ops()
    b, n, heads, dim = (64 if q_only else 128), 256, 8, 512
    inner, nsec = heads * 64, (1 if q_only else 3)
    x, w = grand((b * n, dim), 1), grand((nsec * inner, dim), 2, dim ** -0.5)
    qs, ks = 1 + 0.1 * grand((64,), 3, dtype=torch.float32), 1 + 0.1 * grand((64,), 4, dtype=torch.float32)
    nk, nv = grand((heads, 64), 5), grand((heads, 64), 6)
    q = torch.zeros((b * heads, n, 64), device="cuda", dtype=bf)
    k = torch.zeros((b * heads, n + 8, 64), device="cuda", dtype=bf)
    v = torch.zeros_like(k)
    e = o.qkv_epilogue(bf, heads, n, q=q, q_scale=qs) if q_only else \
        o.qkv_epilogue(bf, heads, n, q=q, k=k, v=v, q_scale=qs, k_scale=ks, key_off=1, null_k=nk, null_v=nv)
    o.linear(x, w, None, epilogue=o.EPI_QKV, epi=e)
    y = (x.float() @ w.float().t()).view(b, n, nsec, heads, 64).permute(2, 0, 3, 1, 4)
    ok, msg = close(q.view(b, heads, n, 64), F.normalize(y[0], dim=-1) * qs, 2e-2, 1e-2)
    assert ok, "q: " + msg
    if not q_only:
        kk, vv = k.view(b, heads, n + 8, 64), v.view(b, heads, n + 8, 64)
        ok, msg = close(kk[:, :, 1:n + 1], F.normalize(y[1], dim=-1) * ks, 2e-2, 1e-2)
        assert ok, "k: " + msg
        ok, msg = close(vv[:, :, 1:n + 1], y[2], 2e-2, 1e-2)
        assert ok, "v: " + msg
        assert torch.equal(kk[:, :, 0], nk.expand(b, -1, -1)) and torch.equal(vv[:, :, 0], nv.expand(b, -1, -1))
        assert float(kk[:, :, n + 1:].abs().max()) == 0.


def test_gemm_generate_shape_ff_geglu_lnfold():
    """FF1 32768 x 2816 x 512 with the GEGLU tile epilogue + row statistics (tc_gemm_kernel<256, 5>) and FF2 32768 x 512 x 1408 with
    the LayerNorm fold and the in-place TMA reduction (tc_gemm_kernel<256, 2>), i.e. x += LN(gate * gelu(a Wx)) W2^T."""
    o = ops()
    M_, K, Fu, Fp, dim = 32768, 512, 1365, 1408, 512
    a = grand((M_, K), 11)
    wx, wg = grand((Fu, K), 12, K ** -0.5), grand((Fu, K), 13, K ** -0.5)
    wxp, wgp = torch.zeros((Fp, K), device="cuda", dtype=bf), torch.zeros((Fp, K), device="cuda", dtype=bf)
    wxp[:Fu], wgp[:Fu] = wx, wg
    w1 = torch.stack((wxp.view(-1, 32, K), wgp.view(-1, 32, K)), 1).reshape(2 * Fp, K).contiguous()
    g3 = 1 + 0.1 * grand((Fu,), 14, dtype=torch.float32)
    w2 = grand((dim, Fu), 15, Fu ** -0.5, dtype=torch.float32)
    w2f = torch.zeros((dim, Fp), device="cuda"); w2f[:, :Fu] = w2 * g3
    w2f = w2f.to(bf).contiguous()
    cvec = w2f.float().sum(1).contiguous()
    x = grand((M_, dim), 16, dtype=torch.float32)
    h = torch.empty((M_, Fp), device="cuda", dtype=bf)
    stats = torch.full((M_, Fp // 32, 2), float("nan"), device="cuda")
    xd = x.clone()
    o.linear(a, w1, h, epilogue=o.EPI_GEGLU, row_stats=stats)
    href = (a.float() @ wg.float().t()) * F.gelu(a.float() @ wx.float().t())
    ok, msg = close(h[:, :Fu], href, 2e-2, 1e-2)
    assert ok, "GEGLU: " + msg
    assert float(h[:, Fu:].abs().max()) == 0.
    hq = h.float().view(M_, Fp // 32, 32)                                                      # statistics of the bf16-rounded outputs, chunk by chunk
    assert torch.allclose(stats[..., 0], hq.sum(-1), atol=1e-3, rtol=1e-5) and torch.allclose(stats[..., 1], (hq * hq).sum(-1), atol=1e-3, rtol=1e-5)
    ok, msg = close(stats[..., 0].sum(-1), href.sum(-1), 5e-3 * float(href.sum(-1).abs().max()), 1e-2)
    assert ok, "row sums: " + msg
    o.linear(h, w2f, xd, epilogue=o.EPI_LNFOLD_RESIDUAL, bias=cvec, resid=xd, row_stats=stats, ln_width=Fu)
    ref = x + F.layer_norm(href, (Fu,)) @ w2f[:, :Fu].float().t()          # w2f = bf16(W2 * gamma): the fold's own operand
    ok, msg = close(xd, ref, 4e-2, 1e-2)
    assert ok, "FF2: " + msg


@pytest.mark.parametrize("M_", [32768, 16384 + 128 * 3], ids=["32768", "16768"])
def test_gemm_generate_shape_wo_residual(M_):
    """attention to_out: x += a Wo^T, 32768 x 512 x 512, in place through the TMA reduction (tc_gemm_kernel<256, 2>)."""
    o = ops()
    a, w = grand((M_, 512), 21), grand((512, 512), 22, 512 ** -0.5)
    x = grand((M_, 512), 23, dtype=torch.float32)
    xd = x.clone()
    o.linear(a, w, xd, epilogue=o.EPI_RESIDUAL, resid=xd)
    ok, msg = close(xd, x + a.float() @ w.float().t(), 5e-4, 1e-3)
    assert ok, msg


@pytest.mark.parametrize("rows", [64 * 229, 64 * 47 + 5], ids=["14656", "3013_ragged"])
def test_gemm_generate_shape_logits(rows):
    """to_logits on the masked rows of a step: rows x 65536 x 512, fp32 out through the TMA-store tiles (tc_gemm_kernel<256, 3>)."""
    o = ops()
    a, w = grand((rows, 512), 31), grand((65536, 512), 32, 512 ** -0.5)
    out = torch.empty((rows + 3, 65536), device="cuda")
    out[rows:] = 7.0
    o.linear(a, w, out[:rows])
    worst = 0.
    for r0 in range(0, rows, 4096):
        r1 = min(r0 + 4096, rows)
        ref = a[r0:r1].float() @ w.float().t()
        worst = max(worst, float((out[r0:r1] - ref).abs().max()))
    assert worst < 3e-4, worst
    assert bool((out[rows:] == 7.0).all()), "rows past M were written"


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def test_gemm_generate_shape_conv3x3_glu():
    """VAE decoder GLU res-block conv: 3x3, 2048 -> 4096 on 16 x 16 maps, batch 64, K = 18432: implicit GEMM (4-D tensor-map A operand)
    with the register epilogue in 128-column tiles, tc_gemm_kernel<128, 0>."""
    o = ops()
    B, H, W, C = 64, 16, 16, 2048
    x = grand((B, C, H, W), 41)
    w = grand((2 * C, C, 3, 3), 42, (9 * C) ** -0.5)
    bias = grand((2 * C,), 43, dtype=torch.float32)
    idx = torch.arange(C, device="cuda").view(-1, 32)
    order = torch.cat((idx, idx + C), 1).reshape(-1)
    wp = w.permute(0, 2, 3, 1).reshape(2 * C, -1)[order].contiguous()
    out = torch.empty((B * H * W, C), device="cuda", dtype=bf)
    o.conv2d(_nhwc(x).view(-1, C), wp, out, B, H, W, C, 2 * C, 1, epilogue=o.EPI_GLU, bias=bias[order].contiguous())
    ref = _nhwc(F.glu(F.conv2d(x.float(), w.float(), bias, padding=1), dim=1)).reshape(-1, C)
    ok, msg = close(out, ref, 2e-2, 1e-2)
    assert ok, msg


def test_gemm_generate_shape_conv4x4_s2():
    """VAE encoder stage: 4x4 stride-2 conv 256 -> 256 from 256 x 256 maps (four parity tensor maps, K = 4096)."""
    o = ops()
    B, H, W, Cin, Cout = 4, 256, 256, 256, 256
    x = grand((B, Cin, H, W), 51)
    w = grand((Cout, Cin, 4, 4), 52, (16 * Cin) ** -0.5)
    bias = grand((Cout,), 53, dtype=torch.float32)
    out = torch.empty((B * (H // 2) * (W // 2), Cout), device="cuda", dtype=bf)
    o.conv2d(_nhwc(x).view(-1, Cin), w.permute(0, 2, 3, 1).reshape(Cout, -1).contiguous(), out, B, H, W, Cin, Cout, 2, bias=bias, act=1)
    ref = _nhwc(F.leaky_relu(F.conv2d(x.float(), w.float(), bias, stride=2, padding=1), 0.1)).reshape(-1, Cout)
    ok, msg = close(out, ref, 2e-2, 1e-2)
    assert ok, msg


def _pack_convt(w):
    from muse_maskgit_pytorch_b200.vqgan_vae import CT_R
    packs = []
    for py in range(2):
        for px in range(2):
            packs.append(torch.cat([w[:, :, CT_R[py][a], CT_R[px][b]].t() for a in range(2) for b in range(2)], dim=1))
    return torch.stack(packs).contiguous()


def test_gemm_generate_shape_convt_and_rgb():
    """VAE decoder tail: ConvTranspose 1024 -> 512 from 32 x 32 (parity scatter), and the last ConvTranspose 256 -> 256 from 128 x 128 fused
    with LeakyReLU and the 1x1 conv to RGB (fp32 NCHW out)."""
    o = ops()
    B, H, W, Cin, Cout = 8, 32, 32, 1024, 512
    x = grand((B, Cin, H, W), 61)
    w = grand((Cin, Cout, 4, 4), 62, (4 * Cin) ** -0.5)
    bias = grand((Cout,), 63, dtype=torch.float32)
    out = torch.empty((B * 4 * H * W, Cout), device="cuda", dtype=bf)
    o.conv_transpose2d(_nhwc(x).view(-1, Cin), _pack_convt(w), out, B, H, W, Cin, Cout, bias=bias)
    ref = _nhwc(F.leaky_relu(F.conv_transpose2d(x.float(), w.float(), bias, stride=2, padding=1), 0.1)).reshape(-1, Cout)
    ok, msg = close(out, ref, 2e-2, 1e-2)
    assert ok, "convT: " + msg
    B, H, W, Cin, Cout = 8, 128, 128, 256, 256
    x = grand((B, Cin, H, W), 64)
    w = grand((Cin, Cout, 4, 4), 65, (4 * Cin) ** -0.5)
    bias, rw, rb = grand((Cout,), 66, dtype=torch.float32), grand((3, Cout), 67, Cout ** -0.5, dtype=torch.float32), grand((3,), 68, dtype=torch.float32)
    img = torch.empty((B, 3, 2 * H, 2 * W), device="cuda")
    o.conv_transpose2d(_nhwc(x).view(-1, Cin), _pack_convt(w), img, B, H, W, Cin, Cout, bias=bias, rgb_w=rw, rgb_b=rb)
    ref = F.conv2d(F.leaky_relu(F.conv_transpose2d(x.float(), w.float(), bias, stride=2, padding=1), 0.1), rw[:, :, None, None], rb)
    ok, msg = close(img, ref, 1e-3, 1e-3)
    assert ok, "convT+RGB: " + msg


def test_attention_c4_sizes():
    """Self-attention with 1025 keys and masked cross-attention with 289 keys at the batch the super-res bench uses (64 sequences x 8 heads)."""
    o = ops()
    B, heads, n = 16, 8, 1024
    for Tk, masked, seed in ((n + 1, False, 71), (289, True, 72)):
        ta = (Tk + 7) // 8 * 8
        q = F.normalize(grand((B * heads, n, 64), seed, dtype=torch.float32), dim=-1).to(bf)
        k = torch.zeros((B * heads, ta, 64), device="cuda", dtype=bf); v = torch.zeros_like(k)
        k[:, :Tk] = F.normalize(grand((B * heads, Tk, 64), seed + 10, dtype=torch.float32), dim=-1).to(bf)
        v[:, :Tk] = grand((B * heads, Tk, 64), seed + 20)
        mask = None
        if masked:
            mask = (torch.rand((B, Tk - 1), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed)) > 0.3)
            mask[1] = False                                                    # one sequence with every context key masked
            mask = mask.to(torch.uint8).contiguous()
        out = torch.empty((B * n, heads * 64), device="cuda", dtype=bf)
        o.attention(q, k, v, out, B, heads, Tk, key_mask=mask, logit_bound=1.02)
        s = 8.0 * torch.einsum("bid,bjd->bij", q.float(), k[:, :Tk].float())
        if masked:
            full = torch.cat((torch.ones((B, 1), device="cuda", dtype=torch.bool), mask.bool()), 1)
            s = s.view(B, heads, n, Tk).masked_fill(~full[:, None, None, :], -torch.finfo(torch.float32).max).view(B * heads, n, Tk)
        ref = torch.einsum("bij,bjd->bid", s.softmax(-1), v[:, :Tk].float()).view(B, heads, n, 64).permute(0, 2, 1, 3).reshape(B * n, heads * 64)
        ok, msg = close(out, ref, 2e-2, 2e-2)
        assert ok, f"Tk={Tk}: " + msg

"""GPU: precision="fp8" — the quantising LayerNorm, the e4m3 wgmma GEMM instantiations and the fp8 transformer end to end.

  mmg_layernorm_fp8: bytes and row scales equal the CPU oracle (tests/fp8_oracle.py) applied to mmg_layernorm's fp32 output, bit for bit,
  with and without the add / x_out / add_from fold;
  mmg_linear_fp8: <256, QKV> (self QKV), <128, QKV> (cross q), <256, GEGLU> (FF1) against fp64 on the dequantised operands, through the
  epilogue's math, at C3 shapes and smaller / ragged M, in both tile orders; unsupported shapes raise.  Which instantiation each case
  reached (tests/gemm_oracle.py's fp8_plan) is asserted from torch.profiler captures taken in a child process
  (test_linear_fp8_cases_reached_their_kernels runs those cases again with MMG_FP8_PROFILE=1), as in tests/test_gpu_gemm.py;
  C3 full-config teacher-forced flip rate against the fp32 oracle; generate() determinism, eager vs CUDA graph; inpaint; MaskGit.forward
  against the fp32 loss; the precision="fp8" rejections.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import fp8_oracle as Q
from tests import gemm_oracle as G
from tests.test_gpu_row_kernels import kernels_of, assert_ran

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
E4 = torch.float8_e4m3fn
PROFILE = os.environ.get("MMG_FP8_PROFILE") == "1"


def M():
    import muse_maskgit_pytorch_b200 as m
    from muse_maskgit_pytorch_b200 import t5
    for d in (128, 512):
        t5.T5_CONFIGS[f"synth-{d}"] = {"d_model": d}
    return m


def ops():
    from muse_maskgit_pytorch_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ quantising LayerNorm
@pytest.mark.parametrize("fold", [False, True], ids=["plain", "add_x_out"])
@pytest.mark.parametrize("rows,width", [(1000, 512), (77, 128), (33, 1024)])
def test_layernorm_fp8_matches_oracle_on_fp32_mode(rows, width, fold):
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(rows + width)
    x = torch.randn((rows, width), device="cuda", generator=g) * 3 + 0.5
    x[5] = 0.                                                      # LN(0) = 0: amax == 0, scale 0, zero bytes
    x[7, 11] = 300.                                                # one large column
    gamma = torch.rand((width,), device="cuda", generator=g) + 0.5
    kw = {}
    if fold:
        kw = dict(add=torch.randn((width,), device="cuda", generator=g), add_from=rows // 2)
    x32, x8 = x.clone(), x.clone()
    y32 = torch.empty((rows, width), device="cuda")
    o.layernorm(x32, gamma, y32, x_out=x32 if fold else None, **kw)
    y8 = torch.empty((rows, width), device="cuda", dtype=E4)
    sc = torch.full((rows,), -1., device="cuda")
    o.layernorm_fp8(x8, gamma, y8, sc, x_out=x8 if fold else None, **kw)
    qb, qs = Q.quantize_rows(y32.cpu().numpy())
    got = y8.view(torch.uint8).cpu().numpy()
    assert np.array_equal(got, qb), int((got != qb).sum())
    assert np.array_equal(sc.cpu().numpy(), qs)
    assert float(sc[5]) == 0. and not got[5].any()
    assert torch.equal(x8, x32)                                    # the x_out fold writes the same (x + add) rows
    if fold:
        assert not torch.equal(x8[rows // 2:], x[rows // 2:]) and torch.equal(x8[:rows // 2], x[:rows // 2])


def test_layernorm_fp8_pads_columns_past_width():
    o = ops()
    x = torch.randn((40, 500), device="cuda")
    y = torch.full((40, 512), 1., device="cuda").to(E4)
    sc = torch.empty((40,), device="cuda")
    o.layernorm_fp8(x, torch.ones((500,), device="cuda"), y, sc)
    y32 = torch.empty((40, 500), device="cuda")
    o.layernorm(x, torch.ones((500,), device="cuda"), y32)
    qb, qs = Q.quantize_rows(y32.cpu().numpy())
    got = y.view(torch.uint8).cpu().numpy()
    assert np.array_equal(got[:, :500], qb) and not got[:, 500:].any() and np.array_equal(sc.cpu().numpy(), qs)


# ------------------------------------------------------------------------------------------------ e4m3 GEMM
@pytest.fixture(scope="module", autouse=True)
def _warm_up():
    if PROFILE and torch.cuda.is_available():
        kernels_of(lambda: torch.ones(8, device="cuda").sum())


def run_planned(fn, kind, M, N, K, bn, order):
    """fn(), one mmg_linear_fp8 call the case builds for tile width bn and tile order order ('n' or 'm' fastest), both checked against
    gemm_oracle.fp8_plan; in the profiling process also that exactly the planned instantiation ran"""
    pbn, mode, nf = G.fp8_plan(kind, M, N, K, torch.cuda.get_device_properties(0).multi_processor_count)
    assert (pbn, nf) == (bn, int(order == "n")), f"built for <{bn}> {order}-fast, the plan gives <{pbn}> n_fast = {nf}"
    if PROFILE:
        _, names = kernels_of(fn)
        assert_ran(names, G.TC(bn, mode, G.E4M3))
    else:
        fn()


def fp8_operands(Mr, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn((Mr, K), device="cuda", generator=g) * 120).clamp(-448, 448).to(E4)
    w = (torch.randn((N, K), device="cuda", generator=g) * 120).clamp(-448, 448).to(E4)
    sa = torch.rand((Mr,), device="cuda", generator=g) * 2e-3 + 1e-4
    sw = torch.rand((N,), device="cuda", generator=g) * 2e-3 + 1e-4
    ad, wd = a.double() * sa.double()[:, None], w.double() * sw.double()[:, None]
    return a, w, sa, sw, ad @ wd.t(), ad.abs() @ wd.abs().t()       # fp64 product of the dequantised operands, and sum |a w|


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


# (256, 'n'): 6 column tiles; (256, 'm'): 18 column tiles; cross-small: 256 rows, one 128-column tile (the bf16 product runs <64, REGS>)
@pytest.mark.parametrize("Mr,K,tokens,heads,cross,bn,order", [(32768, 512, 256, 8, False, 256, "n"), (384, 256, 32, 4, False, 128, "n"),
                                                              (16384, 512, 256, 8, True, 128, "n"), (256, 128, 64, 2, True, 128, "m"),
                                                              (2048, 256, 64, 24, False, 256, "m")],
                         ids=["self-C3", "self-small", "cross-C3", "cross-small", "self-mfast"])
def test_linear_fp8_qkv_vs_fp64(Mr, K, tokens, heads, cross, bn, order):
    o = ops()
    inner = heads * 64
    N = inner if cross else 3 * inner
    a, w, sa, sw, ref, S = fp8_operands(Mr, N, K, Mr + N)
    bsz = Mr // tokens
    g = torch.Generator(device="cuda").manual_seed(3)
    qs, ks = torch.rand((64,), device="cuda", generator=g) + 0.5, torch.rand((64,), device="cuda", generator=g) + 0.5
    q = torch.zeros((bsz * heads, tokens, 64), device="cuda", dtype=torch.bfloat16)
    if cross:
        epi = o.qkv_epilogue(torch.bfloat16, heads, tokens, q=q, q_scale=qs)
    else:
        tka = tokens + 8
        k = torch.zeros((bsz * heads, tka, 64), device="cuda", dtype=torch.bfloat16)
        v = torch.zeros_like(k)
        nk = torch.randn((heads, 64), device="cuda", generator=g).bfloat16()
        nv = torch.randn((heads, 64), device="cuda", generator=g).bfloat16()
        epi = o.qkv_epilogue(torch.bfloat16, heads, tokens, q=q, k=k, v=v, q_scale=qs, k_scale=ks, key_off=1, null_k=nk, null_v=nv)
    run_planned(lambda: o.linear_fp8(a, sa, w, sw, None, epilogue=o.EPI_QKV, epi=epi), G.QKV, Mr, N, K, bn, order)
    # [bsz, tokens, part, heads, 64] fp64 reference, heads laid out [q heads | k heads | v heads] along N
    R = ref.view(bsz, tokens, -1, heads, 64)
    Sm = S.view(bsz, tokens, -1, heads, 64)
    to_bh = lambda t: t.permute(0, 2, 1, 3).reshape(bsz * heads, tokens, 64)
    worst = 0.
    for part, out, scale in ((0, q, qs),) + (() if cross else ((1, k[:, 1:tokens + 1], ks), (2, v[:, 1:tokens + 1], None))):
        r, s = R[:, :, part], Sm[:, :, part]
        if scale is not None:                                          # l2-normalised, then scaled
            nrm = r.norm(dim=-1, keepdim=True)
            ref_o = r / nrm * scale.double()
            tol = 2e-3 * s.amax(dim=-1, keepdim=True) / nrm * scale.double().abs() + 2.0 ** -8 * ref_o.abs() + 1e-6
        else:
            ref_o, tol = r, 1e-3 * s + 2.0 ** -8 * r.abs() + 1e-6
        err = (out.double() - to_bh(ref_o)).abs()
        assert (err <= to_bh(tol)).all(), (part, float((err - to_bh(tol)).max()))
        worst = max(worst, float((err / to_bh(s if scale is None else s.amax(dim=-1, keepdim=True).expand_as(s))).max()))
    if not cross:
        assert torch.equal(k[:, 0], nk.repeat(bsz, 1)) and torch.equal(v[:, 0], nv.repeat(bsz, 1))   # null key / value rows
    print(f"QKV fp8 M={Mr} N={N} K={K}: largest |err| / sum|a w| = {worst:.2e}")


@pytest.mark.parametrize("Mr,N,K,order", [(32768, 2816, 512, "n"), (1000, 2816, 512, "n"), (129, 2816, 256, "n"), (1000, 4352, 512, "m")],
                         ids=["C3", "ragged-1000", "ragged-129", "mfast-17-tiles"])
def test_linear_fp8_geglu_vs_fp64(Mr, N, K, order):
    o = ops()
    a, w, sa, sw, ref, S = fp8_operands(Mr, N, K, Mr)
    h = torch.empty((Mr, N // 2), device="cuda", dtype=torch.bfloat16)
    stats = torch.full((Mr, N // 64, 2), float("nan"), device="cuda")
    run_planned(lambda: o.linear_fp8(a, sa, w, sw, h, epilogue=o.EPI_GEGLU, row_stats=stats), G.GEGLU, Mr, N, K, 256, order)
    R, Sv = ref.view(Mr, N // 64, 2, 32), S.view(Mr, N // 64, 2, 32)
    xr, gr, sx, sg = R[:, :, 0], R[:, :, 1], Sv[:, :, 0], Sv[:, :, 1]
    ref_o = (gr * gelu64(xr)).reshape(Mr, N // 2)
    tol = (1e-3 * (1.13 * gr.abs() * sx + (xr.abs() + 1e-3 * sx) * sg)).reshape(Mr, N // 2) + 2.0 ** -8 * ref_o.abs() + 1e-5
    err = (h.double() - ref_o).abs()
    assert (err <= tol).all(), float((err - tol).max())
    worst = float((err / (gr.abs() * sx + xr.abs() * sg).reshape(Mr, N // 2).clamp(min=1e-30)).max())
    # row_stats: each 64-column chunk's (sum, sum of squares) of its 32 bf16 outputs as written, i.e. of the dequantised values
    hv = h.double().view(Mr, N // 64, 32)
    assert torch.isfinite(stats).all()
    assert torch.allclose(stats[..., 0].double(), hv.sum(-1), rtol=1e-5, atol=1e-5 * float(hv.abs().sum(-1).max()))
    assert torch.allclose(stats[..., 1].double(), (hv * hv).sum(-1), rtol=1e-5, atol=1e-6)
    print(f"GEGLU fp8 M={Mr} K={K}: largest |err| / (|g| sum|a w|_x + |x| sum|a w|_g) = {worst:.2e}")


def test_linear_fp8_rejects_unsupported_shapes():
    from muse_maskgit_pytorch_b200 import _lib
    o = ops()
    a, w, sa, sw, _, _ = fp8_operands(256, 512, 192, 1)           # K % 128 != 0
    h = torch.empty((256, 256), device="cuda", dtype=torch.bfloat16)
    with pytest.raises(_lib.MMGError, match="K % 128"):
        o.linear_fp8(a, sa, w, sw, h, epilogue=o.EPI_GEGLU)
    a, w, sa, sw, _, _ = fp8_operands(256, 384, 128, 2)           # GEGLU N % 256 != 0
    with pytest.raises(_lib.MMGError, match="N % 256"):
        o.linear_fp8(a, sa, w, sw, torch.empty((256, 192), device="cuda", dtype=torch.bfloat16), epilogue=o.EPI_GEGLU)
    a, w, sa, sw, _, _ = fp8_operands(200, 512, 128, 3)           # QKV M % 128 != 0
    q = torch.zeros((200 // 40 * 8, 40, 64), device="cuda", dtype=torch.bfloat16)
    epi = o.qkv_epilogue(torch.bfloat16, 8, 40, q=q, q_scale=torch.ones((64,), device="cuda"))
    with pytest.raises(_lib.MMGError, match="QKV"):
        o.linear_fp8(a, sa, w, sw, None, epilogue=o.EPI_QKV, epi=epi)
    a, w, sa, sw, _, _ = fp8_operands(256, 256, 128, 4)           # epilogues other than QKV / GEGLU
    with pytest.raises(_lib.MMGError, match="QKV or GEGLU"):
        o.linear_fp8(a, sa, w, sw, torch.empty((256, 256), device="cuda", dtype=torch.bfloat16), epilogue=o.EPI_STORE)


def test_linear_fp8_cases_reached_their_kernels():
    """the e4m3 product cases of this file again, in a fresh process, each under torch.profiler: profiler sessions early in a whole-suite
    process make later captures come back empty"""
    if PROFILE:
        pytest.skip("this is the profiling process")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-rP", "-m", "gpu", "-k", "linear_fp8 and vs_fp64",
                        "--no-header", "-p", "no:cacheprovider"], cwd=root, env=dict(os.environ, MMG_FP8_PROFILE="1"), capture_output=True,
                       text=True, timeout=600)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ end to end
PRODUCTS = {"self QKV": ("sa", "wqkv"), "cross q": ("ca", "wq"), "FF1": ("ff", "w1")}


def _c3_fp8(monkeypatch, keep=tuple(PRODUCTS)):
    """The C3 teacher-forced harness of test_gpu_full_config on an fp8 transformer whose products outside `keep` run in bf16 again"""
    from tests import test_gpu_full_config as FC
    m = M()
    bf_tr, _ = FC.base_transformer()
    torch.manual_seed(0)
    tr = m.MaskGitTransformer(t5_name="synth-512", precision="fp8", **FC.TR_BASE)
    tr.load_state_dict(bf_tr.state_dict())
    tr = tr.cuda()
    build = tr._build_pack

    def build_mixed():                                                # every (re)pack puts the bf16 weights back outside `keep`
        P, Pb = build(), bf_tr._packed()
        for name, (part, key) in PRODUCTS.items():
            if name not in keep:
                for lay, lb in zip(P["layers"], Pb["layers"]):
                    del lay[part][key + "_8"]
                    lay[part][key] = lb[part][key]
        return P
    monkeypatch.setattr(tr, "_build_pack", build_mixed)
    vae_cls = m.VQGanVAE                                              # the token loop does not touch the VAE: build it in bf16
    monkeypatch.setattr(m, "VQGanVAE", lambda *a, precision=None, **k: vae_cls(*a, precision="bf16" if precision == "fp8" else precision, **k))
    return FC._c3_teacher_forced(tr)


@pytest.mark.xfail(strict=True, reason="measured on an H100: 660 of 5782 teacher-forced tokens (11.4 %) flip at fp8, above the 8 % bound "
                                       "of bf16; test_c3_teacher_forced_flips_per_fp8_product reports the share of each product")
def test_c3_teacher_forced_flip_rate_fp8(monkeypatch):
    flips, total, per_step, worst_score = _c3_fp8(monkeypatch)
    rate = flips / total
    print(f"C3 full-config teacher-forced flip rate, fp8 QKV / cross q / FF1: {flips}/{total} = {rate:.4f} (per step {per_step}); "
          f"max |score diff| on agreeing tokens {worst_score:.2e}")
    assert rate < 0.08


def test_c3_teacher_forced_flips_per_fp8_product(monkeypatch):
    """one product at a time on e4m3, the other two in bf16: the flips each product brings on its own"""
    for name in PRODUCTS:
        flips, total, per_step, _ = _c3_fp8(monkeypatch, keep=(name,))
        print(f"C3 teacher-forced, only {name} on fp8: {flips}/{total} = {flips / total:.4f} (per step {per_step})")
        assert 0 <= flips < total


def small_maskgit(precision, seed=0):
    m = M()
    torch.manual_seed(seed)
    tr = m.MaskGitTransformer(num_tokens=512, dim=128, seq_len=256, depth=2, heads=2, t5_name="synth-128", precision=precision)
    vae = m.VQGanVAE(dim=16, layers=2, codebook_size=512)
    te = torch.randn((4, 8, 128), generator=torch.Generator().manual_seed(5)).cuda()
    te[1, 5:] = 0.
    tr.encode_text = lambda texts: te[:len(texts)]
    return m.MaskGit(image_size=64, transformer=tr, vae=vae).cuda()


def test_generate_fp8_deterministic_eager_and_graph():
    mg = small_maskgit("fp8")
    mg.sampler_seed = 17
    runs = []
    for graph in (False, False, True, True):
        mg.use_cuda_graph = graph
        torch.manual_seed(1)
        runs.append(mg.generate(["a"] * 3, timesteps=8, return_ids=True))
    for img, ids in runs[1:]:
        assert torch.equal(ids, runs[0][1]) and torch.equal(img, runs[0][0])
    mg32 = small_maskgit("bf16")
    mg32.sampler_seed = 17
    torch.manual_seed(1)
    _, ids_bf = mg32.generate(["a"] * 3, timesteps=8, return_ids=True)
    print(f"fp8 vs bf16 generate() ids agree on {float((ids_bf == runs[0][1]).float().mean()):.3f} of the positions")


def test_inpaint_and_forward_fp8():
    mg8, mg32 = small_maskgit("fp8"), small_maskgit("fp32")
    mg8.sampler_seed = 3
    img = torch.rand((2, 3, 64, 64), generator=torch.Generator().manual_seed(2)).cuda()
    mask = torch.zeros((2, 16, 16), dtype=torch.bool)
    mask[:, 4:12, 4:12] = True
    out, ids = mg8.inpaint(["a"] * 2, img, mask, timesteps=6, return_ids=True)
    enc = mg8.vae.encode_ids(img).reshape(2, -1)
    keep = ~mask.reshape(2, -1).cuda()
    assert torch.equal(ids.reshape(2, -1)[keep], enc[keep]) and torch.isfinite(out).all()
    ids_in = torch.randint(0, 512, (4, 256), generator=torch.Generator().manual_seed(9)).cuda()
    for s in range(3):
        torch.manual_seed(s)
        l8 = float(mg8(ids_in, texts=["a"] * 4))
        torch.manual_seed(s)
        l32 = float(mg32(ids_in, texts=["a"] * 4))
        print(f"MaskGit.forward seed {s}: fp8 {l8:.6f} fp32 {l32:.6f} rel {abs(l8 - l32) / abs(l32):.2e}")
        assert abs(l8 - l32) <= 0.01 * abs(l32)


def test_fp8_rejections():
    m = M()
    with pytest.raises(ValueError, match="dim % 128"):
        m.MaskGitTransformer(num_tokens=512, dim=192, seq_len=256, depth=1, heads=3, t5_name="synth-128", precision="fp8")
    with pytest.raises(ValueError, match="fp8"):
        m.VQGanVAE(dim=16, layers=2, codebook_size=512, precision="fp8")
    from types import SimpleNamespace
    from muse_maskgit_pytorch_b200 import t5, _lib
    with pytest.raises(_lib.MMGError, match="precision"):
        t5.T5Encoder(SimpleNamespace(d_model=64, d_kv=64, d_ff=128, num_layers=1, num_heads=1), precision="fp8")
    mg = small_maskgit("fp8")
    mg.use_native_step = True
    with pytest.raises(ValueError, match="use_native_step"):
        mg.generate(["a"] * 2, timesteps=4)

"""GPU: VQGanVAE precision="fp8" — the per-image quantiser, the e4m3 convolutions and the fp8 VAE end to end.

  mmg_quantize_e4m3_images: bytes and scales equal tests/vae_fp8_oracle.py bit for bit (an all-zero image, ragged B);
  mmg_conv2d_fp8 / mmg_conv_transpose2d_fp8: every instantiation tc_gemm_kernel<BN, 0, __nv_fp8_e4m3> against fp64 on the dequantised
  operands with the bound of tests/vae_fp8_oracle.py, at the real K of the benchmark VAE (dim = 256: 9 x 2048) and at the edges (1x1,
  3x3, 4x4 s2, each conv-transpose parity, CONVT_RGB at N = 64 / 128 / 256, GLU, RESIDUAL, LeakyReLU, multi-image tiles); guard rows
  after the output survive; a torch.profiler capture shows which kernel ran and the CUDA-core counter does not move;
  rejections (Cin % 128, misalignment, tile geometry); the dim = 256 VAE at 512^2 against bf16 (encode_ids) and fp32 (decode_from_ids);
  MaskGit.generate over an fp8 VAE; bitwise determinism.
"""
import numpy as np
import pytest
import torch

from tests import gemm_oracle as G
from tests import vae_fp8_oracle as V
from tests.test_gpu_row_kernels import CAPTURE_RETAKES, assert_ran

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
E4 = torch.float8_e4m3fn
GUARD = 12345.0
RATIOS = {}


def ops():
    from muse_maskgit_pytorch_b200 import ops as o
    return o


def L():
    from muse_maskgit_pytorch_b200 import _lib
    return _lib


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def kernels_of(fn, repeats=8):
    """the libmmg kernels fn() launches, from a torch.profiler capture of `repeats` calls between two runs of small torch kernels.  CUPTI
    now and then drops the activity records of a capture, all or some of them (tests/test_gpu_row_kernels.py); single short launches at
    the start of a capture came back empty every time, so the capture neither starts nor ends on the call, repeats it, and is taken again,
    up to five times, when it saw no libmmg kernel."""
    import time
    from torch.profiler import profile, ProfilerActivity
    names = []
    for attempt in range(6):
        if attempt:
            time.sleep(0.05 * attempt)
            CAPTURE_RETAKES[0] += 1
        torch.cuda.synchronize()
        t = torch.zeros(1024, device="cuda")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(16):
                t.add_(1)
            torch.cuda.synchronize()
            for _ in range(repeats):
                fn()
            torch.cuda.synchronize()
            for _ in range(16):
                t.add_(1)
            torch.cuda.synchronize()
        names = sorted({e.key for e in prof.key_averages() if e.self_device_time_total > 0 and "mmg::" in e.key})
        if names:
            break
    return names


def want_bn(m_tiles, N, rgb):
    bn = G.pick_bn(m_tiles, N, G.CONVT_RGB if rgb else G.STORE, sms())
    return 128 if bn == 256 and not rgb else bn


# ------------------------------------------------------------------------------------------------ quantiser
@pytest.mark.parametrize("B,hw,C", [(3, 7 * 9, 128), (5, 16, 256), (2, 64 * 64, 256), (1, 32 * 32, 2048)])
def test_quantiser_bits_and_scales_match_oracle(B, hw, C):
    g = torch.Generator(device="cuda").manual_seed(B * hw + C)
    x = (torch.randn((B * hw, C), device="cuda", generator=g) * torch.arange(1, B + 1, device="cuda").repeat_interleave(hw)[:, None]).bfloat16()
    if B >= 3:
        x[hw:2 * hw] = 0                                             # an all-zero image
    x[0, 1] = -300.
    q, s = ops().quantize_e4m3_images(x, B)
    bits, sc = V.quantize_images(x, B)
    got = q.view(torch.uint8).cpu().numpy()
    assert np.array_equal(got, bits), int((got != bits).sum())
    assert np.array_equal(s.cpu().numpy(), sc)
    if B >= 3:
        assert float(s[1]) == 0. and not got[hw:2 * hw].any()
    q2, s2 = ops().quantize_e4m3_images(x, B)
    assert torch.equal(q2.view(torch.uint8), q.view(torch.uint8)) and torch.equal(s2, s)


# ------------------------------------------------------------------------------------------------ convolutions against fp64
def _operands(tag, B, H, W, Cin, wrows, K):
    x = V.probe_image(tag, B, H, W, Cin).cuda().bfloat16()
    q, s = ops().quantize_e4m3_images(x.reshape(-1, Cin), B)
    w = V.probe_weight(tag, wrows, K) * 0.05
    from muse_maskgit_pytorch_b200.muse_maskgit import quantize_rows_e4m3
    wq, ws = quantize_rows_e4m3(w.cuda())
    xd = (q.float().reshape(B, -1) * s[:, None]).reshape(B, H, W, Cin)
    wd = wq.float() * ws[:, None]
    return q, s, wq, ws, xd, wd


# (kind, B, H, W, Cin, Cout, epilogue): C5 = the dim = 256 VAE at 512^2 (fmap 32^2, widths 256 .. 2048), C3 = 256^2 (fmap 16^2)
CONV_CASES = {
    "c5_res3x3_K18432": (1, 1, 32, 32, 2048, 2048, G.STORE),
    "c5_glu3x3_K18432": (1, 1, 32, 32, 2048, 4096, G.GLU),
    "c5_res1x1_residual": (0, 2, 32, 32, 2048, 2048, G.RESIDUAL),
    "c5_down4x4s2_leaky": (2, 1, 64, 64, 1024, 2048, G.STORE),
    "c3_glu3x3": (1, 2, 16, 16, 2048, 4096, G.GLU),
    "c3_down4x4s2_first": (2, 1, 128, 128, 256, 256, G.STORE),
    "edge_1x1_bn64": (0, 3, 8, 8, 128, 64, G.STORE),
    "edge_3x3_multi_image_tile": (1, 5, 4, 4, 128, 128, G.STORE),
    "edge_4x4s2_multi_image": (2, 3, 8, 8, 256, 128, G.STORE),
    "edge_glu_small": (1, 3, 4, 8, 128, 256, G.GLU),
    "edge_residual_ragged": (0, 3, 8, 16, 384, 192, G.RESIDUAL),
}


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv2d_fp8_against_fp64(case):
    kind, B, H, W, Cin, Cout, epi = CONV_CASES[case]
    o = ops()
    taps = (1, 9, 16)[kind]
    Ho, Wo = G.conv_out_hw(kind, H, W)
    M, K = B * Ho * Wo, taps * Cin
    q, s, wq, ws, xd, wd = _operands(case, B, H, W, Cin, Cout, K)
    p = {"bias": G.rnd(case + ".b", (Cout,), 0.5).cuda()}
    kw = dict(bias=p["bias"])
    if epi == G.RESIDUAL:
        p["resid"] = G.bf(G.rnd(case + ".r", (M, Cout), 1.0)).cuda()
        kw.update(epilogue=o.EPI_RESIDUAL, resid=p["resid"].bfloat16())
    elif epi == G.GLU:
        kw.update(epilogue=o.EPI_GLU)
    if kind == 2:
        p["act"] = 1
        kw.update(act=1)
    width = Cout // 2 if epi == G.GLU else Cout
    buf = torch.full((M + 64, width), GUARD, device="cuda", dtype=torch.bfloat16)
    out = buf[:M]
    s0 = L().simt_launch_count()
    names = kernels_of(lambda: o.conv2d_fp8(q, s, wq, ws, out, B, H, W, Cin, Cout, kind, **kw))
    assert L().simt_launch_count() == s0
    g = G.tile_geometry(Ho, Wo)
    bn = want_bn(g[3] * g[4] * ((B + g[2] - 1) // g[2]), Cout, False)
    assert_ran(names, f"tc_gemm_kernel<{bn}, 0, __nv_fp8_e4m3>")
    assert bool((buf[M:] == GUARD).all())
    ref, S, A = V.conv_ref(xd, wd, kind, epi, p)
    r = G.worst_ratio(out.float(), ref, V.tolerance(ref, S, A, True))
    RATIOS[case] = r
    print(f"{case}: K = {K}, worst |err| / tol = {r:.3g}")
    assert r <= 1.0


@pytest.mark.parametrize("case", ["res3x3_K18432", "down4x4s2_K16384", "small3x3_K1152"])
def test_promoted_accumulation_against_fp32_bound(case):
    """fp32 outputs, no epilogue terms: |err| against the fp32-accumulation bound alone (tests/gemm_oracle.py's coef(K) s, the bound the
    bf16 kernel meets) and against the full e4m3 bound.  Before promotion these were 4.3, 6.3 and 131 times coef(K) s."""
    kind, B, H, W, Cin, Cout = {"res3x3_K18432": (1, 1, 32, 32, 2048, 2048), "down4x4s2_K16384": (2, 1, 64, 64, 1024, 2048),
                                "small3x3_K1152": (1, 2, 8, 8, 128, 128)}[case]
    taps = (1, 9, 16)[kind]
    Ho, Wo = G.conv_out_hw(kind, H, W)
    q, s, wq, ws, xd, wd = _operands(case, B, H, W, Cin, Cout, taps * Cin)
    out = torch.empty((B * Ho * Wo, Cout), device="cuda")
    ops().conv2d_fp8(q, s, wq, ws, out, B, H, W, Cin, Cout, kind)
    cols = G.im2col(xd, kind)
    acc, sabs = G.product(cols, wd)
    err = (out.double() - acc).abs()
    r32 = float((err / (V.coef(taps * Cin) * sabs)).max())
    ref, S, A = V.conv_ref(xd, wd, kind, G.STORE, {})
    r = G.worst_ratio(out, ref, V.tolerance(ref, S, A, False))
    print(f"{case}: worst |err| / (coef(K) s) = {r32:.3g}, worst |err| / tol = {r:.3g}")
    assert r <= 1.0


CONVT_CASES = {
    "c5_up_2048_1024": (1, 32, 32, 2048, 1024, False),
    "edge_convt_multi_image": (3, 4, 4, 128, 128, False),
    "edge_convt_n64": (2, 8, 8, 256, 64, False),
    "rgb_n64": (2, 16, 16, 128, 64, True),
    "rgb_n128": (2, 16, 16, 256, 128, True),
    "rgb_n256": (1, 32, 32, 256, 256, True),
}


@pytest.mark.parametrize("case", list(CONVT_CASES))
def test_conv_transpose2d_fp8_against_fp64(case):
    B, H, W, Cin, Cout, rgb = CONVT_CASES[case]
    o = ops()
    q, s, wq, ws, xd, wd = _operands(case, B, H, W, Cin, 4 * Cout, 4 * Cin)
    wq, ws, wd = wq.view(4, Cout, 4 * Cin), ws.view(4, Cout), wd.view(4, Cout, 4 * Cin)
    p = {"bias": G.rnd(case + ".b", (Cout,), 0.5).cuda()}
    if rgb:
        p["rgb_w"] = G.rnd(case + ".rw", (3, Cout), 0.2).cuda()
        p["rgb_b"] = G.rnd(case + ".rb", (3,), 0.2).cuda()
        buf = torch.full((B + 1, 3, 2 * H, 2 * W), GUARD, device="cuda")
        out = buf[:B]
        call = lambda: o.conv_transpose2d_fp8(q, s, wq, ws, out, B, H, W, Cin, Cout, bias=p["bias"], rgb_w=p["rgb_w"], rgb_b=p["rgb_b"])
    else:
        buf = torch.full((B * 4 * H * W + 64, Cout), GUARD, device="cuda", dtype=torch.bfloat16)
        out = buf[:B * 4 * H * W]
        call = lambda: o.conv_transpose2d_fp8(q, s, wq, ws, out, B, H, W, Cin, Cout, bias=p["bias"])
    s0 = L().simt_launch_count()
    names = kernels_of(call)
    assert L().simt_launch_count() == s0
    g = G.tile_geometry(H, W)
    bn = want_bn(g[3] * g[4] * ((B + g[2] - 1) // g[2]), Cout, rgb)
    assert_ran(names, f"tc_gemm_kernel<{bn}, 0, __nv_fp8_e4m3>")
    assert bool((buf[B:] == GUARD).all() if rgb else (buf[B * 4 * H * W:] == GUARD).all())
    ref, S, A = V.convt_ref(xd, wd, p, rgb=rgb)
    got = out.float() if rgb else out.float().reshape(B, 2 * H, 2 * W, Cout)
    r = G.worst_ratio(got, ref, V.tolerance(ref, S, A, not rgb))
    RATIOS[case] = r
    print(f"{case}: K = {4 * Cin}, worst |err| / tol = {r:.3g}")
    assert r <= 1.0


def test_rejections():
    o, lib = ops(), L()
    x = torch.zeros((2 * 8 * 8, 64), device="cuda", dtype=E4)
    sc = torch.ones((2,), device="cuda")
    w = torch.zeros((128, 9 * 64), device="cuda", dtype=E4)
    ws = torch.ones((128,), device="cuda")
    out = torch.empty((2 * 64, 128), device="cuda", dtype=torch.bfloat16)
    n0 = lib.launch_count()
    with pytest.raises(lib.MMGError, match="Cin % 128"):
        o.conv2d_fp8(x, sc, w, ws, out, 2, 8, 8, 64, 128, 1)
    big = torch.zeros((2 * 64 * 128 + 8,), device="cuda", dtype=E4)
    xm = big[8:].view(2 * 64, 128)                                   # 8 bytes off a 16-byte boundary
    w = torch.zeros((128, 9 * 128), device="cuda", dtype=E4)
    with pytest.raises(lib.MMGError, match="16-byte"):
        o.conv2d_fp8(xm, sc, w, ws, out, 2, 8, 8, 128, 128, 1)
    x = torch.zeros((2 * 64, 128), device="cuda", dtype=E4)
    with pytest.raises(lib.MMGError, match="kind"):
        o.conv2d_fp8(x, sc, w, ws, out, 2, 8, 8, 128, 128, 3)
    with pytest.raises(lib.MMGError, match="tile geometry"):
        o.conv2d_fp8(torch.zeros((2 * 6 * 6, 128), device="cuda", dtype=E4), sc, w, ws, out, 2, 6, 6, 128, 128, 1)
    wt = torch.zeros((4, 192, 4 * 128), device="cuda", dtype=E4)
    img = torch.empty((2, 3, 16, 16), device="cuda")
    with pytest.raises(lib.MMGError, match="CONVT_RGB"):
        o.conv_transpose2d_fp8(x, sc, wt, torch.ones((4, 192), device="cuda"), img, 2, 8, 8, 128, 192, rgb_w=torch.ones((3, 192), device="cuda"),
                               rgb_b=torch.zeros((3,), device="cuda"))
    with pytest.raises(lib.MMGError, match="16-byte"):
        o.quantize_e4m3_images(torch.zeros((2 * 64 * 128 + 4,), device="cuda", dtype=torch.bfloat16)[4:].view(2 * 64, 128), 2)
    torch.cuda.synchronize()
    assert lib.launch_count() == n0                                  # nothing was launched


# ------------------------------------------------------------------------------------------------ end to end
def _vaes(dim, layers, seed=0):
    import muse_maskgit_pytorch_b200 as M
    torch.manual_seed(seed)
    ref = M.VQGanVAE(dim=dim, layers=layers, codebook_size=65536).cuda()
    out = {}
    for prec in ("bf16", "fp8", "fp32"):
        v = M.VQGanVAE(dim=dim, layers=layers, codebook_size=65536, precision=prec).cuda()
        v.load_state_dict(ref.state_dict())
        out[prec] = v
    return out


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_vae_dim256_512px_end_to_end():
    vaes = _vaes(256, 4)
    g = torch.Generator(device="cuda").manual_seed(3)
    img = torch.rand((2, 3, 512, 512), device="cuda", generator=g) * 2 - 1
    ids_bf16 = vaes["bf16"].encode_ids(img)
    ids_fp8 = vaes["fp8"].encode_ids(img)
    assert ids_fp8.shape == ids_bf16.shape and ids_fp8.dtype == ids_bf16.dtype
    agree = float((ids_fp8 == ids_bf16).double().mean())
    bits_bf16 = ((ids_bf16[..., None] >> torch.arange(16, device="cuda")) & 1)
    bits_fp8 = ((ids_fp8[..., None] >> torch.arange(16, device="cuda")) & 1)
    bit_agree = float((bits_bf16 == bits_fp8).double().mean())
    ids = ids_bf16
    dec = {p: vaes[p].decode_from_ids(ids) for p in ("bf16", "fp8", "fp32")}
    assert dec["fp8"].shape == dec["fp32"].shape and dec["fp8"].dtype == dec["fp32"].dtype
    e8, e16 = _rel_l2(dec["fp8"], dec["fp32"]), _rel_l2(dec["bf16"], dec["fp32"])
    fq8, ids8, _ = vaes["fp8"].encode(img)
    fq16, _, _ = vaes["bf16"].encode(img)
    assert fq8.shape == fq16.shape and fq8.dtype == fq16.dtype and torch.equal(ids8, ids_fp8)
    fwd = vaes["fp8"](img)
    assert fwd.shape == img.shape and fwd.dtype == torch.float32 and bool(torch.isfinite(fwd).all())
    print(f"encode_ids: token agreement fp8 vs bf16 {agree:.4f}, LFQ bit agreement {bit_agree:.4f}; decode_from_ids rel L2 vs fp32: "
          f"fp8 {e8:.4g}, bf16 {e16:.4g}")
    # bounds from the measurement recorded in DESIGN.md (H100: bit agreement 0.975, token agreement 0.667, fp8 rel L2 0.0044), with margin
    assert bit_agree >= 0.95
    assert e8 <= 0.01


def test_generate_with_fp8_vae_same_tokens():
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    res = {}
    for prec in ("bf16", "fp8"):
        torch.manual_seed(0)
        tr = M.MaskGitTransformer(num_tokens=512, dim=128, seq_len=256, depth=2, heads=2, t5_name="synth-128")
        torch.manual_seed(1)
        vae = M.VQGanVAE(dim=256, codebook_size=512, precision=prec)                # the benchmark VAE's widths, 256^2 -> 16^2 tokens
        te = torch.randn((4, 8, 128), generator=torch.Generator().manual_seed(5)).cuda()
        tr.encode_text = lambda texts, te=te: te[:len(texts)]
        mg = M.MaskGit(image_size=256, transformer=tr, vae=vae).cuda()
        mg.sampler_seed = 11
        res[prec] = mg.generate(["a", "b", "c"], timesteps=6, return_ids=True)
        assert mg.vae.precision == prec
    (img16, ids16), (img8, ids8) = res["bf16"], res["fp8"]
    assert torch.equal(ids8, ids16)
    e = _rel_l2(img8, img16)
    print(f"generate(): images over the fp8 VAE vs the bf16 VAE, rel L2 {e:.4g}")
    assert e <= 0.015                                            # measured 0.63 %, the margin of the decode check above


def test_fp8_vae_bitwise_deterministic():
    vaes = _vaes(128, 2, seed=4)
    g = torch.Generator(device="cuda").manual_seed(9)
    img = torch.rand((3, 3, 128, 128), device="cuda", generator=g) * 2 - 1
    v = vaes["fp8"]
    a, b = v(img), v(img)
    assert torch.equal(a, b)
    assert torch.equal(v.encode_ids(img), v.encode_ids(img))

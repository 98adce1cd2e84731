"""CPU: the oracle of VQGanVAE precision="fp8" (tests/vae_fp8_oracle.py) — the per-image quantiser against torch's e4m3 cast, the
restated e4m3 convolutions inside the bound, each planted indexing defect far outside it, and the constructor's width check."""
import numpy as np
import pytest
import torch

from tests import gemm_oracle as G
from tests import vae_fp8_oracle as V


def test_quantiser_matches_torch_cast_with_zero_image_and_ragged_batch():
    B, hw, C = 3, 7 * 5, 128
    x = G.bf(G.rnd("q.x", (B * hw, C), 2.0))
    x[hw:2 * hw] = 0                                     # image 1 all zero
    x[5, 3] = 1000.                                      # a large value in image 0
    bits, sc = V.quantize_images(x, B)
    assert sc.dtype == np.float32 and sc[1] == 0 and not bits[hw:2 * hw].any()
    for b in (0, 2):
        xb = x[b * hw:(b + 1) * hw]
        amax = np.float32(xb.abs().max())
        assert sc[b] == amax / np.float32(448)
        inv = np.float32(448) / amax
        want = (xb * torch.tensor(inv)).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
        assert np.array_equal(bits[b * hw:(b + 1) * hw], want)
    back = V.dequant_images(bits, sc, B)
    assert float((back - x).abs().max()) <= 2.0 ** -4 * float(x.abs().max())


def _conv_case(kind, B, H, W, Cin, Cout, epi_kind, tag):
    x = V.probe_image(tag, B, H, W, Cin)
    taps = (1, 9, 16)[kind]
    w = V.probe_weight(tag, Cout, taps * Cin)
    xb, xs = V.quantize_images(x.reshape(-1, Cin), B)
    wb, ws = V.quantize_weight_rows(w)
    xq, wq = V.e4m3_values(xb).reshape(x.shape), V.e4m3_values(wb)
    xd = (xq.reshape(B, -1) * torch.from_numpy(xs)[:, None]).reshape(x.shape)
    wd = wq * torch.from_numpy(ws)[:, None]
    Ho, Wo = G.conv_out_hw(kind, H, W)
    p = {"bias": G.rnd(tag + ".b", (Cout,), 0.5)}
    if epi_kind == G.RESIDUAL:
        p["resid"] = G.bf(G.rnd(tag + ".r", (B * Ho * Wo, Cout), 1.0))
    if kind == 2:
        p["act"] = 1
    ref, S, A = V.conv_ref(xd, wd, kind, epi_kind, p)
    return (xq, xs, wq, ws, p), ref, V.tolerance(ref, S, A, True)


CONV_CASES = {"3x3": (1, 2, 8, 8, 128, 128, G.STORE), "1x1_residual": (0, 3, 4, 4, 256, 128, G.RESIDUAL),
              "4x4s2_leaky": (2, 2, 8, 8, 128, 64, G.STORE), "3x3_glu": (1, 2, 4, 8, 128, 256, G.GLU)}


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_clean_restatement_inside_bound(case):
    kind, B, H, W, Cin, Cout, epi = CONV_CASES[case]
    (xq, xs, wq, ws, p), ref, tol = _conv_case(kind, B, H, W, Cin, Cout, epi, case)
    got = V.emulate_conv(xq, xs, wq, ws, kind, epi, p)
    assert G.worst_ratio(got, ref, tol) <= 1.0


def _convt_case(B, H, W, Cin, Cout, tag):
    x = V.probe_image(tag, B, H, W, Cin)
    wt = G.bf(G.rnd(tag + ".wt", (Cin, Cout, 4, 4), 1.0))
    wp = G.pack_convt_weight(wt)                                   # [4, Cout, 4 Cin]
    xb, xs = V.quantize_images(x.reshape(-1, Cin), B)
    wb, ws = V.quantize_weight_rows(wp.reshape(-1, 4 * Cin))       # one scale per row of each parity stack
    xq, wq = V.e4m3_values(xb).reshape(x.shape), V.e4m3_values(wb).reshape(wp.shape)
    ws = torch.from_numpy(ws).reshape(4, Cout)
    xd = (xq.reshape(B, -1) * torch.from_numpy(xs)[:, None]).reshape(x.shape)
    wd = wq * ws[:, :, None]
    p = {"bias": G.rnd(tag + ".b", (Cout,), 0.5)}
    ref, S, A = V.convt_ref(xd, wd, p)
    return (xq, xs, wq, ws, p), ref, V.tolerance(ref, S, A, True)


def test_clean_convt_restatement_inside_bound():
    (xq, xs, wq, ws, p), ref, tol = _convt_case(2, 4, 4, 128, 64, "ct")
    assert G.worst_ratio(V.emulate_convt(xq, xs, wq, ws, p), ref, tol) <= 1.0


@pytest.mark.parametrize("defect", V.DEFECTS)
def test_planted_defect_exceeds_bound_100x(defect):
    if defect == "convt_parity_swapped":
        (xq, xs, wq, ws, p), ref, tol = _convt_case(2, 4, 4, 128, 64, "ct")
        got = V.emulate_convt(xq, xs, wq, ws, p, defect=defect)
    else:
        case = "3x3_glu" if defect == "glu_halves_swapped" else "3x3"
        kind, B, H, W, Cin, Cout, epi = CONV_CASES[case]
        (xq, xs, wq, ws, p), ref, tol = _conv_case(kind, B, H, W, Cin, Cout, epi, case)
        got = V.emulate_conv(xq, xs, wq, ws, kind, epi, p, defect=defect)
    r = G.worst_ratio(got, ref, tol)
    print(f"{defect}: worst |err| / tol = {r:.1f}")
    assert r > 100, r


def test_weight_scales_follow_glu_interleave_and_parity_stacks():
    from muse_maskgit_pytorch_b200.muse_maskgit import quantize_rows_e4m3
    w = G.rnd("pk.w", (4 * 64, 512), 1.0)
    w[70] *= 50                                          # one loud row: its scale must not leak into any other row
    q, s = quantize_rows_e4m3(w)
    qs = [quantize_rows_e4m3(w[64 * i:64 * i + 64]) for i in range(4)]
    assert torch.equal(q.view(torch.uint8), torch.cat([t[0] for t in qs]).view(torch.uint8))
    assert torch.equal(s, torch.cat([t[1] for t in qs]))
    bits, sc = V.quantize_weight_rows(w)
    assert np.array_equal(q.view(torch.uint8).numpy(), bits) and np.array_equal(s.numpy(), sc)
    perm = torch.randperm(w.shape[0], generator=torch.Generator().manual_seed(1))   # any row order (the GLU interleave is one)
    qp, sp = quantize_rows_e4m3(w[perm])
    assert torch.equal(qp.view(torch.uint8), q[perm].view(torch.uint8)) and torch.equal(sp, s[perm])


def test_fp8_vae_constructor_checks_conv_widths():
    import muse_maskgit_pytorch_b200 as M
    vae = M.VQGanVAE(dim=128, layers=2, codebook_size=512, precision="fp8")
    assert vae.precision == "fp8" and sorted(set(vae._conv_input_widths())) == [128, 256]
    with pytest.raises(ValueError, match="fp8.*64 input channels"):
        M.VQGanVAE(dim=64, layers=2, codebook_size=512, precision="fp8")
    with pytest.raises(ValueError, match="fp8"):
        M.VQGanVAE(dim=16, layers=2, codebook_size=512, precision="fp8")


@pytest.mark.parametrize("defect", ["drop_kblock", "wrong_image_scale", "next_column_scale"])
def test_planted_defect_exceeds_bound_at_real_K(defect):
    """at the benchmark VAE's K = 9 x 2048 the bound stays tight enough that one dropped k-block, the next image's scale or the next
    column's weight scale moves some output far outside it"""
    (xq, xs, wq, ws, p), ref, tol = _conv_case(1, 2, 4, 4, 2048, 128, G.STORE, "realK")
    assert G.worst_ratio(V.emulate_conv(xq, xs, wq, ws, 1, G.STORE, p), ref, tol) <= 1.0
    r = G.worst_ratio(V.emulate_conv(xq, xs, wq, ws, 1, G.STORE, p, defect=defect), ref, tol)
    print(f"K = 18432, {defect}: worst |err| / tol = {r:.1f}")
    assert r > 10, r


def test_fp8_vae_rejects_feature_maps_without_tile_geometry():
    from muse_maskgit_pytorch_b200.vqgan_vae import VQGanVAE
    for h, w in ((256, 256), (32, 32), (8, 16)):
        VQGanVAE._check_fp8_grid(h, w)
    for h, w in ((96, 96), (48, 48), (6, 6)):
        with pytest.raises(ValueError, match=f"fp8.*{h} x {w}.*bf16"):
            VQGanVAE._check_fp8_grid(h, w)

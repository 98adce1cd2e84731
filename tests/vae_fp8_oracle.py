"""CPU oracle of VQGanVAE precision="fp8": the per-image quantiser (mmg_quantize_e4m3_images), the error bound of an e4m3 convolution
against fp64 on the dequantised operands, and a restatement of the e4m3 convolutions' index arithmetic that can carry one planted defect.
Imports no CUDA code; tests/test_vae_fp8_oracle.py runs it on the CPU and tests/test_gpu_vae_fp8.py holds the kernels to it.

Quantiser.  Image b of a bf16 NHWC map: amax_b = max |x| (an integer max over the bits of |x| on the GPU, which equals the float max),
inv = 448 / amax_b in fp32 (0 when amax_b == 0), q = e4m3 round-to-nearest-even, saturating, of the fp32 product x * inv, and
scale_b = amax_b / 448 in fp32: the rounding of mmg_layernorm_fp8 (tests/fp8_oracle.py) with one scale per image instead of per row.

Bound.  An output row of a convolution reads only its own image, so acc = sum_k qx_k qw_k carries the exact factor
x_scale[b] * w_scale[c], and the only error before the epilogue is the accumulation.  The kernel promotes: each 128-element k-block is
accumulated by four m64nNk32 wgmma from zero and then added into an fp32 sum.  The fp32 sum is held to the bf16 kernel's bound,
tests/gemm_oracle.py's coef (2 ceil(K / 16) u s; u = 2^-24).  Inside a k-block, Hopper's e4m3 MMA is reported (outside this
repository) to keep 13 mantissa bits in its accumulator, so step j of k-block kb may lose up to U8 = 2^-13 of the exact partial sum
|Q_kb,j| it produces plus the magnitudes s_kb,j of the 32 products it aligns, C8 = 2 times over:
    tol = (coef(K) + 3 u) S + C8 U8 S13 + A (+ 2^-8 |ref| for a bf16 output),   S13 = sum_kb sum_(j = 1..4) (|Q_kb,j| + s_kb,j) = s + sum |Q|
(without the s_kb,j term a row whose mass sits in one k32 step measured 1.3x the bound).
where S, S13 and A are what tests/gemm_oracle.py's epilogue makes of s = sum_k |a_k w_k| and of S13 (the 3 u: the two dequantising
multiplies).  Without promotion the error at K = 18 432 was measured at 4.3x coef(K) S (16 384: 6.3x; a k-block-dominated row at
K = 1 152: 131x): DESIGN.md ("FP8 precision", VAE).

Measured worst |err| / tol per case: tests/test_gpu_vae_fp8.py prints it, DESIGN.md ("FP8 precision", VAE) records it."""
import numpy as np
import torch

from tests import fp8_oracle as Q
from tests import gemm_oracle as G

U = 2.0 ** -24
U8 = 2.0 ** -13
C8 = 2.0
KB = 128                                  # elements per e4m3 k-block

DEFECTS = ("wrong_image_scale", "convt_parity_swapped", "glu_halves_swapped", "drop_kblock")


# ------------------------------------------------------------------------------------------------ quantiser
def quantize_images(x, B):
    """x [B * hw, C] (bf16 values, any float dtype) -> (uint8 e4m3 bits [B * hw, C], fp32 scales [B])"""
    x = np.asarray(torch.as_tensor(x).float().cpu().numpy(), dtype=np.float32)
    rows = x.shape[0] // B
    xb = x.reshape(B, -1)
    bits, scales = Q.quantize_rows(xb)
    return bits.reshape(B * rows, -1), scales


def e4m3_values(bits):
    """uint8 e4m3 bits -> float32 values"""
    return torch.from_numpy(np.ascontiguousarray(bits)).view(torch.float8_e4m3fn).float()


def dequant_images(bits, scales, B):
    v = e4m3_values(bits)
    return (v.reshape(B, -1) * torch.as_tensor(scales).float()[:, None]).reshape(v.shape)


def quantize_weight_rows(w2d):
    """the packer's per-row e4m3 weights (muse_maskgit.quantize_rows_e4m3, restated): (bits, scales [rows])"""
    return Q.quantize_rows(np.asarray(w2d.float().numpy(), dtype=np.float32))


# ------------------------------------------------------------------------------------------------ fp64 reference with the bound's scale
def product_fp8(a, w):
    """acc = a w^T in fp64 and the scale the bound grows with, s + (C8 U8 / coef(K)) S13 (see above), so that coef(K) times what the
    epilogue makes of it is the tolerance; a [M, K], w [N, K] (dequantised operands; K a multiple of 128).  Runs on the operands' device."""
    ad, wd = a.double(), w.double()
    K = ad.shape[1]
    P = torch.zeros((ad.shape[0], wd.shape[0]), dtype=torch.float64, device=ad.device)
    s13 = torch.zeros_like(P)
    for k0 in range(0, K, KB):
        Q = torch.zeros_like(P)
        for j in range(0, KB, 32):
            Q += ad[:, k0 + j:k0 + j + 32] @ wd[:, k0 + j:k0 + j + 32].T
            s13 += Q.abs()
        P += Q
    s = ad.abs() @ wd.abs().T
    return P, s + (C8 * U8 / coef(K)) * (s13 + s)


def coef(K):
    """the fp32 part of the bound: the bf16 kernel's accumulation coefficient at K, plus the two dequantising multiplies"""
    return G.coef(G.TC(128, G.M_REGS), K) + 3 * U


def conv_ref(xd, wd, kind, epi_kind, p):
    """xd [B, H, W, Cin] and wd [Cout, taps * Cin] dequantised: (out, S, A) rows = output pixels; S already carries coef(K)"""
    acc, s = product_fp8(G.im2col(xd, kind), wd)
    out, S, A = G.epilogue(epi_kind, acc, s, p)
    return out, coef(wd.shape[1]) * S, A


def convt_ref(xd, wd, p, rgb=False):
    """xd [B, H, W, Cin], wd [4, Cout, 4 Cin] dequantised: CONVT -> [B, 2H, 2W, Cout]; CONVT_RGB -> [B, ch, 2H, 2W]"""
    B, H, W, _ = xd.shape
    outs = []
    for py in range(2):
        for px in range(2):
            acc, s = product_fp8(G.convt_cols(xd, py, px), wd[py * 2 + px])
            out, S, A = G.epilogue(G.CONVT_RGB if rgb else G.CONVT, acc, s, p)
            outs.append((out, coef(wd.shape[2]) * S, A))
    C = outs[0][0].shape[1]
    res = []
    for i in range(3):
        full = torch.zeros((B, 2 * H, 2 * W, C), dtype=torch.float64, device=xd.device)
        for py in range(2):
            for px in range(2):
                full[:, py::2, px::2] = outs[py * 2 + px][i].reshape(B, H, W, C)
        res.append(full.permute(0, 3, 1, 2).contiguous() if rgb else full)
    return tuple(res)


def tolerance(ref, S, A, out_bf16):
    """S from conv_ref / convt_ref (coef(K) included)"""
    tol = S + A
    return tol + 2.0 ** -8 * ref.abs() if out_bf16 else tol


# ------------------------------------------------------------------------------------------------ the e4m3 convolutions, restated
def _acc_fp8(cols_q, wq, defect):
    """fp32 sum over 128-element k-blocks of the e4m3 values (the unscaled accumulator)"""
    K = cols_q.shape[1]
    blocks = list(range(K // KB))
    if defect == "drop_kblock":
        blocks = blocks[:-1]
    acc = torch.zeros((cols_q.shape[0], wq.shape[0]), dtype=torch.float32)
    for i in blocks:
        acc += cols_q[:, KB * i:KB * i + KB] @ wq[:, KB * i:KB * i + KB].T
    return acc


def _row_scales(x_scale, B, rows_per_image, defect):
    img = torch.arange(B).repeat_interleave(rows_per_image)
    if defect == "wrong_image_scale":
        img = (img + 1) % B                      # the next image's scale
    return torch.as_tensor(x_scale).float()[img]


def _glu_swap(acc):
    """the GLU epilogue reading the interleaved [a(32) | gate(32)] blocks the other way round"""
    M, N = acc.shape
    return acc.reshape(M, N // 64, 2, 32).flip(2).reshape(M, N)


def emulate_conv(xq, x_scale, wq, w_scale, kind, epi_kind, p, defect=None, out_bf16=True):
    """xq [B, H, W, Cin], wq [Cout, taps * Cin]: e4m3 values (float); the clean or defective restatement in fp32"""
    B, H, W, _ = xq.shape
    Ho, Wo = G.conv_out_hw(kind, H, W)
    acc = _acc_fp8(G.im2col(xq, kind), wq, defect)
    ws = torch.as_tensor(w_scale).float()
    if defect == "next_column_scale":
        ws = ws.roll(-1)                         # column c dequantised with column c + 1's scale
    acc = acc * _row_scales(x_scale, B, Ho * Wo, defect)[:, None] * ws[None, :]
    if epi_kind == G.GLU and defect == "glu_halves_swapped":
        acc = _glu_swap(acc)
    out, _, _ = G.epilogue(epi_kind, acc, acc.abs(), p, torch.float32)
    return G.bf(out) if out_bf16 else out


def emulate_convt(xq, x_scale, wq, w_scale, p, defect=None, out_bf16=True):
    """wq [4, Cout, 4 Cin], w_scale [4, Cout]: CONVT output [B, 2H, 2W, Cout]"""
    B, H, W, _ = xq.shape
    N = wq.shape[1]
    full = torch.zeros((B, 2 * H, 2 * W, N), dtype=torch.float32)
    for py in range(2):
        for px in range(2):
            acc = _acc_fp8(G.convt_cols(xq, py, px), wq[py * 2 + px], defect)
            acc = acc * _row_scales(x_scale, B, H * W, defect)[:, None] * torch.as_tensor(w_scale[py * 2 + px]).float()[None, :]
            out, _, _ = G.epilogue(G.CONVT, acc, acc.abs(), p, torch.float32)
            qy, qx = (px, py) if defect == "convt_parity_swapped" else (py, px)
            full[:, qy::2, qx::2] = out.reshape(B, H, W, N)
    return G.bf(full) if out_bf16 else full


# ------------------------------------------------------------------------------------------------ probe operands
def probe_image(tag, B, H, W, C, seed=7):
    """bf16 NHWC map: N(0, 1/64) noise, a spike of 4 (times 1 + 2 b on image b) at a sparse, moving set of pixels and channels, so
    that many output rows are dominated by one tap (one k-block) of one image"""
    x = G.rnd(tag + ".x", (B, H, W, C), 1 / 8, seed)
    for b in range(B):
        for y in range(H):
            for xx in range((y * 3 + b) % 4, W, 4):
                x[b, y, xx, (7 * y + 5 * xx + 11 * b) % C] += 4.0 * (1 + 2 * b)
    return G.bf(x)


def probe_weight(tag, N, K, seed=7):
    return G.bf(G.rnd(tag + ".w", (N, K), 1.0, seed))

"""CPU oracle of mmg_linear, mmg_conv2d and mmg_conv_transpose2d: the launcher's choice of kernel restated as one pure function, fp64
references of every epilogue with the scale each output's rounding errors grow with, a derived tolerance per kernel variant, probe
operands, and a restatement of the tiled product's index arithmetic that can carry one planted defect.  Imports no CUDA code;
tests/test_gemm_oracle.py runs it on the CPU and tests/test_gpu_gemm.py holds the kernels to it.

Operation.  acc[r, c] = sum_k a[r, k] w[c, k] over A [M, K] (dense, or the implicit im2col of an NHWC image) and W [N, K], then the
epilogue.  For each output the reference also returns S, the scale its accumulation error grows with: s = sum_k |a_k w_k| for the
accumulator, carried through the epilogue by the magnitude of its derivative (bias and residual add their own magnitude), and A, the
absolute error the epilogue's own fp32 arithmetic may add.  u = 2^-24.

Tolerance  |got - ref| <= coef(variant, K) * S + A (+ 2^-8 |ref| for a bf16 output: one round to nearest to 8 significant bits).
  bf16 operands on the tensor cores (tc_gemm_kernel): products of bf16 values are exact in fp32, so the accumulation is the only error
      before the epilogue.  The tensor core adds each k16 MMA into its fp32 accumulator and truncates instead of rounding to nearest
      (found in the attention work: tests/attention_oracle.py), losing less than one fp32 ulp, 2 u relative, of the partial sum per MMA.
      The partial sums are bounded by s, so coef = C_ACC * ceil(K / 16) * u with C_ACC = 2.
  fp32 through split3 (mmg_split3, then the bf16 kernel over 6K columns): the same truncation over ceil(6K / 16) MMAs, plus the three
      cross terms the split leaves out (mid*lo, lo*mid, lo*lo: |mid| <= 2^-8 |x|, |lo| <= 2^-16 |x|, so 2 * 2^-24 + 2^-32 of |a w|) and
      the split's own residual (hi + mid + lo carries x to 24 bits; at most u |x| more): coef = C_ACC * ceil(6K / 16) * u + 3 u.
  CUDA-core kernel (simt_gemm_kernel<float | __nv_bfloat16>): a sequential fmaf chain over K in fp32, one rounding per step, so the
      classical bound coef = gamma_K = K u / (1 - K u) holds rigorously (bf16 operands are exact in fp32).
  Epilogue terms, in A: each fp32 add or multiply of the bias, residual, leaky slope or LayerNorm fold rounds once (u of a value bounded
      by S); gelu_fast has a documented absolute error of 6e-7 (mmg_common.cuh; 3.1e-7 measured over [-8, 8], up to 900 u relative in the
      negative tail, where the plain fp32 erf form reaches 856 u), and the fp32 erf form stays inside the same 6e-7 + 2 u |x|;
      tanh.approx.f32 has a relative error below 2^-11 (bf16 outputs only; fp32 outputs use tanhf, 2 ulp), so gelu_tanh is off by
      <= 2^-12 |x|; the GLU's ex2.approx / rcp.approx sigmoid is off by (4 + |g|) u relative; the QKV normalisation (a 64-term sum of
      squares in four chains, rsqrtf, two multiplies) by 16 u relative; the LayerNorm fold by its rstd's relative error, which the
      cancellation sum(x^2)/n - mean^2 amplifies by kappa = (E[x^2] + 2 mean^2) / var; the CONVT_RGB dot product by gamma_(N + 2) of
      sum |v w| + |b|.
  Where the output is bf16 the rounding bound 2^-8 |ref| is reached by construction on any large output, so those variants' worst
  |err| / tol sits near 1; the accumulation part of the bound is far from reached (the CPU emulation stays below half of it).

Observed worst |err| / tol per variant over tests/test_gpu_gemm.py: OBSERVED below.

What the old rules let through.  tests/test_gpu_kernels.py allows 2e-2 + 1e-2 |ref| for bf16 outputs and 2e-4 + 1e-3 |ref| for fp32
outputs on random N(0, 1) data.  tests/test_gemm_oracle.py::test_what_the_old_rules_accepted replays the planted defects against
those rules on that kind of data: both rules reject all twelve, since each moves whole rows or columns by O(|ref|).  What that file
could not see is which kernel ran: most routes of the table in DESIGN.md were reached only as a side effect, or never."""
import math

import torch
import torch.nn.functional as F

from oracle import synth

U = 2.0 ** -24
C_ACC = 2.0
GELU_ABS = 6e-7
TANH_APPROX = 2.0 ** -12

# epilogue kinds (include/mmg.h)
STORE, RESIDUAL, GEGLU, GLU, QKV, CONVT, CONVT_RGB, LNFOLD, LFQ_IDS, ARGMIN, GEGLU_TANH, QKV128 = range(12)
# tc_gemm_kernel EPI_MODE values (mmg_gemm_tc.cuh)
M_REGS, M_REDUCE, M_TSTORE, M_QKV, M_GEGLU, M_ACT, M_QKV128 = 0, 2, 3, 4, 5, 6, 7
SPLIT3 = "split3_kernel"
E4M3 = "__nv_fp8_e4m3"


def TC(bn, mode, ta="__nv_bfloat16"):
    return f"tc_gemm_kernel<{bn}, {mode}, {ta}>"


def SIMT(dtype, conv, act):
    return f"simt_gemm_kernel<{'float' if dtype == 'f32' else '__nv_bfloat16'}, {str(bool(conv)).lower()}, {str(bool(act)).lower()}>"


# every bf16 instantiation the launchers can reach, and the CUDA-core ones
TC_VARIANTS = [TC(64, M_REGS), TC(128, M_REGS), TC(256, M_REGS), TC(64, M_REDUCE), TC(128, M_REDUCE), TC(256, M_REDUCE),
               TC(128, M_TSTORE), TC(256, M_TSTORE), TC(128, M_QKV), TC(256, M_QKV), TC(256, M_GEGLU), TC(128, M_ACT)]
SIMT_VARIANTS = [SIMT(t, c, a) for t in ("f32", "bf16") for c, a in ((False, False), (True, False), (False, True))]

# worst |err| / tol per variant in one run of tests/test_gpu_gemm.py on one NVIDIA H100 80GB HBM3 (132 SMs, driver 580.159.03, 700 W power
# limit); a record, not a limit.  Variants with bf16 outputs sit at the half-ulp rounding term by construction; the fp32-output tile
# epilogues (REDUCE, TSTORE at K = 64) show the tensor core's truncation at about 0.7 of the bound.
OBSERVED = {TC(64, M_REGS): 0.996, TC(128, M_REGS): 0.996, TC(256, M_REGS): 0.002, TC(64, M_REDUCE): 0.486, TC(128, M_REDUCE): 0.621,
            TC(256, M_REDUCE): 0.718, TC(128, M_TSTORE): 0.667, TC(256, M_TSTORE): 0.738, TC(128, M_QKV): 0.995, TC(256, M_QKV): 0.996,
            TC(256, M_GEGLU): 0.995, TC(128, M_ACT): 0.996, "split": 0.992, SIMT("f32", False, False): 0.115, SIMT("f32", True, False): 0.005,
            SIMT("f32", False, True): 0.139, SIMT("bf16", False, False): 0.123, SIMT("bf16", True, False): 0.977, SIMT("bf16", False, True): 0.143}

DEFECTS = ("drop_last_kblock", "kblock_twice", "ragged_row_off_by_one", "tile_order_swapped", "tap_dx_dy_swapped", "parity_py_px_swapped",
           "wrong_image_in_tile", "convt_parity_swapped", "geglu_x_gate_swapped", "lnfold_one_slot_short", "qkv_next_head", "null_row_missing")


# ------------------------------------------------------------------------------------------------ dispatch, restated
def pick_bn(m_tiles, N, kind, sms):
    if kind == CONVT_RGB:
        return N
    if N % 256 == 0 and m_tiles * (N // 256) >= 2 * sms:
        return 256
    if N % 128 == 0 and m_tiles * (N // 128) >= sms:
        return 128
    if N % 128 == 0 and N >= 1024:
        return 128
    if N % 64 == 0 and N % 128 != 0:
        return 64
    return 128 if m_tiles * ((N + 127) // 128) >= 96 else 64


def n_fast(N, K, n_tiles):
    return int(N * K * 2 <= (8 << 20) and 1 < n_tiles <= 16)


def tile_geometry(Ho, Wo):
    """(TW, TH, TB, tiles_x, tiles_y) of a conv tile of 128 output pixels, or None where the tensor-core path does not take the image"""
    TW = min(Wo, 128)
    if TW <= 0 or 128 % TW or Wo % TW:
        return None
    TH = min(128 // TW, Ho)
    if Ho % TH or 128 % (TW * TH):
        return None
    return TW, TH, 128 // (TW * TH), Wo // TW, Ho // TH


def is_act(kind, e):
    return kind == GEGLU_TANH or (kind == STORE and e.get("act", 0) == 2)


def tc_plan(kind, e, M, N, K, m_tiles, sms, conv):
    """(tile width, EPI_MODE, n_fast) of plan_tc for bf16 operands.  e: out ('f32' | 'bf16'), act, bias, in_place (out is resid with
    ldr == ldo), ldo, out_aligned (16 bytes), tokens, nq / nk / nv heads, qkv_aligned."""
    bn = pick_bn(m_tiles, N, kind, sms)
    if is_act(kind, e):
        return 128, M_ACT, n_fast(N, K, (N + 127) // 128)
    f32, ldo, al = e.get("out", "f32") == "f32", e.get("ldo", N), e.get("out_aligned", True)
    in_place = (kind == LNFOLD or (kind == RESIDUAL and e.get("act", 0) == 0)) and f32 and e.get("in_place", False) and ldo % 4 == 0 and al and not conv
    plain = kind == STORE and f32 and not conv and not e.get("bias") and e.get("act", 0) == 0 and ldo % 4 == 0 and al
    qkv = (kind == QKV and not f32 and not conv and e["tokens"] % 32 == 0 and M % 128 == 0 and bn in (128, 256) and e.get("qkv_aligned", True)
           and e["nk"] == e["nv"])
    geglu = kind == GEGLU and not f32 and not conv and bn == 256 and ldo % 8 == 0 and al
    mode = M_REDUCE if in_place else M_TSTORE if plain and bn in (128, 256) else M_QKV if qkv else M_GEGLU if geglu else M_REGS
    if mode == M_REGS and bn == 256 and kind != CONVT_RGB:
        bn = 128
    if mode != M_REGS and N % bn:
        raise ValueError("tile epilogue: tile width does not divide N")
    return bn, mode, n_fast(N, K, (N + bn - 1) // bn)


def fp8_plan(kind, M, N, K, sms):
    """(tile width, EPI_MODE, n_fast) of mmg_linear_fp8 (QKV, QKV128 or GEGLU; its argument checks refuse the shapes the tile epilogues
    do not take).  An e4m3 dense product has no register-epilogue instantiation, so it always takes its tile epilogue: QKV and QKV128 at
    256 where pick_bn gives 256 and at 128 otherwise, GEGLU at 256.  This differs from tc_plan at small M: a 256-row cross-attention q
    product with N = 128 runs <128, QKV, e4m3> where the bf16 product of that shape runs <64, REGS>."""
    if kind == GEGLU:
        bn, mode = 256, M_GEGLU
    else:
        bn, mode = 256 if pick_bn((M + 127) // 128, N, kind, sms) == 256 else 128, M_QKV if kind == QKV else M_QKV128
    return bn, mode, n_fast(N, K, N // bn)


def linear_kernels(M, N, K, kind, e, *, dtype="bf16", sms=132, lda=None, ldw=None, a_aligned=True, w_aligned=True, split=False, order=False):
    """[kernel names] one mmg_linear call launches; split: an fp32 ops.linear that goes through mmg_split3 first (ops.linear takes that
    route when fp32_tc() and K % 64 == 0 and N % 64 == 0).  order: return (names, n_fast of the tensor-core launch or None)"""
    names = []
    lda, ldw = lda or K, ldw or K
    if split:
        assert dtype == "f32" and K % 64 == 0 and N % 64 == 0
        names, dtype, K, lda, ldw = [SPLIT3], "bf16", 6 * K, 6 * K, 6 * K
    ldo_ok = e.get("ldo", N) % 8 == 0 or kind in (QKV, CONVT_RGB, LFQ_IDS, ARGMIN)
    tc_ok = dtype == "bf16" and K % 64 == 0 and N % 64 == 0 and lda % 8 == 0 and ldw % 8 == 0 and a_aligned and w_aligned and ldo_ok
    if not tc_ok:
        names = names + [SIMT(dtype, False, is_act(kind, e))]
        return (names, None) if order else names
    bn, mode, nf = tc_plan(kind, e, M, N, K, (M + 127) // 128, sms, False)
    return (names + [TC(bn, mode)], nf) if order else names + [TC(bn, mode)]


def conv_out_hw(kind, H, W):
    s = 2 if kind == 2 else 1
    return H // s, W // s


def conv_kernels(kind, B, H, W, Cin, Cout, epi_kind, e, *, dtype="bf16", sms=132, aligned=True, split=False, order=False):
    names = []
    if split:
        assert dtype == "f32" and Cin % 32 == 0 and Cout % 64 == 0 and kind != 3
        names, dtype, Cin = [SPLIT3], "bf16", 6 * Cin
    Ho, Wo = conv_out_hw(kind, H, W)
    g = tile_geometry(Ho, Wo)
    taps = (1, 9, 16, 25)[kind]
    tc_ok = dtype == "bf16" and kind != 3 and Cin % 64 == 0 and Cout % 64 == 0 and aligned and e.get("ldo", Cout) % 8 == 0 and g is not None
    if not tc_ok:
        names = names + [SIMT(dtype, True, False)]
        return (names, None) if order else names
    m_tiles = g[3] * g[4] * ((B + g[2] - 1) // g[2])
    bn, mode, nf = tc_plan(epi_kind, e, B * Ho * Wo, Cout, taps * Cin, m_tiles, sms, True)
    return (names + [TC(bn, mode)], nf) if order else names + [TC(bn, mode)]


def convt_kernels(B, H, W, Cin, Cout, rgb, *, dtype="bf16", sms=132, ldo=None, split=False, order=False):
    """four launches, one per output parity class; CONVT_RGB off the tensor-core path is an argument error (ValueError)"""
    names = []
    if split:
        assert dtype == "f32" and Cin % 32 == 0 and Cout % 64 == 0
        names, dtype, Cin = [SPLIT3], "bf16", 6 * Cin
    g = tile_geometry(H, W)
    ldo = Cout if ldo is None else ldo
    tc_ok = dtype == "bf16" and Cin % 64 == 0 and Cout % 64 == 0 and (Cout in (64, 128, 256) if rgb else ldo % 8 == 0) and g is not None
    if not tc_ok:
        if rgb:
            raise ValueError("CONVT_RGB needs the bf16 tensor-core path")
        names = names + [SIMT(dtype, True, False)] * 4
        return (names, None) if order else names
    m_tiles = g[3] * g[4] * ((B + g[2] - 1) // g[2])
    bn, mode, nf = tc_plan(CONVT_RGB if rgb else CONVT, {"out": "f32"}, B * H * W, Cout, 4 * Cin, m_tiles, sms, True)
    return (names + [TC(bn, mode)] * 4, nf) if order else names + [TC(bn, mode)] * 4


# ------------------------------------------------------------------------------------------------ operands
def rnd(tag, shape, std=1.0, seed=5):
    return torch.from_numpy(synth.normal(tag, shape, seed)).float() * std


def bf(t):
    return t.to(torch.bfloat16).float()


def probe_dense(tag, M, N, K, bf16=True):
    """a [M, K], w [N, K] fp32 (bf16-representable when bf16): N(0, 1/64) noise; row r of a carries a spike of 4 in k-block r % (K / 64)
    at a column that moves with the row, so each row is dominated by one k-block and rows next to each other (box edges, the ragged last
    block) differ by far more than the bound; w ~ N(0, 1) gives every column and k-block its own signature"""
    a = rnd(tag + ".a", (M, K), 1 / 64)
    w = rnd(tag + ".w", (N, K))
    nkb = max(K // 64, 1)
    r = torch.arange(M)
    a[r, ((r % nkb) * 64 + (r * 7) % 64) % K] += 4.0
    return (bf(a), bf(w)) if bf16 else (a, w)


def probe_image(tag, B, H, W, C, bf16=True):
    """NHWC x ~ N(0, 1/4) with the border pixels raised (+2 on rows 0, H-1 and columns 0, W-1, +1 on the stride-2 border rows 1, H-2 and
    columns 1, W-2): a tap that reads past or short of an edge moves the output far beyond the bound"""
    x = rnd(tag + ".x", (B, H, W, C), 0.5)
    x[:, 0] += 2; x[:, -1] += 2; x[:, :, 0] += 2; x[:, :, -1] += 2
    if H > 3:
        x[:, 1] += 1; x[:, -2] += 1
    if W > 3:
        x[:, :, 1] += 1; x[:, :, -2] += 1
    x = x * (1 + torch.arange(B).float()[:, None, None, None] * 0.5)       # a scale per image
    return bf(x) if bf16 else x


# ------------------------------------------------------------------------------------------------ im2col and packing
def conv_taps(kind):
    k, pad = ((1, 0), (3, 1), (4, 1), (5, 2))[kind]
    return [(r - pad, s - pad) for r in range(k) for s in range(k)], 2 if kind == 2 else 1


def im2col(x, kind, defect=None):
    """[B, H, W, C] -> [B * Ho * Wo, taps * C], tap-major (tap t = r * k + s), zero outside the image; the layout of the packed weights"""
    B, H, W, C = x.shape
    taps, st = conv_taps(kind)
    Ho, Wo = H // st, W // st
    xp = F.pad(x, (0, 0, 3, 3, 3, 3))
    cols = []
    for dy, dx in taps:
        if defect == "tap_dx_dy_swapped":
            dy, dx = dx, dy
        if defect == "parity_py_px_swapped" and kind == 2:
            # tap_map = px * 2 + py: rows of parity px, columns of parity py, at the same half-resolution offsets
            py, px = dy % 2, dx % 2
            hy, hx = (dy - py) // 2, (dx - px) // 2
            ys = 2 * (torch.arange(Ho) + hy) + px
            xs = 2 * (torch.arange(Wo) + hx) + py
        else:
            ys = torch.arange(Ho) * st + dy
            xs = torch.arange(Wo) * st + dx
        cols.append(xp[:, ys + 3][:, :, xs + 3])
    return torch.cat(cols, -1).reshape(B * Ho * Wo, len(taps) * C)


def pack_conv_weight(wt):
    """torch Conv2d weight [Cout, Cin, k, k] -> [Cout, k * k * Cin] (tap-major)"""
    return wt.permute(0, 2, 3, 1).reshape(wt.shape[0], -1)


CT_R = ((1, 3), (0, 2))
CT_D = ((0, -1), (1, 0))


def pack_convt_weight(wt):
    """torch ConvTranspose2d weight [Cin, Cout, 4, 4] -> [4 parity classes, Cout, 4 * Cin] (vqgan_vae.py's packing)"""
    packs = []
    for py in range(2):
        for px in range(2):
            packs.append(torch.cat([wt[:, :, CT_R[py][a], CT_R[px][b]].t() for a in range(2) for b in range(2)], dim=1))
    return torch.stack(packs)


def convt_cols(x, py, px):
    """[B, H, W, C] -> the A operand of parity class (py, px): [B * H * W, 4 * C], tap t = a * 2 + b at input offset (CT_D[py][a], CT_D[px][b])"""
    B, H, W, C = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    cols = []
    for a in range(2):
        for b in range(2):
            dy, dx = CT_D[py][a], CT_D[px][b]
            cols.append(xp[:, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W])
    return torch.cat(cols, -1).reshape(B * H * W, 4 * C)


# ------------------------------------------------------------------------------------------------ epilogues
def _gelu_erf(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2.0)))


def _gelu_tanh(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))


def _leaky(x):
    return torch.where(x > 0, x, 0.1 * x)


def _halves(t):
    """[M, N] in 64-column chunks [x(32) | gate(32)] -> (x, gate), each [M, N / 2]"""
    M, N = t.shape
    c = t.reshape(M, N // 64, 2, 32)
    return c[:, :, 0].reshape(M, N // 2), c[:, :, 1].reshape(M, N // 2)


def epilogue(kind, acc, s, p, dt=torch.float64, defect=None):
    """(out, S, A) for the accumulator acc [M, N] and its scale s, in dtype dt (fp64: the reference; fp32: the emulation).  p holds the
    epilogue's operands: bias [N], act, resid [M, N], out ('f32' | 'bf16'), approx (the bf16 tensor-core path's fast functions),
    QKV: heads, tokens, key_off, q_rows, kv_rows, q_scale, k_scale, null_k, null_v (a dict of outputs q, k, v is returned as out);
    LNFOLD: stats [M, slots, 2], ln_width, cvec (= bias); LFQ_IDS: bits; CONVT_RGB: rgb_w [ch, N], rgb_b [ch] (out: [M, ch])."""
    acc, s = acc.to(dt), s.to(dt)
    z = torch.zeros_like(acc)
    bias = p.get("bias")
    b = z + bias.to(dt) if bias is not None else z
    ab = b.abs()
    approx = p.get("approx", False)
    if kind in (STORE, RESIDUAL, CONVT):
        v = acc + b
        S = s + ab
        if kind == RESIDUAL:
            r = p["resid"].to(dt)
            v, S = v + r, S + r.abs()
        if kind == CONVT or p.get("act", 0) == 1:
            v = _leaky(v)
        elif p.get("act", 0) == 2:
            v = v.clamp_min(0)
        return v, S, 3 * U * S
    if kind == CONVT_RGB:
        v = _leaky(acc + b)
        S = s + ab
        rw, rb = p["rgb_w"].to(dt), p["rgb_b"].to(dt)
        out = v @ rw.T + rb
        n = acc.shape[1] + 2
        gam = n * U / (1 - n * U)
        return out, S @ rw.abs().T, (2 * U * S) @ rw.abs().T + gam * (v.abs() @ rw.abs().T + rb.abs())
    if kind in (GEGLU, GEGLU_TANH):
        x, g = _halves(acc)
        sx, sg = _halves(s)
        if defect == "geglu_x_gate_swapped":
            x, g = g, x
        ge = _gelu_erf(x) if kind == GEGLU else _gelu_tanh(x)
        out = g * ge
        S = ge.abs() * sg + 1.13 * g.abs() * sx
        if kind == GEGLU:
            err = GELU_ABS + 2 * U * x.abs()
        else:
            err = (TANH_APPROX if approx else 3 * U) * x.abs()
        return out, S, g.abs() * err + 2 * U * out.abs()
    if kind == GLU:
        x, g = _halves(acc + b)
        sx, sg = _halves(s + ab)
        sig = torch.sigmoid(g)
        out = x * sig
        S = sig * sx + x.abs() * sig * (1 - sig) * sg
        return out, S, (4 + g.abs() + 2) * U * out.abs()
    if kind == LNFOLD:
        st = p["stats"].to(dt)                           # [M, slots, 2]
        if defect == "lnfold_one_slot_short":
            st = st[:, :-1]
        n, slots = p["ln_width"], st.shape[1]
        sx, sq = st[..., 0].sum(1), st[..., 1].sum(1)
        mean = sx / n
        var = (sq / n - mean * mean).clamp_min(0)
        rstd = 1 / torch.sqrt(var + 1e-5)
        c = b
        lin = acc - mean[:, None] * c
        r = p["resid"].to(dt)
        out = rstd[:, None] * lin + r
        sabs = st[..., 0].abs().sum(1) / n
        dvar = (slots + 2) * U * (sq / n + 2 * mean.abs() * sabs + mean * mean)
        drel = 0.5 * dvar / (var + 1e-5) + 3 * U
        dmean = (slots + 1) * U * sabs
        A = rstd[:, None] * (dmean[:, None] * c.abs() + U * (mean[:, None] * c).abs() + U * lin.abs()) + drel[:, None] * (rstd[:, None] * lin).abs() \
            + U * out.abs()
        return out, rstd[:, None] * s, A
    if kind == QKV:
        return _qkv(acc, s, p, dt, defect)
    raise ValueError(kind)


def _qkv(acc, s, p, dt, defect):
    """q / k / v head layouts of the QKV epilogue: rows r = b * tokens + t; head chunk c = which * heads + h"""
    M, N = acc.shape
    H, T, ko = p["heads"], p["tokens"], p["key_off"]
    Bq = M // T
    nq, nk = p.get("nq", H), p.get("nk", H)
    out, S, A = {}, {}, {}
    chunks = acc.reshape(Bq, T, N // 64, 64)
    schunks = s.reshape(Bq, T, N // 64, 64)
    groups = [("q", nq, p.get("q_scale")), ("k", nk, p.get("k_scale")), ("v", nk, None)]
    c0 = 0
    for name, nh, sc in groups:
        if nh == 0:
            continue
        x = chunks[:, :, c0:c0 + nh].to(dt)             # [Bq, T, nh, 64]
        sx = schunks[:, :, c0:c0 + nh].to(dt)
        c0 += nh
        if sc is not None:
            norm = x.norm(dim=-1, keepdim=True).clamp_min(1e-12)
            xh = x / norm
            val = xh * sc.to(dt)
            sv = sc.to(dt).abs() * (sx + xh.abs() * (sx * xh.abs()).sum(-1, keepdim=True)) / norm
            av = 16 * U * val.abs()
        else:
            val, sv, av = x, sx, 2 * U * x.abs()
        rows = p["q_rows"] if name == "q" else p["kv_rows"]
        off = 0 if name == "q" else ko
        o = torch.zeros((Bq, H, rows, 64), dtype=dt)
        so, ao = torch.zeros_like(o), torch.zeros_like(o)
        hidx = torch.arange(nh)
        if defect == "qkv_next_head":
            hidx = (hidx + 1) % H
        o[:, hidx, off:off + T] = val.transpose(1, 2)
        so[:, hidx, off:off + T] = sv.transpose(1, 2)
        ao[:, hidx, off:off + T] = av.transpose(1, 2)
        nul = p.get("null_" + name)
        if name != "q" and nul is not None and defect != "null_row_missing":
            o[:, :, 0] = nul.to(dt)
            so[:, :, 0] = 0
            ao[:, :, 0] = 0
        out[name], S[name], A[name] = o, so, ao
    return out, S, A


def coef(variant, K):
    """the accumulation coefficient of a variant name (from linear_kernels etc.) over the product's K (before any split)"""
    if variant.startswith("simt_gemm_kernel"):
        return K * U / (1 - K * U)
    if variant == "split":
        return C_ACC * math.ceil(6 * K / 16) * U + 3 * U
    return C_ACC * math.ceil(K / 16) * U


def tolerance(variant, K, ref, S, A, out_bf16):
    tol = coef(variant, K) * S + A
    return tol + 2.0 ** -8 * ref.abs() if out_bf16 else tol


def worst_ratio(got, ref, tol):
    got = got.double()
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / tol)          # positions neither side writes: 0 / 0
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------ references
def product(a, w):
    """acc = a w^T and s = |a| |w|^T in fp64"""
    ad, wd = a.double(), w.double()
    return ad @ wd.T, ad.abs() @ wd.abs().T


def linear_ref(a, w, kind, p):
    acc, s = product(a, w)
    return epilogue(kind, acc, s, p)


def conv_ref(x, wp, kind, epi_kind, p):
    """x [B, H, W, Cin] NHWC, wp packed [Cout, taps * Cin]: rows of the result are output pixels (b, y, x)"""
    acc, s = product(im2col(x, kind), wp)
    return epilogue(epi_kind, acc, s, p)


def convt_ref(x, wp, p, rgb=False):
    """x [B, H, W, Cin], wp [4, Cout, 4 Cin]: CONVT -> [B, 2H, 2W, Cout]; CONVT_RGB -> [B, ch, 2H, 2W].  Returns (out, S, A) in that layout"""
    B, H, W, _ = x.shape
    N = wp.shape[1]
    outs = []
    for py in range(2):
        for px in range(2):
            acc, s = product(convt_cols(x, py, px), wp[py * 2 + px])
            outs.append(epilogue(CONVT_RGB if rgb else CONVT, acc, s, p))
    C = outs[0][0].shape[1]
    res = []
    for i in range(3):
        full = torch.zeros((B, 2 * H, 2 * W, C), dtype=torch.float64)
        for py in range(2):
            for px in range(2):
                full[:, py::2, px::2] = outs[py * 2 + px][i].reshape(B, H, W, C)
        res.append(full.permute(0, 3, 1, 2).contiguous() if rgb else full)
    return tuple(res)


# ------------------------------------------------------------------------------------------------ the tiled product, restated
def tiled_acc(cols, w, plan, *, defect=None, conv_geom=None):
    """fp32 accumulator of the tiled product over 64-column k-blocks as tc_gemm_kernel schedules it: `plan` = (bn, n_fast).  The index
    arithmetic is restated (tile order, k-block ring, row map of a tile), the tensor core's rounding is not: each k-block is one fp32
    product.  conv_geom = (B, Ho, Wo, TW, TH, TB, tiles_x, tiles_y) maps a conv tile's 128 rows to output pixels.  Rows a tile does not
    write stay 0."""
    M, K = cols.shape
    N = w.shape[0]
    bn, nf = plan
    nkb = K // 64
    kbs = [cols[:, 64 * i:64 * i + 64].float() @ w[:, 64 * i:64 * i + 64].float().T for i in range(nkb)]
    use = list(range(nkb))
    if defect == "drop_last_kblock":
        use = use[:-1]
    if defect == "kblock_twice" and nkb > 1:
        use[-1] = nkb - 2                                 # a stale ring slot: the previous k-block read again in place of the last
    full = torch.zeros((M, N), dtype=torch.float32)
    for i in use:
        full += kbs[i]
    if conv_geom is None:
        nm = (M + 127) // 128
        rows_of = lambda m: torch.arange(m * 128, m * 128 + 128)
    else:
        B, Ho, Wo, TW, TH, TB, tx, ty = conv_geom
        nm = tx * ty * ((B + TB - 1) // TB)

        def rows_of(m):
            xt, yt, bt = m % tx, (m // tx) % ty, m // (tx * ty)
            r = torch.arange(128)
            px, py, tb = r % TW, (r // TW) % TH, r // (TW * TH)
            b = bt * TB + tb
            return (b * Ho + yt * TH + py) * Wo + xt * TW + px, b
    nn_ = (N + bn - 1) // bn
    out = torch.zeros((M, N), dtype=torch.float32)
    for t in range(nm * nn_):
        m, n = (t // nn_, t % nn_) if nf else (t % nm, t // nm)
        sm, sn = m, n                                      # the tile the producer loaded
        if defect == "tile_order_swapped" and nf:
            sm, sn = t % nm, t // nm
        cs, csrc = slice(n * bn, min(N, n * bn + bn)), slice(sn * bn, min(N, sn * bn + bn))
        if conv_geom is None:
            dst, src = rows_of(m), rows_of(sm)
            if defect == "ragged_row_off_by_one" and m == nm - 1 and M % 128:
                edge = m * 128 + (M - m * 128 - 1) // 16 * 16      # the last 16-row box of the ragged block is read one row down
                src = torch.where(dst >= edge, src + 1, src)
            ok = (dst < M) & (src < M)
            out[dst[ok], cs] = full[src[ok], csrc]
        else:
            dst, bd = rows_of(m)
            src, bs = rows_of(sm)
            if defect == "wrong_image_in_tile":
                B, Ho, Wo, TW, TH, TB, tx, ty = conv_geom
                bt = m // (tx * ty)
                tb = torch.arange(128) // (TW * TH)
                bd = bt + tb                               # the tile's image index without the TB stride
                dst = dst - (bt * TB + tb) * Ho * Wo + bd * Ho * Wo
            ok = (bd < conv_geom[0]) & (bs < conv_geom[0])
            out[dst[ok], cs] = full[src[ok], csrc]
    return out


def emulate_linear(a, w, kind, p, plan, defect=None, out_bf16=False):
    """the clean or defective restatement of one dense product: fp32 k-block accumulation, the epilogue in fp32, the output rounding"""
    acc = tiled_acc(a, w, plan, defect=defect)
    out, _, _ = epilogue(kind, acc, acc.abs(), p, torch.float32, defect)
    return _round(out, out_bf16)


def emulate_conv(x, wp, kind, epi_kind, p, plan, geom, defect=None, out_bf16=False):
    B, H, W, _ = x.shape
    Ho, Wo = conv_out_hw(kind, H, W)
    acc = tiled_acc(im2col(x, kind, defect), wp, plan, defect=defect, conv_geom=(B, Ho, Wo) + tuple(geom))
    out, _, _ = epilogue(epi_kind, acc, acc.abs(), p, torch.float32, defect)
    return _round(out, out_bf16)


def emulate_convt(x, wp, p, plan, geom, defect=None, out_bf16=False):
    B, H, W, _ = x.shape
    N = wp.shape[1]
    full = torch.zeros((B, 2 * H, 2 * W, N), dtype=torch.float32)
    for py in range(2):
        for px in range(2):
            acc = tiled_acc(convt_cols(x, py, px), wp[py * 2 + px], plan, defect=defect, conv_geom=(B, H, W) + tuple(geom))
            out, _, _ = epilogue(CONVT, acc, acc.abs(), p, torch.float32, defect)
            qy, qx = (px, py) if defect == "convt_parity_swapped" else (py, px)
            full[:, qy::2, qx::2] = out.reshape(B, H, W, N)
    return _round(full, out_bf16)


def _round(out, out_bf16):
    if isinstance(out, dict):
        return {k: _round(v, out_bf16) for k, v in out.items()}
    return bf(out) if out_bf16 else out.float()


def old_tolerance(ref, out_bf16):
    return 2e-2 + 1e-2 * ref.abs() if out_bf16 else 2e-4 + 1e-3 * ref.abs()

"""GPU tests of the HBM-bound row kernels (mmg_elementwise.cu: LayerNorm, final LayerNorm + CFG combine, GroupNorm, the first conv)
and the VQ lookups (mmg_vq.cu), instantiation by instantiation, against fp64 torch on the exact operand values.

Every case names the kernel instantiation its shape is chosen to reach and asserts, from a torch.profiler capture of the call, that
exactly that instantiation ran: a case that falls to another dispatch branch fails and lists the kernels it saw.

Tolerances (u = 2^-24, the fp32 unit roundoff):
  fp32 outputs   64 u times the row scale (max |x| * rstd for a normalisation: the fp32 mean and variance carry the rounding of sums of
                 up to 128 terms per lane plus a 5-level warp tree, relative to the largest input; sum |w x| for a convolution) + 8 u |ref|.
  bf16 outputs   the same absolute term + 2^-8 |ref|: one round-to-nearest to bf16 (2^-9 relative) with room for the fp32 error before it.
  VQ ids / codes bit-exact: dyadic operands (oracle.synth.dyadic) make every partial sum exact in fp32, in any summation order."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import synth, muse_oracle as O
from tests import util

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

U = 2.0 ** -24
BF = torch.bfloat16
F32 = torch.float32


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def MMGError():
    from muse_maskgit_pytorch_b200._lib import MMGError as E
    return E


def rnd(name, shape, std=1.0, seed=5):
    return torch.from_numpy(synth.normal(name, shape, seed, std))


def dyadic(name, shape, bits=4, span=1.0):
    return torch.from_numpy(synth.dyadic(name, shape, 5, bits=bits, span=span))


# ------------------------------------------------------------------------------------------------ which kernel ran
@pytest.fixture(scope="module", autouse=True)
def _profiler_ready():
    """one throw-away capture: the first CUPTI session of a process pays its set-up inside the capture"""
    if torch.cuda.is_available():
        kernels_of(lambda: torch.ones(8, device="cuda").sum())


CAPTURE_RETAKES = [0]              # captures taken again because they recorded fewer libmmg kernels than were launched


def kernels_of(fn):
    """Runs fn() under torch.profiler and returns (its result, the names of the libmmg kernels it launched).  fn must give the same result
    when called again (in-place operands are built inside it).  The CUPTI activity records of a capture are now and then lost, all of them
    or only some (a split3 product without its GEMM, three of the four conv-transpose launches): a capture that recorded fewer libmmg
    kernels than mmg_launch_count() rose by during it is taken again, after a pause that grows with each retake, up to five times: the
    losses come in short bursts, and three captures in a row of the same small kernel have come back empty."""
    import time
    from torch.profiler import profile, ProfilerActivity
    from muse_maskgit_pytorch_b200 import _lib
    for attempt in range(6):
        if attempt:
            time.sleep(0.05 * attempt)
        torch.cuda.synchronize()
        launched = _lib.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        launched = _lib.launch_count() - launched
        ev = [e for e in prof.key_averages() if e.self_device_time_total > 0 and "mmg::" in e.key]
        names = sorted({e.key for e in ev})
        if names and sum(e.count for e in ev) >= launched:
            break
        CAPTURE_RETAKES[0] += 1
    return out, names


def assert_ran(names, *want):
    """Every kernel in `want` (a demangled instantiation, e.g. 'layernorm_vec_kernel<__nv_bfloat16, __nv_bfloat16, 6>') ran, and nothing
    else from libmmg did."""
    missing = [w for w in want if not any(w in n for n in names)]
    extra = [n for n in names if not any(w in n for w in want)]
    assert not missing and not extra, f"expected {list(want)}; missing {missing}; libmmg kernels seen: {names}"


def check(got, ref, atol, bf16_out, what):
    """|got - ref| <= atol (+ 8 u |ref| for fp32, + 2^-8 |ref| for bf16), elementwise; ref fp64 on the CPU, atol broadcastable."""
    got = got.double().cpu()
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output at {(~torch.isfinite(got)).nonzero()[:4].tolist()}"
    tol = atol + (2.0 ** -8 if bf16_out else 8 * U) * ref.abs()
    err = (got - ref).abs()
    bad = err > tol
    if bool(bad.any()):
        idx = np.unravel_index(int((err - tol).argmax()), err.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} elements out of tolerance; worst at {tuple(int(v) for v in idx)}: got {got[idx].item():.6e} "
                             f"want {ref[idx].item():.6e} (err {err[idx].item():.3e}, tol {tol[idx].item():.3e})")


# ------------------------------------------------------------------------------------------------ LayerNorm
def edge_rows(tag, rows, width, bf16_in):
    """[rows, width] fp32 rows (bf16-representable when bf16_in): N(0.5, 2^2) with, where the row exists, the rows that break one-pass
    statistics and unguarded arithmetic mixed in: row 0 |mean| / std = 3000, row 2 = 300, row 6 = 1000, row 3 constant, row 4 +-2^55
    (squares summed over 4096 columns stay below the fp32 range)."""
    x = rnd(tag, (rows, width)) * 2 + 0.5
    z = rnd(tag + ".z", (rows, width))
    sign = torch.where(torch.from_numpy(synth.uniform(tag + ".s", (width,), 5)) < 0.5, -1.0, 1.0)
    edges = {0: -3000 + z[0], 2: 300 + z[min(2, rows - 1)], 3: torch.full((width,), 0.37), 4: sign * 2.0 ** 55, 6: 1000 + z[min(6, rows - 1)]}
    for r, v in edges.items():
        if r < rows:
            x[r] = v
    return x.to(BF).float() if bf16_in else x


def ln_ref(x, g):
    """fp64 LayerNorm (biased variance, eps 1e-5) and the per-row scale max |x| * rstd the fp32 statistics are accurate relative to"""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = (((xd - mean) ** 2).mean(-1, keepdim=True) + 1e-5).rsqrt()
    return (xd - mean) * rstd * g.double(), xd.abs().amax(-1, keepdim=True) * rstd


R2, VEC, SCALAR = "layernorm_rows2_kernel<{}>", "layernorm_vec_kernel<{}, {}, {}>", "layernorm_kernel<{}, {}>"
TN = {F32: "float", BF: "__nv_bfloat16"}
# (x dtype, y dtype, width, ldx, ldy, rows, add, instantiation): the dispatch in mmg_layernorm —
#   rows2<CH>     fp32 -> bf16, ldx == ldy == width == 128 CH, 16-byte aligned, x_out NULL or == x;
#   vec<CH>       16-byte aligned rows, ldx / ldy multiples of VN (4 fp32 / 8 bf16 input columns), width % VN == 0 with add / x_out,
#                 CH = the smallest of 4, 6, 8, 16 (32: fp32 input) with CH * 32 * VN >= max(width, ldy);
#   scalar        everything else with width <= 2048 (any ldy).
LN_CASES = [
    (F32, BF, 128, 128, 128, 77, True, R2.format(1)),
    (F32, BF, 256, 256, 256, 7, False, R2.format(2)),
    (F32, BF, 256, 256, 256, 15, True, R2.format(2)),
    (F32, BF, 512, 512, 512, 1, False, R2.format(4)),
    (F32, BF, 512, 512, 512, 15, True, R2.format(4)),
    (F32, F32, 128, 128, 128, 7, False, VEC.format("float", "float", 4)),
    (F32, F32, 512, 512, 520, 15, True, VEC.format("float", "float", 6)),
    (F32, F32, 768, 768, 768, 77, False, VEC.format("float", "float", 6)),
    (F32, F32, 1000, 1000, 1000, 15, True, VEC.format("float", "float", 8)),
    (F32, F32, 1365, 1408, 1408, 77, False, VEC.format("float", "float", 16)),
    (F32, F32, 2048, 2048, 2048, 7, True, VEC.format("float", "float", 16)),
    (F32, F32, 2730, 2752, 2752, 15, False, VEC.format("float", "float", 32)),      # the dim-1024 FeedForward's inner LayerNorm
    (F32, F32, 4096, 4096, 4096, 7, True, VEC.format("float", "float", 32)),
    (F32, BF, 128, 128, 136, 7, True, VEC.format("float", "__nv_bfloat16", 4)),
    (F32, BF, 768, 768, 768, 15, False, VEC.format("float", "__nv_bfloat16", 6)),
    (F32, BF, 512, 520, 520, 77, True, VEC.format("float", "__nv_bfloat16", 6)),
    (F32, BF, 1000, 1000, 1024, 7, False, VEC.format("float", "__nv_bfloat16", 8)),
    (F32, BF, 2048, 2048, 2048, 15, True, VEC.format("float", "__nv_bfloat16", 16)),
    (F32, BF, 4096, 4096, 4096, 7, False, VEC.format("float", "__nv_bfloat16", 32)),
    (F32, BF, 3000, 3000, 3072, 1, True, VEC.format("float", "__nv_bfloat16", 32)),
    (BF, BF, 1000, 1000, 1000, 1, False, VEC.format("__nv_bfloat16", "__nv_bfloat16", 4)),
    (BF, BF, 256, 256, 256, 7, True, VEC.format("__nv_bfloat16", "__nv_bfloat16", 4)),
    (BF, BF, 1365, 1408, 1408, 15, False, VEC.format("__nv_bfloat16", "__nv_bfloat16", 6)),
    (BF, BF, 2048, 2048, 2048, 77, True, VEC.format("__nv_bfloat16", "__nv_bfloat16", 8)),
    (BF, BF, 4096, 4096, 4096, 7, False, VEC.format("__nv_bfloat16", "__nv_bfloat16", 16)),
    (F32, F32, 1365, 1365, 1365, 15, False, SCALAR.format("float", "float")),          # ldx % 4 != 0
    (F32, F32, 1365, 1368, 1368, 77, True, SCALAR.format("float", "float")),           # width % 4 != 0 with add
    (F32, F32, 1365, 1365, 2560, 7, False, SCALAR.format("float", "float")),           # ldy past the register-held 2048 columns
    (F32, F32, 2048, 2050, 2560, 7, True, SCALAR.format("float", "float")),
    (F32, BF, 1000, 1002, 1002, 15, False, SCALAR.format("float", "__nv_bfloat16")),
    (F32, BF, 1365, 1368, 1368, 7, True, SCALAR.format("float", "__nv_bfloat16")),
    (F32, BF, 2000, 2002, 2560, 15, False, SCALAR.format("float", "__nv_bfloat16")),
    (BF, BF, 1000, 1004, 1004, 15, False, SCALAR.format("__nv_bfloat16", "__nv_bfloat16")),   # ldx % 8 != 0
    (BF, BF, 1365, 1368, 1368, 7, True, SCALAR.format("__nv_bfloat16", "__nv_bfloat16")),
    (BF, BF, 2000, 2004, 2560, 1, False, SCALAR.format("__nv_bfloat16", "__nv_bfloat16")),
]


def _ln_id(c):
    return f"{'bf16' if c[0] == BF else 'f32'}-{'bf16' if c[1] == BF else 'f32'}-w{c[2]}-ldx{c[3]}-ldy{c[4]}-r{c[5]}{'-add' if c[6] else ''}"


@pytest.mark.parametrize("case", LN_CASES, ids=[_ln_id(c) for c in LN_CASES])
def test_layernorm_variants(case):
    xdt, ydt, width, ldx, ldy, rows, with_add, want = case
    tag = _ln_id(case)
    x = edge_rows(tag, rows, width, xdt == BF)
    g = 1 + 0.1 * rnd(tag + ".g", (width,))
    xp = torch.full((rows, ldx), float("nan")); xp[:, :width] = x                   # padding columns must never be read
    add_from = 5 if rows > 5 else 0                                                  # rows 4 and 5 share a rows2 warp
    add = rnd(tag + ".a", (width,)).cuda() if with_add else None
    x_out = with_add and xdt == F32                                                  # in place, as the transformer blocks call it
    xin = x.clone()
    if with_add:
        xin[add_from:] = (x[add_from:] + add.cpu())                                  # one fp32 add, as in the kernel
    gd = g.cuda()

    def run():
        xd = xp.to(xdt).cuda()
        y = torch.full((rows, ldy), float("nan"), device="cuda", dtype=ydt)
        ops().layernorm(xd, gd, y, width=width, add=add, x_out=xd if x_out else None, add_from=add_from)
        return xd, y
    (xd, y), names = kernels_of(run)
    assert_ran(names, want)
    ref, scale = ln_ref(xin, g)
    check(y[:, :width], ref, 64 * U * scale * float(g.abs().max()), ydt == BF, want)
    nz = (y[:, width:].float() != 0).nonzero()
    assert len(nz) == 0, f"{want}: padding columns [width, ldy) must be 0; {len(nz)} are not, e.g. (row, col - width) {nz[:4].tolist()}"
    if x_out:
        got = xd[:, :width].cpu()
        assert torch.equal(got, xin), f"x_out: rows >= add_from must hold x + add, rows below it x (max diff {(got - xin).abs().max()})"


@pytest.mark.parametrize("xdt,width,ldx,ldy", [(F32, 4097, 4100, 4100), (BF, 4100, 4104, 4104), (F32, 2049, 2050, 2050),
                                               (F32, 3000, 3000, 4100), (BF, 2100, 2100, 2104)])
def test_layernorm_rejects_widths_no_kernel_takes(xdt, width, ldx, ldy):
    """past 4096 columns nothing holds the row; past 2048 only the vectorised kernels do (the scalar one keeps 2048 in registers):
    a host-side argument error, before any launch"""
    x = torch.zeros((3, ldx), device="cuda", dtype=xdt)
    y = torch.zeros((3, ldy), device="cuda", dtype=xdt)
    g = torch.ones(width, device="cuda")
    with pytest.raises(MMGError(), match="mmg_layernorm: width"):
        ops().layernorm(x, g, y, width=width)
    assert float(y.float().abs().max()) == 0.


# ------------------------------------------------------------------------------------------------ final LayerNorm + CFG combine
def _fe_nv(dim):
    return 1 if dim <= 128 else 2 if dim <= 256 else 4 if dim <= 512 else 8 if dim <= 1024 else 16


@pytest.mark.parametrize("e_dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("dim", [128, 256, 512, 1024, 2048, 200])
def test_final_embed_variants(dim, e_dtype):
    """final_embed_kernel<TE, NV>: NV float4 per lane, NV = the smallest of 1, 2, 4, 8, 16 with 128 NV >= dim (200: a ragged last
    chunk, the c + 3 < dim tail); with and without the null branch, cond_scale 1 and 3."""
    B, n, nm = 3, 16, 5
    tag = f"fe{dim}"
    xc, xn = edge_rows(tag + "c", B * n, dim, False), edge_rows(tag + "n", B * n, dim, False)
    g = 1 + 0.1 * rnd(tag + ".g", (dim,))
    gen = torch.Generator().manual_seed(dim)
    mp = torch.stack([torch.sort(torch.randperm(n, generator=gen)[:nm]).values for _ in range(B)]).int()
    mp[0, 0] = 0                                                                      # the offset row 0 is sampled
    rows = (torch.arange(B)[:, None] * n + mp.long()).reshape(-1)
    lc, sc = ln_ref(xc[rows], g)
    ln_, sn = ln_ref(xn[rows], g)
    want = f"final_embed_kernel<{TN[e_dtype]}, {_fe_nv(dim)}>"
    xcd, xnd, gd, mpd = xc.cuda(), xn.cuda(), g.cuda(), mp.cuda()
    for null, s in ((True, 3.0), (True, 1.0), (False, 3.0)):
        e = torch.full((B * nm, dim), float("nan"), device="cuda", dtype=e_dtype)
        _, names = kernels_of(lambda: ops().final_embed(xcd, xnd if null else None, gd, mpd, e, B, n, nm, s))
        assert_ran(names, want)
        ref = ln_ + (lc - ln_) * s if null else lc
        scale = (abs(s) * sc + abs(1 - s) * sn) if null else sc
        check(e, ref, 64 * U * scale * float(g.abs().max()), e_dtype == BF, f"{want} null={null} s={s}")


@pytest.mark.parametrize("e_dtype", [F32, BF], ids=["f32", "bf16"])
def test_final_embed_flat_batch(e_dtype):
    """the B = 1 form MaskGit's sampling tail uses: positions index all b * n rows of the stream at once, no null branch, scale 1"""
    b, n, dim, R = 4, 40, 512, 70
    x = edge_rows("fef", b * n, dim, False)
    g = 1 + 0.1 * rnd("fef.g", (dim,))
    pos = torch.sort(torch.randperm(b * n, generator=torch.Generator().manual_seed(7))[:R]).values.int()
    pos[0] = 0
    e = torch.full((R, dim), float("nan"), device="cuda", dtype=e_dtype)
    _, names = kernels_of(lambda: ops().final_embed(x.cuda(), None, g.cuda(), pos.cuda(), e, 1, b * n, R, 1.))
    assert_ran(names, f"final_embed_kernel<{TN[e_dtype]}, 4>")
    ref, scale = ln_ref(x[pos.long()], g)
    check(e, ref, 64 * U * scale * float(g.abs().max()), e_dtype == BF, "final_embed flat")


# ------------------------------------------------------------------------------------------------ GroupNorm
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("B,HW,C,groups", [(2, 3, 32, 32), (3, 1, 64, 16), (2, 1, 16, 16), (1, 100, 96, 32), (2, 128 * 128, 128, 16)],
                         ids=["one-channel-groups", "HW1", "HW1-one-channel", "cg3", "vae-slab"])
def test_groupnorm_variants(dtype, act, B, HW, C, groups):
    """groupnorm_kernel<T>, in place over NHWC [B, HW, C]; every (batch, group) has its own offset and scale, so statistics leaking
    between groups or batch entries would show.  A group of one element normalises to exactly beta."""
    cg = C // groups
    tag = f"gn{B}.{HW}.{C}.{groups}"
    off = (rnd(tag + ".o", (B, 1, groups, 1)) * 4).expand(B, HW, groups, cg)
    mul = torch.exp(rnd(tag + ".m", (B, 1, groups, 1)) * 0.7).expand(B, HW, groups, cg)
    x = (off + mul * rnd(tag, (B, HW, groups, cg))).reshape(B, HW, C)
    if dtype == BF:
        x = x.to(BF).float()
    g, be = 1 + 0.1 * rnd(tag + ".g", (C,)), 0.1 * rnd(tag + ".b", (C,))
    xd, names = kernels_of(lambda: ops().groupnorm_(x.to(dtype).cuda(), g.cuda(), be.cuda(), B, HW, C, groups, act=act))
    assert_ran(names, f"groupnorm_kernel<{TN[dtype]}>")
    xg = x.double().view(B, HW, groups, cg)
    mean = xg.mean((1, 3), keepdim=True)
    rstd = (((xg - mean) ** 2).mean((1, 3), keepdim=True) + 1e-5).rsqrt()
    ref = ((xg - mean) * rstd).reshape(B, HW, C) * g.double() + be.double()
    if act:
        ref = F.leaky_relu(ref, 0.1)
    scale = (xg.abs().amax((1, 3), keepdim=True) * rstd).expand(B, HW, groups, cg).reshape(B, HW, C)
    check(xd, ref, 64 * U * scale * float(g.abs().max()) + 8 * U * float(be.abs().max()), dtype == BF, f"groupnorm act={act}")


# ------------------------------------------------------------------------------------------------ first conv
CI_MAX_SMEM = 200 * 1024


def _conv_in_smem(Cout, C, ks):
    return (Cout + 8) * C * ks * ks * 4


@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("B,C,H,W,Cout,ks,bias", [(1, 3, 7, 13, 16, 1, True), (2, 4, 9, 5, 64, 3, False), (1, 1, 33, 17, 128, 5, True),
                                                  (2, 3, 12, 20, 64, 5, True), (1, 1, 11, 7, 1024, 1, False), (3, 3, 23, 29, 96, 3, True),
                                                  (2, 4, 37, 41, 253, 7, True), (1, 1, 19, 3, 40, 7, False)])
def test_conv_in_variants(dtype, B, C, H, W, Cout, ks, bias):
    """conv_in_kernel<T>: ks x ks, pad ks / 2, NCHW fp32 image -> NHWC; odd non-square images with B H W % 8 != 0, Cout past one thread per
    channel (1024), the largest Cout the 200 KB weight + patch buffer admits at 7 x 7 x 4 (253), and 2 x 37 x 41 = 380 groups of 8 pixels
    (more than the 2 x #SM persistent CTAs: the grid-stride loop runs)"""
    if (B, C, H, W, Cout, ks) == (2, 4, 37, 41, 253, 7):
        assert _conv_in_smem(Cout, C, ks) <= CI_MAX_SMEM < _conv_in_smem(Cout + 1, C, ks)
    tag = f"ci{B}.{C}.{H}.{W}.{Cout}.{ks}"
    img = torch.from_numpy(synth.uniform(tag, (B, C, H, W), 5))
    w = rnd(tag + ".w", (Cout, C, ks, ks), std=(C * ks * ks) ** -0.5)
    b = rnd(tag + ".b", (Cout,)) if bias else None
    out = torch.full((B * H * W, Cout), float("nan"), device="cuda", dtype=dtype)
    _, names = kernels_of(lambda: ops().conv_in(img.cuda(), w.cuda(), None if b is None else b.cuda(), out, ksize=ks))
    assert_ran(names, f"conv_in_kernel<{TN[dtype]}>")
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(-1, Cout)
    ref = nhwc(F.conv2d(img.double(), w.double(), None if b is None else b.double(), padding=ks // 2))
    mag = nhwc(F.conv2d(img.double().abs(), w.double().abs(), None if b is None else b.double().abs(), padding=ks // 2))
    check(out, ref, 64 * U * mag, dtype == BF, f"conv_in ks={ks}")


def test_conv_in_rejects_cout_past_shared_memory():
    img = torch.zeros((1, 4, 8, 8), device="cuda")
    w = torch.zeros((254, 4, 7, 7), device="cuda")
    out = torch.zeros((64, 254), device="cuda")
    with pytest.raises(MMGError(), match="shared memory"):
        ops().conv_in(img, w, None, out, ksize=7)


# ------------------------------------------------------------------------------------------------ LFQ encode
def lfq_ref(x, w, b, bits):
    proj = x.double() if w is None else x.double() @ w.double().t() + (0 if b is None else b.double())
    return ((proj > 0).long() * (2 ** torch.arange(bits - 1, -1, -1))).sum(-1)


def split3_rows(w):
    """[hi | mid | lo] bf16 rows of w padded to 64 (the w_split operand of mmg_vq_lfq_encode; longer when 3 * bits > 64, where the
    launcher does not use it)"""
    hi = w.to(BF); r1 = w - hi.float(); mid = r1.to(BF); lo = (r1 - mid.float()).to(BF)
    assert torch.equal(hi.float() + mid.float() + lo.float(), w) and bool((mid != 0).any())
    bits, D = w.shape
    w3 = torch.zeros((max(64, 3 * bits), D), dtype=BF)
    w3[:bits], w3[bits:2 * bits], w3[2 * bits:3 * bits] = hi, mid, lo
    return w3


LFQ_CASES = [   # (T, D, bits, projection, bias, instantiation ('{}' = token type))
    (300, 512, 12, True, True, "lfq_encode_kernel<{}, 16>"),
    (333, 256, 16, True, False, "lfq_encode_kernel<{}, 16>"),
    (301, 384, 17, True, True, "lfq_encode_kernel<{}, 24>"),
    (129, 2048, 24, True, True, "lfq_encode_kernel<{}, 24>"),
    (77, 96, 12, True, True, "lfq_encode_generic_kernel<{}, 24>"),
    (50, 200, 24, True, False, "lfq_encode_generic_kernel<{}, 24>"),
    (64, 13, 13, False, False, "lfq_encode_generic_kernel<{}, 24>"),
    (33, 24, 24, False, False, "lfq_encode_generic_kernel<{}, 24>"),
]


@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("T,D,bits,proj,bias,want", LFQ_CASES, ids=[f"T{c[0]}-D{c[1]}-b{c[2]}{'' if c[3] else '-identity'}" for c in LFQ_CASES])
def test_vq_lfq_encode_variants(dtype, T, D, bits, proj, bias, want):
    """CUDA-core LFQ lookup: the fast kernel (D % 128 == 0, a projection) at bits <= 16 and 17..24, the generic kernel for other D and for
    the identity projection; some tokens and projected values exactly 0 (bit 0)"""
    tag = f"lfq{T}.{D}.{bits}"
    x = dyadic(tag, (T, D), bits=4, span=2.0)
    x[T // 2] = 0.
    w = dyadic(tag + ".w", (bits, D)) if proj else None
    b = dyadic(tag + ".b", (bits,)) if bias else None
    ids = torch.full((T,), -1, dtype=torch.int64, device="cuda")
    _, names = kernels_of(lambda: ops().vq_lfq_encode(x.to(dtype).cuda(), None if w is None else w.cuda(), None if b is None else b.cuda(), ids, bits))
    assert_ran(names, want.format(TN[dtype]))
    assert torch.equal(ids.cpu(), lfq_ref(x, w, b, bits))


@pytest.mark.parametrize("T,bits,route", [(1000, 21, "wgmma"), (130, 8, "wgmma"), (1000, 22, "cuda-core"), (777, 21, "fp32-tokens")])
def test_vq_lfq_encode_w_split_route(T, bits, route):
    """bf16 tokens with the 3-way split of project_in take the wgmma route (LFQ_IDS epilogue) while 3 * bits <= 64; past that, or with
    fp32 tokens, the CUDA-core kernel ignores the split.  T ragged against the 128-row tiles.  The split really has a mid term (w carries
    bits below bf16's 8), and every partial sum is exact in fp32: x on a 2^-3 grid in [-1, 1), w on 2^-12, |x.w| < 2^8."""
    D = 256
    tag = f"lfqs{T}.{bits}"
    x = dyadic(tag, (T, D), bits=3, span=1.0)
    w = dyadic(tag + ".w", (bits, D)) + dyadic(tag + ".w2", (bits, D)) * 2.0 ** -8
    b = dyadic(tag + ".b", (bits,))
    dtype = F32 if route == "fp32-tokens" else BF
    ids = torch.full((T,), -1, dtype=torch.int64, device="cuda")
    _, names = kernels_of(lambda: ops().vq_lfq_encode(x.to(dtype).cuda(), w.cuda(), b.cuda(), ids, bits, w_split=split3_rows(w).cuda()))
    if route == "wgmma":
        assert_ran(names, "tc_gemm_kernel<")
    else:
        assert_ran(names, f"lfq_encode_kernel<{TN[dtype]}, 24>")
    assert torch.equal(ids.cpu(), lfq_ref(x, w, b, bits))


# ------------------------------------------------------------------------------------------------ LFQ decode (ids -> codes)
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
@pytest.mark.parametrize("T,D,bits,proj", [(100, 13, 13, False), (64, 24, 24, False), (130, 255, 24, True), (100, 600, 16, True),
                                           (65, 512, 9, True), (1, 1027, 1, True)])
def test_vq_decode_codes_variants(dtype, T, D, bits, proj):
    """vq_decode_codes_kernel<T>: identity projection (odd D == bits), bits = 24, odd D (unaligned pairs for bf16 stores), D > 512 (more
    than one grid column), T not a multiple of 64; dyadic weights make fp32 outputs exact and bf16 ones a single rounding of it"""
    tag = f"dec{T}.{D}.{bits}"
    ids = torch.from_numpy((synth.uniform(tag, (T,), 5) * 2 ** bits).astype(np.int64))
    ids[0] = 2 ** bits - 1
    w = dyadic(tag + ".w", (D, bits)) if proj else None
    b = dyadic(tag + ".b", (D,)) if proj else None
    out = torch.full((T, D), float("nan"), device="cuda", dtype=dtype)
    _, names = kernels_of(lambda: ops().vq_decode_codes(ids.cuda(), None if w is None else w.cuda(), None if b is None else b.cuda(), out, bits))
    assert_ran(names, f"vq_decode_codes_kernel<{TN[dtype]}>")
    codes = ((ids[:, None] >> torch.arange(bits - 1, -1, -1)) & 1).double() * 2 - 1
    ref = codes if w is None else codes @ w.double().t() + b.double()
    assert torch.equal(out.cpu(), ref.to(dtype)), f"max diff {(out.double().cpu() - ref).abs().max()}"


# ------------------------------------------------------------------------------------------------ explicit codebook
@pytest.mark.parametrize("T,K,D,dups", [(130, 40, 37, ((30, 5),)), (77, 200, 37, ((150, 10), (199, 64))), (300, 777, 96, ((700, 33), (401, 400))),
                                        (64, 64, 16, ((63, 0),)), (5, 1, 3, ())])
def test_vq_l2_argmin_variants(T, K, D, dups):
    """64 tokens x 64 codes per CTA, D staged 16 channels at a time: K < 64, K and D off the tiles, ragged T.  Each (dup, orig) pair is
    an exact duplicate code in another 64-code tile and some tokens equal it: the lower index must win the tie."""
    tag = f"l2{T}.{K}.{D}"
    x = dyadic(tag, (T, D), bits=3, span=2.0)
    cb = dyadic(tag + ".cb", (K, D), bits=3, span=2.0)
    for i, (dup, orig) in enumerate(dups):
        cb[dup] = cb[orig]
        x[i::7] = cb[orig]
    ids = torch.full((T,), -1, dtype=torch.int64, device="cuda")
    _, names = kernels_of(lambda: ops().vq_l2_argmin(x.cuda(), cb.cuda(), ids))
    assert_ran(names, "vq_init_kernel", "vq_l2_argmin_kernel", "vq_finish_kernel")
    d = (cb.double() ** 2).sum(-1)[None] - 2 * x.double() @ cb.double().t()
    ref = d.argmin(-1)                                                               # first index of the minimum
    assert torch.equal(ids.cpu(), ref), f"tokens {(ids.cpu() != ref).nonzero().flatten()[:8].tolist()}: got {ids.cpu()[ids.cpu() != ref][:8].tolist()}"
    for i, (dup, orig) in enumerate(dups):
        assert bool((ids.cpu()[i::7] == min(dup, orig)).all())


# ------------------------------------------------------------------------------------------------ where users meet the width limit
def test_transformer_dim1024_fp32_forward_vs_oracle():
    """precision="fp32" does not fold the FeedForward's inner LayerNorm into the GEMMs: at dim 1024 it normalises rows of
    F = int(1024 * 8 / 3) = 2730 columns (ld 2752), on layernorm_vec_kernel<float, float, 32>"""
    import muse_maskgit_pytorch_b200 as m
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    V, dim, n, heads = 256, 1024, 64, 16
    tr = m.MaskGitTransformer(num_tokens=V, dim=dim, seq_len=n, depth=1, heads=heads, t5_name="synth-128", precision="fp32")
    sd = util.transformer_sd(V, dim, n, 1, heads, seed=31, text_dim=128)
    full = tr.state_dict(); full.update(sd); tr.load_state_dict(full); tr.cuda()
    te = util.text_embeds("d1024.te", 2, 8, 128, 31)
    ids = torch.from_numpy((synth.uniform("d1024.ids", (2, n), 31) * (V + 1)).astype(np.int64))
    ref, ref_embed = O.forward_with_cond_scale(sd, dict(heads=heads, depth=1), ids, te, cond_scale=3.)
    (got, embed), names = kernels_of(lambda: tr.forward_with_cond_scale(ids.cuda(), text_embeds=te.cuda(), cond_scale=3., return_embed=True))
    assert any("layernorm_vec_kernel<float, float, 32>" in k for k in names), names
    e_err = float((embed.cpu().double() - ref_embed.double()).abs().max())
    l_err = float((got.cpu().double() - ref.double()).abs().max())
    print(f"dim 1024 fp32: embed max |err| {e_err:.3e}, CFG logits max |err| {l_err:.3e} (max |logit| {float(ref.abs().max()):.3e})")
    assert e_err < 5e-5 and l_err < 2e-4 * max(1.0, float(ref.abs().max()))

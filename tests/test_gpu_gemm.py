"""GPU tests of mmg_linear, mmg_conv2d and mmg_conv_transpose2d, variant by variant, against the fp64 references and derived tolerances of
tests/gemm_oracle.py.

Behind the three entry points sit twelve bf16 instantiations of tc_gemm_kernel<BN, EPI_MODE> and six of simt_gemm_kernel<T, CONV, ACT>.
Every case names the kernels the restated dispatch (gemm_oracle.linear_kernels / conv_kernels / convt_kernels, at this card's SM count)
says its arguments reach, checks every element against fp64 within the bound, writes into a buffer whose rows past M and columns past N
hold a guard value that must survive, and checks how mmg_simt_launch_count() and mmg_simt_fallback_count() moved.  Which kernels ran is
asserted from torch.profiler captures taken in a child process (test_every_case_reached_its_kernel runs this file again with
MMG_GEMM_PROFILE=1), as in tests/test_gpu_attention.py.  The last test prints the case count and worst |err| / tol per variant."""
import os
import subprocess
import sys

import pytest
import torch

from tests import gemm_oracle as G
from tests.test_gpu_row_kernels import kernels_of, assert_ran

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

BF, F32 = torch.bfloat16, torch.float32
FILL = -77.0
STATS = {}                         # variant -> [cases, worst err / tol]
PROFILE = os.environ.get("MMG_GEMM_PROFILE") == "1"


def L():
    from muse_maskgit_pytorch_b200 import _lib
    return _lib


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module", autouse=True)
def _warm_up():
    if PROFILE and torch.cuda.is_available():
        kernels_of(lambda: torch.ones(8, device="cuda").sum())


def observed(fn, want):
    """fn() with the rise of the CUDA-core counters checked against the CUDA-core launches in `want` (+1 per launch; the fallback counter +1
    for a bf16 call); in the profiling process, where a capture may run fn again, only that exactly the kernels in `want` ran"""
    if PROFILE:
        out, names = kernels_of(fn)
        assert_ran(names, *set(want))
        return out
    s0, f0 = L().simt_launch_count(), L().simt_fallback_count()
    out = fn()
    torch.cuda.synchronize()
    simt = [n for n in want if n.startswith("simt")]
    fb = int(any("__nv_bfloat16" in n for n in simt))
    assert L().simt_launch_count() - s0 == len(simt), f"{want}: CUDA-core launches moved by {L().simt_launch_count() - s0}"
    assert L().simt_fallback_count() - f0 == fb, f"{want}: fallback counter moved by {L().simt_fallback_count() - f0}"
    return out


ORDER = {"n": 1, "m": 0}            # a case label's tile order -> n_fast


def stat_key(variant, nf):
    """STATS key: a tensor-core variant with the tile order it ran in"""
    if variant.startswith("tc_gemm_kernel") and nf is not None:
        return f"{variant} {'n-fast' if nf else 'm-fast'}"
    return variant


def record(variant, got, ref, tol, what, nf=None):
    r = G.worst_ratio(got, ref, tol)
    st = STATS.setdefault(stat_key(variant, nf), [0, 0.0])
    st[0] += 1; st[1] = max(st[1], r)
    if r > 1.0:
        got = got.double()
        err = torch.where((got - ref).abs() == 0, torch.zeros_like(ref), (got - ref).abs() / tol)
        idx = tuple(int(i) for i in (err == err.max()).nonzero()[0])
        raise AssertionError(f"{variant} {what}: worst err / tol {r:.3g} at {idx}: got {float(got[idx]):.6e} want {float(ref[idx]):.6e}; "
                             f"{int((err > 1).sum())} elements out of tolerance")
    return r


def main_variant(want, split):
    return "split" if split else want[-1]


def dev_matrix(t, dtype, ld, off=0):
    """t [rows, cols] -> a device [rows, ld] view (columns past cols zero) starting `off` elements into its allocation"""
    rows, cols = t.shape
    buf = torch.zeros(rows * ld + off + 64, dtype=dtype, device="cuda")
    v = buf[off:off + rows * ld].view(rows, ld)
    v[:, :cols] = t.to(dtype).cuda()
    return v


def guard_buf(rows, cols, dtype, off=0):
    buf = torch.full((rows * cols + off + 64,), FILL, dtype=dtype, device="cuda")
    return buf, buf[off:off + rows * cols].view(rows, cols)


def assert_guard(buf, view, written):
    """every element of buf outside view[written] still holds FILL"""
    keep = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    mark = torch.zeros(view.shape, dtype=torch.bool, device="cuda")
    mark[written] = True
    off = view.storage_offset() - buf.storage_offset()
    keep[off:off + view.numel()] = ~mark.reshape(-1)
    assert bool((buf[keep] == FILL).all()), "the guard around the output was written"


# ------------------------------------------------------------------------------------------------ dense products
HALF = (G.GEGLU, G.GLU, G.GEGLU_TANH)


def run_linear(tag, M, N, K, kind=G.STORE, *, dtype="bf16", out="f32", bias=False, act=0, resid=None, ldo_pad=0, lda_pad=0, ldw_pad=0,
               a_off=0, w_off=0, out_off=0, split=False, stats_slots=0, want=None, order=None, expect=None):
    """one mmg_linear call on probe operands.  resid: None, 'oop' (own buffer) or 'inplace' (out is resid).  split: fp32 through
    ops.linear (mmg_split3 + the bf16 kernel).  stats_slots: GEGLU row_stats slots (LNFOLD: the statistics are inputs).  order: the tile
    order ('n' or 'm' fastest) the case is built for, and expect: the kernels it is built for, both asserted against the restated dispatch;
    want: the kernels, where the dispatch depends on state the oracle does not see (fp32_tc)."""
    a, w = G.probe_dense(tag, M, N, K, bf16=dtype == "bf16")
    tdt = BF if dtype == "bf16" else F32
    odt = BF if out == "bf16" else F32
    p = {"act": act, "approx": out == "bf16"}
    if bias or kind in (G.LNFOLD, G.GLU):
        p["bias"] = G.rnd(tag + ".b", (N,))
    Nout = N // 2 if kind in HALF else N
    lda, ldw, ldo = K + lda_pad, K + ldw_pad, Nout + ldo_pad
    e = {"out": out, "act": act, "bias": "bias" in p, "in_place": resid == "inplace", "ldo": ldo,
         "out_aligned": (out_off * (2 if out == "bf16" else 4)) % 16 == 0}
    nf = None
    if want is None:
        want, nf = G.linear_kernels(M, N, K, kind, e, dtype=dtype, sms=sms(), lda=lda, ldw=ldw, a_aligned=(a_off * 2) % 16 == 0 or dtype == "f32",
                                    w_aligned=(w_off * 2) % 16 == 0 or dtype == "f32", split=split, order=True)
    assert expect is None or want == expect, (want, expect)
    assert order is None or nf == ORDER[order], f"built for {order}-fast tiles, the dispatch gives n_fast = {nf}"
    buf, o = guard_buf(M + 3, ldo, odt, out_off)
    r_dev = None
    if kind in (G.RESIDUAL, G.LNFOLD):
        rv = G.rnd(tag + ".r", (M, N))
        rv = G.bf(rv) if out == "bf16" else rv
        p["resid"] = rv
        if resid == "inplace":
            r_dev = o
        else:
            r_dev = torch.full((M + 1, ldo), FILL, dtype=odt, device="cuda"); r_dev[:M, :N] = rv.to(odt).cuda()
    st_dev = None
    if kind == G.LNFOLD:
        h = G.rnd(tag + ".h", (M, 256)) * 0.8 + 0.3
        st = torch.stack([h.reshape(M, 4, 64).sum(-1), (h * h).reshape(M, 4, 64).sum(-1)], -1)
        p.update(stats=st, ln_width=256)
        st_dev = st.cuda().contiguous()
    if kind == G.GEGLU and stats_slots:
        st_dev = torch.full((M, stats_slots, 2), FILL, dtype=F32, device="cuda")
    bias_dev = p["bias"].cuda() if "bias" in p else None
    r_in = p["resid"].to(odt).cuda() if resid == "inplace" else None

    def reset():                                     # an in-place call starts from the residual every time (a capture may repeat it)
        if r_in is not None:
            o[:M, :N] = r_in
    if split:
        a_d, w_d = a.cuda(), w.cuda()
        call = lambda: ops().linear(a_d, w_d, o[:M], epilogue=kind, bias=bias_dev, act=act, resid=None if r_dev is None else r_dev[:M],
                                   row_stats=st_dev, ln_width=p.get("ln_width", 0))
    else:
        a_d, w_d = dev_matrix(a, tdt, lda, a_off), dev_matrix(w, tdt, ldw, w_off)
        args = L().LinearArgs()
        args.a, args.w = a_d.data_ptr(), w_d.data_ptr()
        args.M, args.N, args.K, args.lda, args.ldw = M, N, K, lda, ldw
        args.dtype, args.epilogue = (L().BF16 if dtype == "bf16" else L().F32), kind
        args.epi = ops()._epi(o, ldo, bias_dev, act, r_dev, ldo if r_dev is not None else 0, st_dev, p.get("ln_width", 0))
        call = lambda: L().call("mmg_linear", args)
    observed(lambda: (reset(), call()), want)
    ref, S, A = G.linear_ref(a, w, kind, p)
    got = o[:M, :Nout].cpu()
    variant = main_variant(want, split)
    record(variant, got, ref, G.tolerance(variant, K, ref, S, A, out == "bf16"), tag, nf)
    assert_guard(buf, o, (slice(0, M), slice(0, Nout)))
    if kind == G.GEGLU and stats_slots:
        sv = st_dev.cpu()
        o32 = got.double().reshape(M, N // 64, 32)
        want_st = torch.stack([o32.sum(-1), (o32 * o32).sum(-1)], -1)
        bound = 32 * G.U * torch.stack([o32.abs().sum(-1), (o32 * o32).sum(-1)], -1) + 1e-30   # 32-term fp32 sums
        assert bool(((sv[:, :N // 64].double() - want_st).abs() <= bound).all()), "GEGLU row statistics"
        assert bool((sv[:, N // 64:] == FILL).all())
    return got


# Tile orders: N-fastest while N * K * 2 <= 8 MiB and there are 2..16 column tiles, M-fastest otherwise.  The M-fast shapes below have 17
# or 18 column tiles: N = 1088 at BN = 64, 2176 at 128, 4352 (M = 2048, so that BN = 256 is chosen) at 256.
# REGS at 64 and 128, both tile orders, a ragged last row block; STORE with bias and leaky, fp32 and bf16 out
@pytest.mark.parametrize("out", ["f32", "bf16"])
@pytest.mark.parametrize("M,N,K,order", [(300, 192, 192, "n"), (300, 1088, 64, "m"), (130, 1024, 128, "n"), (300, 2176, 64, "m"),
                                         (300, 256, 4160, "n")],
                         ids=["bn64-nfast", "bn64-mfast", "bn128-nfast", "bn128-mfast", "bn64-nfast-longK"])
def test_store_bias_leaky(M, N, K, order, out):
    run_linear(f"store{M}.{N}.{K}", M, N, K, bias=True, act=1, out=out, order=order)


@pytest.mark.parametrize("M,N,K,order", [(300, 192, 128, "n"), (300, 1088, 128, "m"), (300, 1024, 64, "n"), (300, 2176, 64, "m"),
                                         (8400, 1024, 64, "n"), (2048, 4352, 64, "m")],
                         ids=["bn64-nfast", "bn64-mfast", "bn128-nfast", "bn128-mfast", "bn256-nfast", "bn256-mfast"])
def test_residual_in_place_reduce(M, N, K, order):
    bn = {192: 64, 1088: 64, 1024: 128 if M == 300 else 256, 2176: 128, 4352: 256}[N]
    run_linear(f"red{M}.{N}", M, N, K, G.RESIDUAL, bias=True, resid="inplace", order=order, expect=[G.TC(bn, G.M_REDUCE)])


@pytest.mark.parametrize("M,N,K,order", [(300, 1024, 64, "n"), (300, 2176, 64, "m"), (8400, 1024, 64, "n"), (2048, 4352, 64, "m")],
                         ids=["bn128-nfast", "bn128-mfast", "bn256-nfast", "bn256-mfast"])
def test_plain_fp32_tile_store(M, N, K, order):
    bn = 128 if M == 300 else 256
    run_linear(f"tst{M}.{N}", M, N, K, ldo_pad=32, order=order, expect=[G.TC(bn, G.M_TSTORE)])


@pytest.mark.parametrize("route", ["oop-bn64", "oop-bn128", "oop-lowered-256", "bf16", "act", "inplace-ldo4", "inplace-misaligned"])
def test_residual_register_routes(route):
    """out != resid (the prefetch route, with the next chunk's residual fetched early: every register-epilogue RESIDUAL runs at BN <= 128,
    since plan_tc lowers BN = 256 to 128 for all but CONVT_RGB), bf16 RESIDUAL, RESIDUAL with act, and in place where the TMA reduction
    does not take it: ldo % 8 != 0 (which also takes bf16 operands to the CUDA cores) and an `out` 8 bytes off a 16-byte boundary, which
    reaches the register epilogue in place with its residual read and its output written element by element"""
    M, N = {"oop-bn128": (300, 1024), "oop-lowered-256": (8400, 1024)}.get(route, (300, 192))
    kw = {"oop-bn64": dict(resid="oop"), "oop-bn128": dict(resid="oop"), "oop-lowered-256": dict(resid="oop", expect=[G.TC(128, G.M_REGS)]),
          "bf16": dict(resid="oop", out="bf16"), "act": dict(resid="inplace", act=1),
          "inplace-ldo4": dict(resid="inplace", ldo_pad=4, expect=[G.SIMT("bf16", False, False)]),
          "inplace-misaligned": dict(resid="inplace", out_off=2, expect=[G.TC(64, G.M_REGS)])}[route]
    run_linear(f"res.{route}", M, N, 128, G.RESIDUAL, bias=True, **kw)


@pytest.mark.parametrize("case", ["store-f32", "store-bf16", "geglu-bf16", "geglu-f32", "act-bf16"])
def test_output_off_a_16_byte_boundary(case):
    """an `out` 8 bytes past a 16-byte boundary with ldo % 8 == 0: the register epilogues write it element by element instead of with
    16-byte vector stores"""
    kind, out, N = {"store-f32": (G.STORE, "f32", 192), "store-bf16": (G.STORE, "bf16", 192), "geglu-bf16": (G.GEGLU, "bf16", 256),
                    "geglu-f32": (G.GEGLU, "f32", 256), "act-bf16": (G.GEGLU_TANH, "bf16", 256)}[case]
    off = 4 if out == "bf16" else 2
    run_linear(f"mis.{case}", 300, N, 128, kind, out=out, bias=kind == G.STORE, act=1 if kind == G.STORE else 0, out_off=off,
               expect=[G.TC(128, G.M_ACT)] if kind == G.GEGLU_TANH else [G.TC(64, G.M_REGS)])


@pytest.mark.parametrize("M,N", [(300, 192), (8400, 1024)], ids=["bn64", "bn128"])
def test_lnfold_out_of_place(M, N):
    run_linear(f"ln{M}", M, N, 128, G.LNFOLD, resid="oop")


@pytest.mark.parametrize("M,N", [(300, 192), (300, 1024)], ids=["bn64", "bn128"])
def test_lnfold_in_place(M, N):
    run_linear(f"lni{M}.{N}", M, N, 128, G.LNFOLD, resid="inplace")


@pytest.mark.parametrize("stats", [0, 1], ids=["nostats", "stats"])
@pytest.mark.parametrize("out", ["f32", "bf16"])
@pytest.mark.parametrize("M,N", [(300, 192), (300, 1024), (8400, 1024), (2048, 4352)], ids=["bn64", "bn128", "bn256-nfast", "bn256-mfast"])
def test_geglu(M, N, out, stats):
    order = "m" if N == 4352 else "n"
    run_linear(f"geglu{M}.{N}", M, N, 64 if N == 4352 else 128, G.GEGLU, out=out, stats_slots=N // 64 + 1 if stats else 0, order=order)


@pytest.mark.parametrize("N", [192, 1024])
def test_glu_with_bias(N):
    run_linear(f"glu{N}", 300, N, 128, G.GLU, out="bf16")


@pytest.mark.parametrize("out", ["f32", "bf16"])
@pytest.mark.parametrize("N", [192, 256, 2176])
@pytest.mark.parametrize("kind", ["relu", "geglu_tanh"])
def test_act_epilogues(kind, N, out):
    """TC_EPI_ACT at N % 128 == 64 (half-empty last tile) and == 0, N-fast and (17 column tiles) M-fast, bf16 and through split3"""
    k = G.STORE if kind == "relu" else G.GEGLU_TANH
    run_linear(f"act.{kind}{N}", 300, N, 128, k, out=out, act=2 if kind == "relu" else 0, bias=kind == "relu", order="m" if N == 2176 else "n")
    run_linear(f"act.s.{kind}{N}", 300, N, 128, k, out=out, dtype="f32", split=True, act=2 if kind == "relu" else 0, bias=kind == "relu")


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("kind", ["relu", "geglu_tanh"])
def test_act_on_cuda_cores(kind, dtype):
    """simt_gemm_kernel<T, false, true>: bf16 through K % 64 != 0, fp32 with fp32_tc(False)"""
    k = G.STORE if kind == "relu" else G.GEGLU_TANH
    run_linear(f"actcc.{kind}", 200, 192, 96, k, dtype=dtype, out="f32", act=2 if kind == "relu" else 0, bias=kind == "relu")


# ------------------------------------------------------------------------------------------------ QKV
def run_qkv(tag, Bq, T, heads, *, out="bf16", nq=True, key_off=1, null=True, split=False, order=None):
    M, K = Bq * T, 128
    nqh = heads if nq else 0
    N = (nqh + 2 * heads) * 64
    a, w = G.probe_dense(tag, M, N, K, bf16=not split)
    odt = BF if out == "bf16" else F32
    p = {"heads": heads, "tokens": T, "key_off": key_off, "q_rows": T + 1, "kv_rows": key_off + T + 2, "nq": nqh, "nk": heads,
         "q_scale": 1 + 0.1 * G.rnd(tag + ".qs", (64,)), "k_scale": 1 + 0.1 * G.rnd(tag + ".ks", (64,))}
    if null:
        p["null_k"], p["null_v"] = G.bf(G.rnd(tag + ".nk", (heads, 64))), G.bf(G.rnd(tag + ".nv", (heads, 64)))
    bufs = {n: torch.full((Bq * heads, p["q_rows"] if n == "q" else p["kv_rows"], 64), FILL, dtype=odt, device="cuda") for n in "qkv"}
    d = lambda t: t.cuda().to(odt) if t is not None else None
    qs, ks = p["q_scale"].cuda(), p["k_scale"].cuda()
    nk_d, nv_d = d(p.get("null_k")), d(p.get("null_v"))          # held until the launch: the epilogue block keeps raw pointers
    e = ops().qkv_epilogue(odt, heads, T, q=bufs["q"] if nq else None, k=bufs["k"], v=bufs["v"], q_scale=qs, k_scale=ks, key_off=key_off,
                           null_k=nk_d, null_v=nv_d)
    if not nq:
        e.nq_heads = 0
    want, nf = G.linear_kernels(M, N, K, G.QKV, {"out": out, "tokens": T, "nk": heads, "nv": heads}, dtype="f32" if split else "bf16",
                                sms=sms(), split=split, order=True)
    assert order is None or nf == ORDER[order], f"built for {order}-fast tiles, the dispatch gives n_fast = {nf}"
    tdt = F32 if split else BF
    a_d, w_d = a.to(tdt).cuda(), w.to(tdt).cuda()
    observed(lambda: ops().linear(a_d, w_d, None, epilogue=G.QKV, epi=e), want)
    ref, S, A = G.linear_ref(a, w, G.QKV, p)
    variant = main_variant(want, split)
    for n in ("q", "k", "v") if nq else ("k", "v"):
        got = bufs[n].cpu().view(Bq, heads, -1, 64)
        written = torch.zeros(got.shape, dtype=torch.bool)
        off = 0 if n == "q" else key_off
        written[:, :, off:off + T] = True
        if n != "q" and null:
            written[:, :, 0] = True
        assert bool((got[~written] == FILL).all()), f"{n}: rows outside the head layout were written"
        g = torch.where(written, got.double(), ref[n])
        record(variant, g, ref[n], G.tolerance(variant, K, ref[n], S[n], A[n], out == "bf16") + (~written).double(), f"{tag} {n}", nf)
    if not nq:
        assert bool((bufs["q"] == FILL).all())


@pytest.mark.parametrize("case", ["tiles128", "tiles128-mfast", "tiles128-noq", "regs64", "regs128-tok48", "tiles256", "tiles256-mfast", "f32", "split"])
def test_qkv(case):
    """the tile epilogue at 128 and 256 in both tile orders (and with nq_heads == 0: the context K / V projection), the register epilogue
    at 64 (heads == 1) and at 128 with tokens % 32 != 0, fp32 out, and fp32 through split3"""
    kw = {"tiles128": (32, 64, 4, {"order": "n"}), "tiles128-mfast": (2, 64, 12, {"order": "m"}), "tiles128-noq": (48, 64, 4, {"nq": False}),
          "regs64": (3, 50, 1, {}), "regs128-tok48": (43, 48, 4, {}), "tiles256": (88, 64, 8, {"order": "n"}),
          "tiles256-mfast": (30, 64, 24, {"order": "m"}), "f32": (3, 50, 2, {"out": "f32"}), "split": (3, 50, 2, {"out": "f32", "split": True})}[case]
    run_qkv(f"qkv.{case}", kw[0], kw[1], kw[2], **kw[3])


# ------------------------------------------------------------------------------------------------ LFQ ids and argmin (bit-exact)
@pytest.mark.parametrize("dtype", ["bf16", "f32"])
def test_lfq_ids(dtype):
    M, K, bits = 300, 128, 10
    a = G.rnd("lfq.a", (M, K))
    a = torch.sign(a) * (0.25 + a.abs().clamp(max=1.5))
    w = G.rnd("lfq.w", (64, K), 2.0 ** -10)
    for i in range(bits):
        w[i, (i * 11) % K] += 1.0
        w[bits + i, (i * 11) % K] += 2.0 ** -9
        w[2 * bits + i, (i * 11 + 3) % K] += 2.0 ** -12
    a, w = G.bf(a), G.bf(w)
    bias = G.rnd("lfq.b", (bits,), 0.01)
    acc = a.double() @ w.double().T
    v = acc[:, :bits] + acc[:, bits:2 * bits] + acc[:, 2 * bits:3 * bits] + bias.double()
    assert float(v.abs().min()) > 0.05                  # far from the sign boundary: the ids are exact
    want_ids = ((v > 0).long() << torch.arange(bits - 1, -1, -1)).sum(1)
    out = torch.full((M + 2,), -5, dtype=torch.int64, device="cuda")
    args = L().LinearArgs()
    tdt = BF if dtype == "bf16" else F32
    a_d, w_d, b_d = a.to(tdt).cuda(), w.to(tdt).cuda(), bias.cuda()
    args.a, args.w, args.M, args.N, args.K, args.lda, args.ldw = a_d.data_ptr(), w_d.data_ptr(), M, 64, K, K, K
    args.dtype, args.epilogue = (L().BF16 if dtype == "bf16" else L().F32), G.LFQ_IDS
    e = L().EpilogueArgs(); e.out = out.data_ptr(); e.ldo = 1; e.out_dtype = L().F32; e.bias = b_d.data_ptr(); e.ln_width = bits
    args.epi = e
    want = G.linear_kernels(M, 64, K, G.LFQ_IDS, {"ldo": 1}, dtype=dtype, sms=sms())
    observed(lambda: L().call("mmg_linear", args), want)
    got = out.cpu()
    assert torch.equal(got[:M], want_ids) and bool((got[M:] == -5).all())
    STATS.setdefault(want[-1] + " (LFQ ids, exact)", [0, 0.0])[0] += 1


@pytest.mark.parametrize("N,dtype", [(256, "bf16"), (1024, "bf16"), (200, "bf16"), (256, "f32")], ids=["n256", "n1024", "n200-cc", "f32"])
def test_argmin(N, dtype):
    """nearest code with tied codes across a 64-column chunk (40 / 100) and across column tiles (10 / N - 20): the lowest index wins"""
    M, D = 300, 64
    cb = G.bf(G.rnd(f"am{N}.cb", (N, D)))
    cb[100] = cb[40]; cb[N - 20] = cb[10]
    norms = (cb.double() ** 2).sum(1).float()
    target = (torch.arange(M) * 37) % N
    target[::3] = 100; target[1::3] = N - 20
    x = G.bf(cb[target] + G.rnd(f"am{N}.x", (M, D), 0.05))
    d = norms.double()[None] - 2 * x.double() @ cb.double().T
    srt = d.sort(1).values
    want_ids = torch.tensor([int((d[r] == d[r].min()).nonzero()[0]) for r in range(M)])
    gap = (srt[:, 1] - srt[:, 0]).clone()
    tied = (want_ids == 40) | (want_ids == 10)
    gap[tied] = srt[tied, 2] - srt[tied, 0]
    assert float(gap.min()) > 1.0
    out = torch.full((M + 2,), -1, dtype=torch.int64, device="cuda")
    tdt = BF if dtype == "bf16" else F32
    x_d, cb_d, n_d = x.to(tdt).cuda(), cb.to(tdt).cuda(), norms.cuda()
    args = L().LinearArgs()
    args.a, args.w, args.M, args.N, args.K, args.lda, args.ldw = x_d.data_ptr(), cb_d.data_ptr(), M, N, D, D, D
    args.dtype, args.epilogue = (L().BF16 if dtype == "bf16" else L().F32), G.ARGMIN
    e = L().EpilogueArgs(); e.out = out.data_ptr(); e.ldo = 1; e.out_dtype = L().F32; e.bias = n_d.data_ptr()
    args.epi = e
    want = G.linear_kernels(M, N, D, G.ARGMIN, {"ldo": 1}, dtype=dtype, sms=sms())
    observed(lambda: L().call("mmg_linear", args), want)
    got = out.cpu()
    assert torch.equal(got[:M] & 0xFFFFFFFF, want_ids), f"{int(((got[:M] & 0xFFFFFFFF) != want_ids).sum())} rows differ"
    assert bool((got[M:] == -1).all())
    STATS.setdefault(want[-1] + " (argmin, exact)", [0, 0.0])[0] += 1


# ------------------------------------------------------------------------------------------------ fallbacks and strided operands
@pytest.mark.parametrize("trigger", ["K%64", "N%64", "lda%8", "ldw%8", "a_off", "w_off", "ldo%8"])
def test_bf16_fallback_triggers(trigger):
    M, N, K = 200, 192, 128
    kw = {"K%64": dict(K=96), "N%64": dict(N=200), "lda%8": dict(lda_pad=4), "ldw%8": dict(ldw_pad=4), "a_off": dict(a_off=4),
          "w_off": dict(w_off=4), "ldo%8": dict(ldo_pad=4)}[trigger]
    M, N, K = M, kw.pop("N", N), kw.pop("K", K)
    want = G.linear_kernels(M, N, K, G.STORE, {"out": "f32", "bias": True, "ldo": N + kw.get("ldo_pad", 0)}, sms=sms(),
                            lda=K + kw.get("lda_pad", 0), ldw=K + kw.get("ldw_pad", 0), a_aligned="a_off" not in kw, w_aligned="w_off" not in kw)
    assert want == [G.SIMT("bf16", False, False)]
    run_linear(f"fb.{trigger}", M, N, K, bias=True, act=1, **kw)


def test_fp32_on_cuda_cores():
    was = ops().fp32_tc()
    ops().fp32_tc(False)
    try:
        run_linear("cc.f32", 300, 192, 128, dtype="f32", bias=True, act=1, want=[G.SIMT("f32", False, False)])
    finally:
        ops().fp32_tc(was)


@pytest.mark.parametrize("pads", [(8, 16, 64), (64, 8, 8)], ids=["lda8-ldw16-ldo64", "lda64-ldw8-ldo8"])
def test_strided_operands(pads):
    """lda, ldw > K and ldo > N, which ops.linear cannot express: the wgmma kernel reads and writes only its rows' first K / N columns"""
    run_linear(f"strided{pads}", 300, 192, 128, bias=True, lda_pad=pads[0], ldw_pad=pads[1], ldo_pad=pads[2])
    run_linear(f"strided.bf{pads}", 300, 1024, 64, out="bf16", lda_pad=pads[0], ldw_pad=pads[1], ldo_pad=pads[2])


def test_split3_fp32_store():
    run_linear("split.store", 300, 192, 128, dtype="f32", bias=True, act=1, split=True)
    run_linear("split.res", 300, 192, 128, G.RESIDUAL, dtype="f32", resid="inplace", split=True)


# ------------------------------------------------------------------------------------------------ convolutions
def run_conv(tag, kind, B, H, W, Cin, Cout, epi=G.STORE, *, dtype="bf16", out="f32", split=False):
    x = G.probe_image(tag, B, H, W, Cin, bf16=not split and dtype == "bf16")
    k = (1, 3, 4, 5)[kind]
    wp = G.pack_conv_weight(G.rnd(tag + ".w", (Cout, Cin, k, k), 0.2))
    wp = G.bf(wp) if not split and dtype == "bf16" else wp
    Ho, Wo = G.conv_out_hw(kind, H, W)
    M = B * Ho * Wo
    Nout = Cout // 2 if epi == G.GLU else Cout
    p = {"bias": G.rnd(tag + ".b", (Cout,)), "act": 1 if epi == G.STORE else 0}
    odt = BF if out == "bf16" else F32
    buf, o = guard_buf(M + 3, Nout, odt)
    resid = None
    if epi == G.RESIDUAL:
        rv = G.rnd(tag + ".r", (M, Cout))
        p["resid"] = G.bf(rv) if out == "bf16" else rv
        resid = p["resid"].to(odt).cuda()
    want, nf = G.conv_kernels(kind, B, H, W, Cin, Cout, epi, {"out": out, "bias": True, "act": p["act"], "ldo": Nout}, dtype=dtype, sms=sms(),
                              split=split, order=True)
    tdt = BF if dtype == "bf16" else F32
    x_d, w_d, b_d = x.to(tdt).cuda().contiguous(), wp.to(tdt).cuda().contiguous(), p["bias"].cuda()
    observed(lambda: ops().conv2d(x_d, w_d, o[:M], B, H, W, Cin, Cout, kind, epilogue=epi, bias=b_d, act=p["act"], resid=resid), want)
    ref, S, A = G.conv_ref(x, wp, kind, epi, p)
    variant = main_variant(want, split)
    got = o[:M].cpu()
    record(variant, got, ref, G.tolerance(variant, wp.shape[1], ref, S, A, out == "bf16"), tag, nf)
    assert_guard(buf, o, (slice(0, M), slice(0, Nout)))


# (kind, B, H, W, Cin, Cout): TW = Wo < 128 with TH capped at Ho and TB > 1, B not a multiple of TB; Wo a multiple of 128 above 128;
# non-power-of-two Ho with TW = 128; stride 2 with TB = 2; the rejected geometries and kind 3 on the CUDA cores
CONV = [(1, 3, 8, 8, 64, 64), (1, 3, 4, 16, 64, 128), (0, 1, 2, 256, 64, 64), (1, 1, 6, 128, 64, 64), (2, 3, 16, 16, 64, 128),
        (1, 2, 16, 16, 128, 192), (3, 2, 8, 8, 64, 64), (1, 2, 6, 6, 64, 64), (1, 2, 8, 8, 32, 64)]


@pytest.mark.parametrize("out", ["f32", "bf16"])
@pytest.mark.parametrize("c", CONV, ids=[f"k{c[0]}-B{c[1]}-{c[2]}x{c[3]}-{c[4]}to{c[5]}" for c in CONV])
def test_conv(c, out):
    run_conv(f"conv{c}", *c, out=out)


@pytest.mark.parametrize("epi", [G.RESIDUAL, G.GLU], ids=["residual", "glu"])
def test_conv_epilogues(epi):
    run_conv(f"conv.e{epi}", 0, 3, 8, 8, 64, 128, epi, out="bf16" if epi == G.GLU else "f32")
    run_conv(f"conv.e{epi}.cc", 1, 2, 6, 6, 64, 128, epi, out="bf16" if epi == G.GLU else "f32")


@pytest.mark.parametrize("kind", [1, 2, 3])
def test_conv_fp32(kind):
    """fp32 through split3 (kinds 1, 2) and on the CUDA cores (kind 3)"""
    run_conv(f"conv.f32.{kind}", kind, 2, 8, 8, 32, 64, dtype="f32", split=kind != 3)


def run_convt(tag, B, H, W, Cin, Cout, rgb=0, *, out="bf16", dtype="bf16"):
    x = G.probe_image(tag, B, H, W, Cin, bf16=dtype == "bf16")
    wp = G.pack_convt_weight(G.rnd(tag + ".w", (Cin, Cout, 4, 4), 0.2))
    wp = G.bf(wp) if dtype == "bf16" else wp
    p = {"bias": G.rnd(tag + ".b", (Cout,))}
    if rgb:
        p.update(rgb_w=G.rnd(tag + ".rw", (rgb, Cout), 0.1), rgb_b=G.rnd(tag + ".rb", (rgb,)))
        out = "f32"
    odt = BF if out == "bf16" else F32
    n = B * (rgb or Cout) * 4 * H * W
    buf, o = guard_buf(n, 1, odt)
    o = o.view(B, rgb, 2 * H, 2 * W) if rgb else o.view(B * 4 * H * W, Cout)
    want, nf = G.convt_kernels(B, H, W, Cin, Cout, bool(rgb), dtype=dtype, sms=sms(), split=dtype == "f32" and ops().fp32_tc(), order=True)
    tdt = BF if dtype == "bf16" else F32
    x_d, w_d = x.to(tdt).cuda().contiguous(), wp.to(tdt).cuda().contiguous()
    rw = p["rgb_w"].cuda() if rgb else None
    rb = p["rgb_b"].cuda() if rgb else None
    observed(lambda: ops().conv_transpose2d(x_d, w_d, o, B, H, W, Cin, Cout, bias=p["bias"].cuda(), rgb_w=rw, rgb_b=rb), want)
    ref, S, A = G.convt_ref(x, wp, p, bool(rgb))
    variant = main_variant(want, want[0] == G.SPLIT3)
    got = o.cpu().reshape(ref.shape)
    record(variant, got, ref, G.tolerance(variant, wp.shape[2], ref, S, A, out == "bf16"), tag, nf)
    assert bool((buf[n:] == FILL).all())


CONVT = [(3, 8, 8, 64, 64), (1, 2, 128, 64, 128), (2, 4, 16, 128, 64), (2, 3, 3, 64, 64), (2, 8, 8, 32, 64)]


@pytest.mark.parametrize("c", CONVT, ids=[f"B{c[0]}-{c[1]}x{c[2]}-{c[3]}to{c[4]}" for c in CONVT])
def test_conv_transpose(c):
    run_convt(f"ct{c}", *c)


@pytest.mark.parametrize("N,ch", [(64, 1), (128, 3), (256, 4), (128, 4)])
def test_conv_transpose_rgb(N, ch):
    run_convt(f"ctrgb{N}.{ch}", 3, 8, 8, 64, N, ch)


def test_conv_transpose_fp32():
    run_convt("ct.f32", 2, 8, 8, 32, 64, dtype="f32", out="f32")


# ------------------------------------------------------------------------------------------------ argument errors and the fixes
def _raises_launching_nothing(name, args):
    l0, s0, f0 = L().launch_count(), L().simt_launch_count(), L().simt_fallback_count()
    with pytest.raises(L().MMGError):
        L().call(name, args)
    torch.cuda.synchronize()
    assert (L().launch_count(), L().simt_launch_count(), L().simt_fallback_count()) == (l0, s0, f0), name


def _lin(M, N, K, kind=G.STORE, dtype="bf16"):
    a = torch.zeros((max(M, 1) * max(K, 1) + 64,), dtype=BF, device="cuda")
    o = torch.zeros((max(M, 1) * max(N, 1) + 64,), dtype=F32, device="cuda")
    args = L().LinearArgs()
    args.a = args.w = a.data_ptr()
    args.M, args.N, args.K, args.lda, args.ldw = M, N, K, max(K, 8), max(K, 8)
    args.dtype, args.epilogue = (L().BF16 if dtype == "bf16" else L().F32), kind
    e = L().EpilogueArgs(); e.out = o.data_ptr(); e.ldo = max(N, 8); e.out_dtype = L().F32
    args.epi = e
    return args, (a, o)


def test_linear_argument_errors():
    keep = []
    for M, N, K in ((0, 64, 64), (64, 0, 64), (64, 64, 0)):
        args, k = _lin(M, N, K); keep.append(k)
        _raises_launching_nothing("mmg_linear", args)
    args, k = _lin(64, 256, 64, G.GEGLU); keep.append(k)
    st = torch.zeros((64, 3, 2), device="cuda"); keep.append(st)
    args.epi.row_stats = st.data_ptr(); args.epi.stats_slots = 3                   # 3 < 256 / 64
    _raises_launching_nothing("mmg_linear", args)
    args, k = _lin(64, 128, 64, G.LFQ_IDS); keep.append(k)
    args.epi.ln_width = 10
    _raises_launching_nothing("mmg_linear", args)
    # LNFOLD and QKV address their outputs with 16-byte vector accesses only: an output 8 bytes off a 16-byte boundary is refused
    buf = torch.zeros(64 * 256 + 64, device="cuda"); keep.append(buf)
    args, k = _lin(64, 64, 64, G.LNFOLD); keep.append(k)
    e = args.epi
    e.out, e.resid, e.ldr, e.bias, e.row_stats, e.ln_width, e.stats_slots = buf.data_ptr() + 8, buf.data_ptr() + 8, 64, buf.data_ptr(), buf.data_ptr(), 64, 1
    _raises_launching_nothing("mmg_linear", args)
    args, k = _lin(64, 192, 64, G.QKV); keep.append(k)
    e = args.epi
    e.heads, e.tokens, e.q_rows, e.kv_rows, e.nq_heads, e.nk_heads, e.nv_heads = 1, 16, 16, 17, 1, 1, 1
    e.q_out, e.k_out, e.v_out, e.q_scale, e.k_scale = buf.data_ptr() + 8, buf.data_ptr(), buf.data_ptr(), buf.data_ptr(), buf.data_ptr()
    _raises_launching_nothing("mmg_linear", args)


def _conv_args(B, H, W, Cin, Cout, kind, dtype="bf16"):
    x = torch.zeros((4096,), dtype=BF, device="cuda")
    o = torch.zeros((4096,), dtype=F32, device="cuda")
    a = L().Conv2dArgs()
    a.x = a.w = x.data_ptr(); a.B, a.H, a.W, a.Cin, a.Cout, a.kind = B, H, W, Cin, Cout, kind
    a.dtype = L().BF16 if dtype == "bf16" else L().F32; a.epilogue = G.STORE
    e = L().EpilogueArgs(); e.out = o.data_ptr(); e.ldo = 64; e.out_dtype = L().F32
    a.epi = e
    return a, (x, o)


@pytest.mark.parametrize("dims", [(0, 8, 8, 64, 64), (2, 8, 0, 64, 64), (2, 0, 8, 64, 64), (2, 8, 8, 0, 64), (2, 8, 8, 64, 0), (-1, 8, 8, 64, 64)],
                         ids=["B0", "W0", "H0", "Cin0", "Cout0", "Bneg"])
def test_conv2d_rejects_empty_geometry(dims):
    """mmg_conv2d validates B, H, W, Cin and Cout > 0 before it computes a tile geometry or launches (W = 0 used to reach 128 % 0)"""
    a, keep = _conv_args(*dims, 1)
    _raises_launching_nothing("mmg_conv2d", a)


def test_conv2d_stride2_odd_height():
    a, keep = _conv_args(1, 7, 8, 64, 64, 2)
    _raises_launching_nothing("mmg_conv2d", a)


@pytest.mark.parametrize("case", ["geometry", "fp32", "N192"])
def test_convt_rgb_off_the_tensor_cores_is_rejected_before_counting(case):
    """CONVT_RGB where the tensor-core path does not take the call: MMG_EINVAL, and the fallback counter does not move"""
    H, Cout, dtype = {"geometry": (3, 64, "bf16"), "fp32": (8, 64, "f32"), "N192": (8, 192, "bf16")}[case]
    x = torch.zeros((2 * H * H * 64 + 64,), dtype=BF if dtype == "bf16" else F32, device="cuda")
    w = torch.zeros((4 * Cout * 256 + 64,), dtype=x.dtype, device="cuda")
    o = torch.zeros((2 * 3 * 4 * H * H,), device="cuda")
    rw, rb = torch.zeros((3, Cout), device="cuda"), torch.zeros(3, device="cuda")
    a = L().ConvTranspose2dArgs()
    a.x, a.w, a.B, a.H, a.W, a.Cin, a.Cout = x.data_ptr(), w.data_ptr(), 2, H, H, 64, Cout
    a.dtype, a.epilogue = (L().BF16 if dtype == "bf16" else L().F32), G.CONVT_RGB
    e = L().EpilogueArgs(); e.out = o.data_ptr(); e.out_dtype = L().F32; e.rgb_w = rw.data_ptr(); e.rgb_b = rb.data_ptr(); e.rgb_channels = 3
    a.epi = e
    with pytest.raises(ValueError):
        G.convt_kernels(2, H, H, 64, Cout, True, dtype=dtype)
    _raises_launching_nothing("mmg_conv_transpose2d", a)


# ------------------------------------------------------------------------------------------------ repeatability
@pytest.mark.parametrize("case", ["regs", "act", "conv"])
def test_eager_runs_and_graph_replay_are_bit_identical(case):
    a, w = G.probe_dense("rep", 300, 192, 128)
    a_d, w_d = a.to(BF).cuda(), w.to(BF).cuda()
    b_d = G.rnd("rep.b", (192,)).cuda()
    x = G.probe_image("rep.x", 3, 8, 8, 64).to(BF).cuda()
    wc = G.bf(G.pack_conv_weight(G.rnd("rep.wc", (64, 64, 3, 3), 0.2))).to(BF).cuda()
    out = torch.empty((300, 192), device="cuda") if case != "conv" else torch.empty((192, 64), device="cuda")
    if case == "regs":
        run = lambda: ops().linear(a_d, w_d, out, bias=b_d, act=1)
    elif case == "act":
        run = lambda: ops().linear(a_d, w_d, out, bias=b_d, act=2)
    else:
        run = lambda: ops().conv2d(x, wc, out, 3, 8, 8, 64, 64, 1, bias=b_d, act=1)
    eager = []
    for _ in range(2):
        out.fill_(FILL); run(); torch.cuda.synchronize()
        eager.append(out.clone())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    out.fill_(FILL)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager[0], eager[1]) and torch.equal(eager[0], out)


# ------------------------------------------------------------------------------------------------ which kernel ran
def test_every_case_reached_its_kernel():
    """this file again, in a fresh process, with every case under torch.profiler"""
    if PROFILE:
        pytest.skip("this is the profiling process")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-rP", "-m", "gpu", "--no-header", "-p", "no:cacheprovider"],
                       cwd=root, env=dict(os.environ, MMG_GEMM_PROFILE="1"), capture_output=True, text=True, timeout=480)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ report
def test_every_variant_was_reached(request):
    """per variant: the cases above that reached it and the worst |err| / tol (the figures recorded in tests/gemm_oracle.py)"""
    if request.config.getoption("keyword") or not STATS:
        pytest.skip("a report over the whole file")
    print(torch.cuda.get_device_name(), f"{sms()} SMs")
    for variant, (cases, worst) in sorted(STATS.items()):
        print(f"{variant:56s} cases {cases:3d}  worst err / tol {worst:.3f}")
    from tests.test_gpu_row_kernels import CAPTURE_RETAKES
    print(f"profiler captures taken again after a shortfall of kernel records: {CAPTURE_RETAKES[0]}")
    seen = " ".join(STATS)
    missing = [v for v in G.TC_VARIANTS + G.SIMT_VARIANTS if v not in seen]
    # both tile orders for every tensor-core instantiation; CONVT_RGB at N = 256 is one column tile, so M-fast only
    missing += [stat_key(v, nf) for v in G.TC_VARIANTS for nf in (0, 1) if not (v == G.TC(256, G.M_REGS) and nf == 1)
                and stat_key(v, nf) not in STATS]
    assert not missing, missing

"""Per-kernel microbenchmarks at the C3 (B=64) shapes: CUDA-event timing with an L2 flush between iterations, achieved
TFLOP/s or GB/s against the H100 data sheet (or MEASURED_PEAKS.json).  Also the command ncu wraps (`--only <name>` runs one kernel a few times).
usage: python scripts/kernel_bench.py [--only gemm|ln|sample|attn|conv|vq] [--iters 5]"""
import argparse
import json
import os
import subprocess
import sys
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from muse_maskgit_pytorch_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--only", default="")
ap.add_argument("--iters", type=int, default=5)
args = ap.parse_args()
pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
# bench.py's figures: the H100 SXM data sheet (dense bf16, HBM3) unless MEASURED_PEAKS.json is present
PK_T, PK_B = pk.get("bf16_tflops_sustained", pk.get("bf16_tflops", 989.0)), pk.get("hbm_gbs", 3350.0)
PK_SRC = "measured" if pk else "H100 SXM data sheet"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
bf = torch.bfloat16


def timeit(fn, iters=args.iters):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts), sum(ts) / len(ts)


def report(name, ms, flops=None, bytes_=None):
    s = f"{name:58s} best {ms[0] * 1e3:9.1f} us  avg {ms[1] * 1e3:9.1f} us"
    if flops:
        t = flops / (ms[0] * 1e-3) / 1e12
        s += f"  {t:8.1f} TFLOP/s ({t / PK_T:5.1%} of {PK_T:.0f})"
    if bytes_:
        g = bytes_ / (ms[0] * 1e-3) / 1e9
        s += f"  {g:8.1f} GB/s ({g / PK_B:5.1%} of {PK_B:.0f})"
    print(s, flush=True)


def want(k):
    return not args.only or k in args.only.split(",")


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


print(f"# {torch.cuda.get_device_name()}  nvidia-smi name, power.limit [W], clocks.max.sm [MHz]: {smi('name,power.limit,clocks.max.sm') or 'unavailable'}"
      f"  peaks: {PK_T:.0f} TFLOP/s, {PK_B:.0f} GB/s ({PK_SRC})", flush=True)

R = 2 * 64 * 256            # rows of a CFG decode step at B=64
SMS = torch.cuda.get_device_properties(0).multi_processor_count


def tc_tile_n(M, N):
    """The wgmma kernel's tile width for a tile epilogue (mmg_gemm.cu pick_bn)."""
    mt = (M + 127) // 128
    if N % 256 == 0 and mt * (N // 256) >= 2 * SMS:
        return 256
    if N % 128 == 0 and (mt * (N // 128) >= SMS or N >= 1024):
        return 128
    return 64 if (N % 64 == 0 and N % 128 != 0) else (128 if mt * ((N + 127) // 128) >= 96 else 64)


def gemm_case(kind, M, N, K):
    """Operands and the launch that generate() makes for one product (muse_maskgit.py _run_blocks / _ff_tail, the fused tail)."""
    heads, n = 8, 256
    a = torch.randn((M, K), device="cuda").to(bf); w = (torch.randn((N, K), device="cuda") * K ** -0.5).to(bf)
    if kind == "qkv":           # self-attention: q, k, v heads, l2-normalised q / k, null k / v in key row 0
        bh, tk = M // n * heads, (n + 1 + 7) // 8 * 8
        q = torch.empty((bh, n, 64), device="cuda", dtype=bf); k = torch.zeros((bh, tk, 64), device="cuda", dtype=bf); v = torch.zeros_like(k)
        qs, ks = torch.rand(64, device="cuda") + 0.5, torch.rand(64, device="cuda") + 0.5
        nk, nv = torch.randn((heads, 64), device="cuda").to(bf), torch.randn((heads, 64), device="cuda").to(bf)
        e = ops.qkv_epilogue(bf, heads, n, q=q, k=k, v=v, q_scale=qs, k_scale=ks, key_off=1, null_k=nk, null_v=nv)
        # the epilogue block holds raw pointers: the closure keeps the tensors behind them alive
        return lambda keep=(q, k, v, qs, ks, nk, nv): ops.linear(a, w, None, epilogue=ops.EPI_QKV, epi=e)
    if kind == "q":             # cross-attention queries
        q = torch.empty((M // n * heads, n, 64), device="cuda", dtype=bf); qs = torch.rand(64, device="cuda") + 0.5
        e = ops.qkv_epilogue(bf, heads, n, q=q, q_scale=qs)
        return lambda keep=(q, qs): ops.linear(a, w, None, epilogue=ops.EPI_QKV, epi=e)
    if kind == "resid":         # to_out: x += ao @ W^T in place
        x = torch.zeros((M, N), device="cuda")
        return lambda: ops.linear(a, w, x, epilogue=ops.EPI_RESIDUAL, resid=x)
    if kind == "geglu":         # FF1: GEGLU + per-chunk row statistics
        h = torch.empty((M, N // 2), device="cuda", dtype=bf); st = torch.zeros((M, N // 64, 2), device="cuda")
        return lambda: ops.linear(a, w, h, epilogue=ops.EPI_GEGLU, row_stats=st)
    if kind == "lnfold":        # FF2: folded LayerNorm of h (statistics of FF1's 44 chunks) + residual, in place
        x = torch.zeros((M, N), device="cuda"); st = torch.ones((M, 44, 2), device="cuda") * 31; cv = torch.randn(N, device="cuda")
        return lambda: ops.linear(a, w, x, epilogue=ops.EPI_LNFOLD_RESIDUAL, bias=cv, resid=x, row_stats=st, ln_width=1365)
    out = torch.empty((M, N), device="cuda")   # "tstore": the fused tail's sample GEMM, fp32 [rows, 4096] (contiguous W here)
    return lambda: ops.linear(a, w, out)


if want("gemm"):
    # the products generate() launches at C3, per layer, and a K sweep of each: time per call = tiles per CTA x (per-tile fixed cost +
    # K / 64 x per-k-block cost).  The intercept is the epilogue + pipeline refill, the slope is set against the k-block at the
    # data-sheet tensor rate (128 x BN x 64 x 2 FLOP at 4096 FLOP / cycle / SM).
    for name, kind, M, N, K in [("qkv      (self)   ", "qkv", R, 1536, 512), ("to_out   (self)  +x", "resid", R, 512, 512),
                                ("q        (cross)  ", "q", R // 2, 512, 512), ("to_out   (cross) +x", "resid", R // 2, 512, 512),
                                ("ff1 geglu+stats   ", "geglu", R, 2816, 512), ("ff2 lnfold      +x", "lnfold", R, 512, 1408),
                                ("tail sample f32   ", "tstore", 16384, 4096, 512)]:
        bn = tc_tile_n(M, N)
        tiles = (M + 127) // 128 * ((N + bn - 1) // bn)
        per_cta = -(-tiles // min(tiles, SMS))
        pts = []
        for f in (1, 2, 4):
            fn = gemm_case(kind, M, N, K * f)
            ms = timeit(fn)
            mhz = smi("clocks.sm")
            report(f"gemm {name} M={M} N={N} K={K * f} BN={bn}", ms, flops=2.0 * M * N * K * f)
            pts.append((K * f / 64, ms[0] * 1e3 / per_cta, float(mhz) if mhz.replace(".", "").isdigit() else float("nan")))
            del fn
            torch.cuda.empty_cache()
        xs, ys = [p[0] for p in pts], [p[1] for p in pts]
        xm, ym = sum(xs) / 3, sum(ys) / 3
        slope = sum((x - xm) * (y - ym) for x, y in zip(xs, ys)) / sum((x - xm) ** 2 for x in xs)
        icpt = ym - slope * xm
        clk = min(p[2] for p in pts)
        print(f"    K sweep: {per_cta} tiles/CTA  intercept {icpt:.2f} us/tile  slope {slope * 1e3:.1f} ns/k-block = {slope * clk:.0f} cycles at "
              f"{clk:.0f} MHz (peak rate {128 * bn * 64 * 2 // 4096})", flush=True)
    for name, M, N, K, odt in [("logits M=16384 N=65536 K=512 fp32 out", 16384, 65536, 512, torch.float32),
                               ("logits M=64 N=65536 K=512 fp32 out", 64, 65536, 512, torch.float32), ("square 8192^3 bf16 out", 8192, 8192, 8192, bf)]:
        a = torch.randn((M, K), device="cuda").to(bf); w = (torch.randn((N, K), device="cuda") * K ** -0.5).to(bf)
        out = torch.empty((M, N), device="cuda", dtype=odt)
        report("gemm " + name, timeit(lambda: ops.linear(a, w, out)), flops=2.0 * M * N * K)
        del a, w, out

if want("ln"):
    x = torch.randn((R, 512), device="cuda"); g = torch.ones(512, device="cuda"); y = torch.empty((R, 512), device="cuda", dtype=bf)
    report("layernorm 32768x512 f32->bf16", timeit(lambda: ops.layernorm(x, g, y)), bytes_=R * 512 * 6)
    h = torch.randn((R, 1408), device="cuda").to(bf); g3 = torch.ones(1408, device="cuda"); hn = torch.empty_like(h)
    report("layernorm 32768x1365(1408) bf16->bf16", timeit(lambda: ops.layernorm(h, g3, hn, width=1365)), bytes_=R * 1408 * 4)

if want("sample"):
    for rows in (16384, 10240, 64):
        V, n, b = 65536, 256, 64
        nm = rows // b
        lg = torch.randn((rows, V), device="cuda") * 0.58
        mp = torch.arange(nm, device="cuda", dtype=torch.int32).repeat(b, 1).contiguous()
        ids = torch.full((b, n), V, device="cuda", dtype=torch.long); sc = torch.zeros((b, n), device="cuda")
        report(f"logits_sample rows={rows} V=65536 k=6554 T=1 (philox)", timeit(lambda: ops.logits_sample(lg, mp, ids, sc, nm, 6554, 1.0, seed=1)), bytes_=rows * V * 4)
        report(f"logits_sample rows={rows} V=65536 k=6554 T=0", timeit(lambda: ops.logits_sample(lg, mp, ids, sc, nm, 6554, 0.0, seed=1)), bytes_=rows * V * 4)
        del lg

if want("fused"):
    # to_logits + sampling tail: materialised (GEMM -> [rows, V] fp32 -> sampler) vs fused (candidate lists out of the GEMM epilogue)
    V, K, n, b, k = 65536, 512, 256, 64, 6554
    w = (torch.randn((V, K), device="cuda") * K ** -0.5).to(bf)
    for rows in (16384, 10240, 4096, 64):
        nm = rows // b
        e = torch.randn((rows, K), device="cuda").to(bf)
        mp = torch.arange(nm, device="cuda", dtype=torch.int32).repeat(b, 1).contiguous()
        ids = torch.full((b, n), V, device="cuda", dtype=torch.long); sc = torch.zeros((b, n), device="cuda")
        lg = torch.empty((rows, V), device="cuda")
        def unfused():
            ops.linear(e, w, lg); ops.logits_sample(lg, mp, ids, sc, nm, k, 1.0, seed=1)
        report(f"tail materialised rows={rows}: logits GEMM + logits_sample", timeit(unfused), flops=2.0 * rows * V * K)
        ws = torch.empty((ops.logits_fused_workspace_bytes(rows, V, K, k),), dtype=torch.uint8, device="cuda"); st = torch.zeros((2,), dtype=torch.int32, device="cuda")
        report(f"tail fused        rows={rows}: mmg_logits_fused (6 launches)", timeit(lambda: ops.logits_fused(e, w, mp, ids, sc, nm, k, 1.0, ws, st, rows_capacity=rows, seed=1)), flops=2.0 * rows * V * K)
        print(f"    fallback rows so far {st.tolist()}", flush=True)
        del lg, ws

if want("attn"):
    for name, B, Tq, Tk, masked in [("self  B=128 h=8 Tq=256 Tk=257", 128, 256, 257, False), ("cross B=64 h=8 Tq=256 Tk=33", 64, 256, 33, True)]:
        heads = 8
        q = torch.nn.functional.normalize(torch.randn((B * heads, Tq, 64), device="cuda"), dim=-1).to(bf)
        alloc = (Tk + 7) // 8 * 8
        k = torch.zeros((B * heads, alloc, 64), device="cuda", dtype=bf); k[:, :Tk] = torch.nn.functional.normalize(torch.randn((B * heads, Tk, 64), device="cuda"), dim=-1).to(bf)
        v = torch.zeros_like(k); v[:, :Tk] = torch.randn((B * heads, Tk, 64), device="cuda").to(bf)
        out = torch.empty((B * Tq, heads * 64), device="cuda", dtype=bf)
        km = (torch.rand((B, Tk - 1), device="cuda") > 0.2).to(torch.uint8) if masked else None
        report("attention " + name + " two-pass", timeit(lambda: ops.attention(q, k, v, out, B, heads, Tk, key_mask=km)), flops=4.0 * B * heads * Tq * Tk * 64)
        report("attention " + name + " single-pass", timeit(lambda: ops.attention(q, k, v, out, B, heads, Tk, key_mask=km, logit_bound=1.02)), flops=4.0 * B * heads * Tq * Tk * 64)

if want("conv"):
    B = 64
    for name, H, Cin, Cout, kind in [("3x3 2048->4096 @16 GLU", 16, 2048, 4096, 1), ("1x1 2048->2048 @16", 16, 2048, 2048, 0)]:
        x = torch.randn((B * H * H, Cin), device="cuda").to(bf)
        taps = 9 if kind == 1 else 1
        w = (torch.randn((Cout, taps * Cin), device="cuda") * (taps * Cin) ** -0.5).to(bf)
        if kind == 1:
            out = torch.empty((B * H * H, Cout // 2), device="cuda", dtype=bf); bias = torch.zeros(Cout, device="cuda")
            fn = lambda: ops.conv2d(x, w, out, B, H, H, Cin, Cout, 1, epilogue=ops.EPI_GLU, bias=bias)
        else:
            out = torch.empty((B * H * H, Cout), device="cuda", dtype=bf); fn = lambda: ops.conv2d(x, w, out, B, H, H, Cin, Cout, 0)
        report("conv2d " + name, timeit(fn), flops=2.0 * B * H * H * Cout * taps * Cin)
        del x, w, out
    for name, H, Cin, Cout, rgb in [("convT 2048->1024 @16", 16, 2048, 1024, False), ("convT 1024->512 @32", 32, 1024, 512, False), ("convT 512->256 @64", 64, 512, 256, False),
                                    ("convT 256->256 @128 + fused 1x1->3", 128, 256, 256, True)]:
        x = torch.randn((B * H * H, Cin), device="cuda").to(bf)
        w = (torch.randn((4, Cout, 4 * Cin), device="cuda") * (4 * Cin) ** -0.5).to(bf); bias = torch.zeros(Cout, device="cuda")
        if rgb:
            out = torch.empty((B, 3, 2 * H, 2 * H), device="cuda"); rw = torch.randn((3, Cout), device="cuda"); rb = torch.zeros(3, device="cuda")
            fn = lambda: ops.conv_transpose2d(x, w, out, B, H, H, Cin, Cout, bias=bias, rgb_w=rw, rgb_b=rb)
        else:
            out = torch.empty((B * 4 * H * H, Cout), device="cuda", dtype=bf); fn = lambda: ops.conv_transpose2d(x, w, out, B, H, H, Cin, Cout, bias=bias)
        report("conv_transpose2d " + name, timeit(fn), flops=2.0 * B * H * H * Cout * 16 * Cin)
        del x, w, out

if want("vq"):
    T, D, bits = 16384, 2048, 16
    x = torch.randn((T, D), device="cuda").to(bf); w = torch.randn((bits, D), device="cuda"); bb = torch.zeros(bits, device="cuda")
    ids = torch.empty((T,), device="cuda", dtype=torch.long)
    report("vq_lfq_encode T=16384 D=2048 bits=16 (bf16 fmap)", timeit(lambda: ops.vq_lfq_encode(x, w, bb, ids, bits)), bytes_=T * (D * 2 + 8))
    hi = w.to(bf); r1 = w - hi.float(); mid = r1.to(bf); lo = (r1 - mid.float()).to(bf)
    w3 = torch.zeros((64, D), device="cuda", dtype=bf); w3[:16], w3[16:32], w3[32:48] = hi, mid, lo
    report("vq LFQ via wgmma GEMM + LFQ_IDS epilogue (bf16 fmap)", timeit(lambda: ops.linear(x, w3, ids, epilogue=ops.EPI_LFQ_IDS, bias=bb, ln_width=bits)), bytes_=T * (D * 2 + 8))
    xf = x.float(); report("vq_lfq_encode T=16384 D=2048 bits=16 (fp32 fmap)", timeit(lambda: ops.vq_lfq_encode(xf, w, bb, ids, bits)), bytes_=T * (D * 4 + 8))
    T2, K2, D2 = 256, 8192, 256
    x2 = torch.randn((T2, D2), device="cuda"); cb = torch.randn((K2, D2), device="cuda"); ids2 = torch.empty((T2,), device="cuda", dtype=torch.long)
    report("vq_l2_argmin T=256 K=8192 D=256 (scan regime)", timeit(lambda: ops.vq_l2_argmin(x2, cb, ids2)), bytes_=K2 * D2 * 4 + T2 * D2 * 4, flops=2.0 * T2 * K2 * D2)

"""Per-kernel microbenchmarks at the C3 (B=64) shapes: CUDA-event timing with an L2 flush between iterations, achieved
TFLOP/s or GB/s against MEASURED_PEAKS.json.  Also the command ncu wraps (`--only <name>` runs one kernel a few times).
usage: python scripts/kernel_bench.py [--only gemm|ln|sample|attn|conv|vq] [--iters 5]"""
import argparse
import json
import os
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
PK_T, PK_B = pk.get("bf16_tflops", 1590.0), pk.get("hbm_gbs", 6650.0)
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
        s += f"  {t:8.1f} TFLOP/s ({t / PK_T:5.1%} of measured {PK_T:.0f})"
    if bytes_:
        g = bytes_ / (ms[0] * 1e-3) / 1e9
        s += f"  {g:8.1f} GB/s ({g / PK_B:5.1%} of measured {PK_B:.0f})"
    print(s, flush=True)


def want(k):
    return not args.only or k in args.only.split(",")


R = 2 * 64 * 256            # rows of a CFG decode step at B=64
if want("gemm"):
    for name, M, N, K, epi in [("qkv  M=32768 N=1536 K=512", R, 1536, 512, "store_bf16"), ("wo   M=32768 N=512 K=512 +resid", R, 512, 512, "resid"),
                               ("ff1  M=32768 N=2816 K=512 geglu", R, 2816, 512, "geglu"), ("ff1  M=32768 N=2816 K=512 geglu+rowstats", R, 2816, 512, "geglu_stats"),
                               ("ff2  M=32768 N=512 K=1408 +resid", R, 512, 1408, "resid"), ("ff2  M=32768 N=512 K=1408 lnfold+resid", R, 512, 1408, "lnfold"),
                               ("logits M=10240 N=65536 K=512 fp32 out", 10240, 65536, 512, "store_f32"), ("logits M=16384 N=65536 K=512 fp32 out", 16384, 65536, 512, "store_f32"),
                               ("logits M=64 N=65536 K=512 fp32 out", 64, 65536, 512, "store_f32"), ("square 8192^3 bf16 out", 8192, 8192, 8192, "store_bf16")]:
        a = torch.randn((M, K), device="cuda").to(bf); w = (torch.randn((N, K), device="cuda") * K ** -0.5).to(bf)
        if epi == "store_bf16":
            out = torch.empty((M, N), device="cuda", dtype=bf); fn = lambda: ops.linear(a, w, out)
        elif epi == "store_f32":
            out = torch.empty((M, N), device="cuda"); fn = lambda: ops.linear(a, w, out)
        elif epi == "resid":
            out = torch.zeros((M, N), device="cuda"); fn = lambda: ops.linear(a, w, out, epilogue=ops.EPI_RESIDUAL, resid=out)
        elif epi == "geglu_stats":
            out = torch.empty((M, N // 2), device="cuda", dtype=bf); st = torch.zeros((M, N // 64, 2), device="cuda"); fn = lambda: ops.linear(a, w, out, epilogue=ops.EPI_GEGLU, row_stats=st)
        elif epi == "lnfold":
            out = torch.zeros((M, N), device="cuda"); st = torch.ones((M, K // 32, 2), device="cuda") * 31; cv = torch.zeros(N, device="cuda")
            fn = lambda: ops.linear(a, w, out, epilogue=ops.EPI_LNFOLD_RESIDUAL, bias=cv, resid=out, row_stats=st, ln_width=1365)
        else:
            out = torch.empty((M, N // 2), device="cuda", dtype=bf); e = ops._epi(out, N // 2); fn = lambda: ops.linear(a, w, None, epilogue=ops.EPI_GEGLU, epi=e)
        report("gemm " + name, timeit(fn), flops=2.0 * M * N * K)
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

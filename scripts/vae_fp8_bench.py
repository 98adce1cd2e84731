"""VQGanVAE precision="fp8" against "bf16" on one GPU: each e4m3 convolution of the benchmark VAE (dim = 256) at C5 (512^2) and C3
(256^2) shapes against its bf16 twin, the per-image quantiser, C5 encode + decode images/s, and C3 generate() with an fp8 transformer over
a bf16 VAE against the same over an fp8 VAE.  Arms alternate round by round; times are the best of --iters with an L2 flush before each.
The card's name, power limit and SM clocks are read in the same process.
usage: python scripts/vae_fp8_bench.py [--rounds 3] [--iters 10] [--batch 4] [--gen-batch 64] [--out results/vae_fp8_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import muse_maskgit_pytorch_b200 as M  # noqa: E402
from muse_maskgit_pytorch_b200 import ops, t5  # noqa: E402
from muse_maskgit_pytorch_b200.muse_maskgit import quantize_rows_e4m3  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--batch", type=int, default=4, help="images per VAE call (per-conv table and C5 encode + decode)")
ap.add_argument("--gen-batch", type=int, default=64, help="images per C3 generate() call")
ap.add_argument("--steps", type=int, default=18)
ap.add_argument("--out", default="")
args = ap.parse_args()
assert torch.cuda.is_available(), "vae_fp8_bench.py measures on the GPU; there is no CPU fallback"
torch.set_grad_enabled(False)
bf = torch.bfloat16


def smi():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def best_ms(fn, iters):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts)


def convs(B, fmap):
    """(name, kind, B, H, W, Cin, Cout, epilogue) of the dim = 256 VAE's implicit-GEMM convolutions for a fmap x fmap latent grid;
    kind 'ct' = conv-transpose (its four parity launches), 'rgb' = the last conv-transpose with the fused 1x1"""
    out = []
    s = fmap * 16
    for cin, cout in ((256, 256), (256, 512), (512, 1024), (1024, 2048)):
        out.append((f"down {cin}->{cout} @{s}", 2, B, s, s, cin, cout, ops.EPI_STORE)); s //= 2
    out.append((f"res 3x3 2048 @{fmap}", 1, B, fmap, fmap, 2048, 2048, ops.EPI_STORE))
    out.append((f"glu 3x3 2048->4096 @{fmap}", 1, B, fmap, fmap, 2048, 4096, ops.EPI_GLU))
    out.append((f"res 1x1 2048 + resid @{fmap}", 0, B, fmap, fmap, 2048, 2048, ops.EPI_RESIDUAL))
    s = fmap
    for cin, cout in ((2048, 1024), (1024, 512), (512, 256)):
        out.append((f"up {cin}->{cout} @{s}", "ct", B, s, s, cin, cout, None)); s *= 2
    out.append((f"up+rgb 256->256 @{s}", "rgb", B, s, s, 256, 256, None))
    return out


def conv_arms(kind, B, H, W, Cin, Cout, epi):
    """(bf16 fn, fp8 conv fn, quantiser fn, GFLOP)"""
    g = torch.Generator(device="cuda").manual_seed(Cin + Cout + H)
    x = (torch.randn((B * H * W, Cin), device="cuda", generator=g) * 0.5).to(bf)
    bias = torch.randn((Cout,), device="cuda", generator=g) * 0.1
    q, s = ops.quantize_e4m3_images(x, B)
    quant = lambda: ops.quantize_e4m3_images(x, B, q, s)
    if kind in ("ct", "rgb"):
        w = torch.randn((4 * Cout, 4 * Cin), device="cuda", generator=g) * 0.02
        wb, (wq, ws) = w.to(bf).view(4, Cout, 4 * Cin), quantize_rows_e4m3(w)
        wq, ws = wq.view(4, Cout, 4 * Cin), ws.view(4, Cout)
        if kind == "rgb":
            out = torch.empty((B, 3, 2 * H, 2 * W), device="cuda")
            rw, rb = torch.randn((3, Cout), device="cuda", generator=g) * 0.05, torch.zeros((3,), device="cuda")
            f16 = lambda: ops.conv_transpose2d(x, wb, out, B, H, W, Cin, Cout, bias=bias, rgb_w=rw, rgb_b=rb)
            f8 = lambda: ops.conv_transpose2d_fp8(q, s, wq, ws, out, B, H, W, Cin, Cout, bias=bias, rgb_w=rw, rgb_b=rb)
        else:
            out = torch.empty((B * 4 * H * W, Cout), device="cuda", dtype=bf)
            f16 = lambda: ops.conv_transpose2d(x, wb, out, B, H, W, Cin, Cout, bias=bias)
            f8 = lambda: ops.conv_transpose2d_fp8(q, s, wq, ws, out, B, H, W, Cin, Cout, bias=bias)
        return f16, f8, quant, 2.0 * B * 4 * H * W * Cout * 4 * Cin / 1e9
    taps = (1, 9, 16)[kind]
    Ho, Wo = (H // 2, W // 2) if kind == 2 else (H, W)
    w = torch.randn((Cout, taps * Cin), device="cuda", generator=g) * 0.02
    wb, (wq, ws) = w.to(bf), quantize_rows_e4m3(w)
    out = torch.empty((B * Ho * Wo, Cout // 2 if epi == ops.EPI_GLU else Cout), device="cuda", dtype=bf)
    kw = dict(epilogue=epi, bias=bias, act=1 if kind == 2 else 0)
    if epi == ops.EPI_RESIDUAL:
        kw["resid"] = x
    f16 = lambda: ops.conv2d(x, wb, out, B, H, W, Cin, Cout, kind, **kw)
    f8 = lambda: ops.conv2d_fp8(q, s, wq, ws, out, B, H, W, Cin, Cout, kind, **kw)
    return f16, f8, quant, 2.0 * B * Ho * Wo * Cout * taps * Cin / 1e9


res = {"gpu": smi(), "args": vars(args), "convs": [], "c5": {}, "c3_generate": {}}
print("GPU:", res["gpu"])

# ---- per convolution
for cfg, fmap in (("C5", 32), ("C3", 16)):
    for name, *c in convs(args.batch, fmap):
        f16, f8, quant, gf = conv_arms(*c)
        t = {"bf16": [], "fp8": [], "quant": []}
        for _ in range(args.rounds):
            t["bf16"].append(best_ms(f16, args.iters)); t["fp8"].append(best_ms(f8, args.iters)); t["quant"].append(best_ms(quant, args.iters))
        row = {"config": cfg, "conv": name, "gflop": gf, **{k + "_us": 1e3 * min(v) for k, v in t.items()}}
        row["bf16_tflops"] = gf / row["bf16_us"] * 1e3
        row["fp8_tflops"] = gf / row["fp8_us"] * 1e3
        res["convs"].append(row)
        print(f"{cfg} {name:32s} bf16 {row['bf16_us']:9.1f} us ({row['bf16_tflops']:6.1f} TFLOP/s)  fp8 {row['fp8_us']:9.1f} us "
              f"({row['fp8_tflops']:6.1f} TFLOP/s)  quantiser {row['quant_us']:8.1f} us  fp8 + quantiser / bf16 "
              f"{(row['fp8_us'] + row['quant_us']) / row['bf16_us']:.3f}", flush=True)
        del f16, f8, quant
    torch.cuda.empty_cache()

# ---- C5: encode + decode of 512^2 images
torch.manual_seed(0)
base = M.VQGanVAE(dim=256, codebook_size=65536).cuda()
vaes = {}
for prec in ("bf16", "fp8"):
    v = M.VQGanVAE(dim=256, codebook_size=65536, precision=prec).cuda()
    v.load_state_dict(base.state_dict())
    vaes[prec] = v
del base
img = torch.rand((args.batch, 3, 512, 512), device="cuda") * 2 - 1
t = {p: [] for p in vaes}
for _ in range(args.rounds):
    for p, v in vaes.items():
        t[p].append(best_ms(lambda: v(img), max(3, args.iters // 2)))
for p in vaes:
    res["c5"][p] = {"ms": min(t[p]), "images_per_s": args.batch / min(t[p]) * 1e3}
    print(f"C5 encode + decode ({args.batch} x 512^2), {p} VAE: {min(t[p]):.2f} ms, {res['c5'][p]['images_per_s']:.1f} images/s", flush=True)
del vaes, img
torch.cuda.empty_cache()

# ---- C3: generate() with an fp8 transformer over a bf16 / fp8 VAE
t5.T5_CONFIGS["synth-768"] = {"d_model": 768}
torch.manual_seed(0)
tr = M.MaskGitTransformer(num_tokens=65536, seq_len=256, dim=512, depth=8, dim_head=64, heads=8, ff_mult=4, t5_name="synth-768",
                          precision="fp8")
te = torch.randn((args.gen_batch, 16, 768), generator=torch.Generator().manual_seed(5)).cuda()
tr.encode_text = lambda texts: te[:len(texts)]
torch.manual_seed(1)
vb = M.VQGanVAE(dim=256, codebook_size=65536)
vf = M.VQGanVAE(dim=256, codebook_size=65536, precision="fp8")
vf.load_state_dict(vb.state_dict())
mgs = {"bf16": M.MaskGit(image_size=256, transformer=tr, vae=vb).cuda(), "fp8": M.MaskGit(image_size=256, transformer=tr, vae=vf).cuda()}
texts = ["a"] * args.gen_batch
t = {p: [] for p in mgs}
for p, mg in mgs.items():
    mg.generate(texts, timesteps=args.steps)                      # warm-up (graph capture, packing)
for _ in range(args.rounds):
    for p, mg in mgs.items():
        torch.cuda.synchronize(); t0 = time.perf_counter()
        mg.generate(texts, timesteps=args.steps)
        torch.cuda.synchronize(); t[p].append(time.perf_counter() - t0)
for p in mgs:
    res["c3_generate"][p + "_vae"] = {"s": min(t[p]), "images_per_s": args.gen_batch / min(t[p]), "all_s": t[p]}
    print(f"C3 generate() ({args.gen_batch} images, {args.steps} steps), fp8 transformer over a {p} VAE: {min(t[p]) * 1e3:.1f} ms, "
          f"{args.gen_batch / min(t[p]):.1f} images/s  (rounds: {', '.join(f'{x * 1e3:.1f}' for x in t[p])} ms)", flush=True)
print("GPU (after):", smi())
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)

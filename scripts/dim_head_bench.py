"""What 128-wide attention heads cost: the same inner width (512) as 8 heads x 64 or 4 heads x 128, in one process.

  attention: mmg_attention (heads 8, dh 64) against mmg_attention_d128 (heads 4, dh 128) on the C3 self-attention (128 sequences = 64 images
             x CFG, 256 queries, 256 keys + the null key), the C3 cross-attention (64 sequences, 32 text keys + null, key mask) and the C4
             self-attention (64 sequences, 1024 queries, 1024 keys + null); single-pass softmax (unit q, k, logit bound 1.02, scale 8), as
             the model calls them.  The QK^T and PV FLOPs are equal for both layouts: 4 B Tq Tk 512.
  QKV:       the C3 self-attention QKV product (32768 x 1536 x 512) with the EPI_QKV and the EPI_QKV128 epilogue.
  generate:  C3-architecture generate() images/s (dim 512, depth 8, V 65536, 8 x 64 vs 4 x 128 heads, bf16, 18 steps), the two layouts
             alternated over --rounds.
CUDA events around --iters calls after a warm-up; TFLOP/s from the shape-derived FLOPs.  The card's name and power limit are read in the
same process.
usage: python scripts/dim_head_bench.py [--rounds 3] [--iters 30] [--batch 8] [--out results.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import muse_maskgit_pytorch_b200 as M  # noqa: E402
from muse_maskgit_pytorch_b200 import ops, t5  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=30)
ap.add_argument("--batch", type=int, default=8, help="images per generate() call")
ap.add_argument("--out", default="")
args = ap.parse_args()
assert torch.cuda.is_available(), "dim_head_bench.py measures on the GPU; there is no CPU fallback"
torch.set_grad_enabled(False)
dev = "cuda"


def smi():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30)
    return r.stdout.strip()


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e-3          # seconds per call


INNER = 512
SHAPES = [("C3 self  B=128 Tq=256 Tk=257", 128, 256, 257, False),
          ("C3 cross B=64  Tq=256 Tk=33 masked", 64, 256, 33, True),
          ("C4 self  B=64  Tq=1024 Tk=1025", 64, 1024, 1025, False)]
results = dict(card=smi(), attention=[], qkv=[], generate=[])
print("card (name, power limit, max SM clock):", results["card"])

g = torch.Generator(device=dev).manual_seed(0)
for name, B, Tq, Tk, masked in SHAPES:
    row = dict(shape=name)
    for heads, dh in ((8, 64), (4, 128)):
        q = F.normalize(torch.randn((B * heads, Tq, dh), device=dev, generator=g), dim=-1).to(torch.bfloat16)
        k = F.normalize(torch.randn((B * heads, (Tk + 7) // 8 * 8, dh), device=dev, generator=g), dim=-1).to(torch.bfloat16)
        v = torch.randn((B * heads, (Tk + 7) // 8 * 8, dh), device=dev, generator=g).to(torch.bfloat16)
        out = torch.empty((B * Tq, INNER), device=dev, dtype=torch.bfloat16)
        km = (torch.rand((B, Tk - 1), device=dev, generator=g) < 0.75).to(torch.uint8) if masked else None
        t = timed(lambda: ops.attention(q, k, v, out, B, heads, Tk, key_mask=km, logit_bound=1.02), args.iters)
        row[f"{heads}x{dh}"] = dict(us=t * 1e6, tflops=4.0 * B * Tq * Tk * INNER / t / 1e12)
    results["attention"].append(row)
    print(f"attention {name}: " + ", ".join(f"{kk} {vv['us']:.1f} us {vv['tflops']:.1f} TFLOP/s" for kk, vv in row.items() if kk != "shape"))

rows, tokens, dim = 128 * 256, 256, 512
a = torch.randn((rows, dim), device=dev, generator=g).to(torch.bfloat16)
w = (torch.randn((3 * INNER, dim), device=dev, generator=g) / dim ** 0.5).to(torch.bfloat16)
row = dict(shape=f"C3 self QKV {rows} x {3 * INNER} x {dim}")
for heads, dh in ((8, 64), (4, 128)):
    q = torch.empty((rows // tokens * heads, tokens, dh), device=dev, dtype=torch.bfloat16)
    k = torch.zeros((rows // tokens * heads, tokens + 8, dh), device=dev, dtype=torch.bfloat16); v = torch.zeros_like(k)
    sc = torch.ones(dh, device=dev)
    nk = torch.zeros((heads, dh), device=dev, dtype=torch.bfloat16)
    epi = ops.qkv_epilogue(torch.bfloat16, heads, tokens, q=q, k=k, v=v, q_scale=sc, k_scale=sc, key_off=1, null_k=nk, null_v=nk)
    t = timed(lambda: ops.linear(a, w, None, epilogue=ops.qkv_kind(q), epi=epi), args.iters)
    row[f"{heads}x{dh}"] = dict(us=t * 1e6, tflops=2.0 * rows * 3 * INNER * dim / t / 1e12)
results["qkv"].append(row)
print(f"QKV {row['shape']}: " + ", ".join(f"{kk} {vv['us']:.1f} us {vv['tflops']:.1f} TFLOP/s" for kk, vv in row.items() if kk != "shape"))

t5.T5_CONFIGS["synth-512"] = {"d_model": 512}
models = {}
for heads, dh in ((8, 64), (4, 128)):
    torch.manual_seed(0)
    tr = M.MaskGitTransformer(num_tokens=65536, seq_len=256, dim=512, depth=8, dim_head=dh, heads=heads, ff_mult=4, t5_name="synth-512",
                              precision="bf16")
    vae = M.VQGanVAE(dim=64, codebook_size=65536, precision="bf16")
    mg = M.MaskGit(image_size=256, transformer=tr.cuda(), vae=vae.cuda()).cuda()
    te = torch.randn((args.batch, 32, 512), generator=torch.Generator().manual_seed(1)).cuda()
    tr.encode_text = lambda texts, te=te: te
    mg.sampler_seed = 3
    mg.generate(texts=["a"] * args.batch, timesteps=18)          # warm-up: packing, workspaces, graph capture
    models[f"{heads}x{dh}"] = mg
for r in range(args.rounds):
    for key, mg in models.items():
        torch.cuda.synchronize()
        a_, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a_.record()
        mg.generate(texts=["a"] * args.batch, timesteps=18)
        b_.record()
        torch.cuda.synchronize()
        ips = args.batch / (a_.elapsed_time(b_) * 1e-3)
        results["generate"].append(dict(round=r, layout=key, images_per_s=ips))
        print(f"generate C3 architecture, {key} heads, batch {args.batch}, round {r}: {ips:.2f} images/s")
if args.out:
    with open(args.out, "w") as f:
        json.dump(results, f, indent=1)

"""The VAE decoder's convolutions at C3 (bench.py: 64 images, 16 x 16 latents, dim 256, bf16) in this tree's libmmg.so against another
build of the library (--parent-lib, e.g. a parent revision built into a side directory), alternated in one process.

Every mmg_conv2d / mmg_conv_transpose2d call of one VQGanVAE.decode_from_ids is recorded with its tensors and replayed on its own:
best of --iters with an L2 flush before each, per build and round, and TFLOP/s from the shapes.  The products' outputs of the two builds
are compared (bytes, and max |diff| for the fused RGB projection, whose fp32 sum the change may reorder).  decode_from_ids is timed whole
the same way.  The card's name, power limit and SM clocks are read in the same process.
usage: python scripts/vae_decode_bench.py --parent-lib DIR/libmmg.so [--rounds 3] [--iters 20] [--out results.json]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import muse_maskgit_pytorch_b200 as M  # noqa: E402
from muse_maskgit_pytorch_b200 import _lib, ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--parent-lib", required=True, help="the other build of libmmg.so")
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--latent", type=int, default=16)
ap.add_argument("--out", default="")
args = ap.parse_args()
assert torch.cuda.is_available(), "vae_decode_bench.py measures on the GPU; there is no CPU fallback"
torch.set_grad_enabled(False)


def smi():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


# the two builds: _lib.lib() returns whichever handle _lib._lib holds
libs = {"change": _lib.lib()}
_lib._lib, _lib.LIB_PATH = None, os.path.abspath(args.parent_lib)
libs["parent"] = _lib.lib()
assert ctypes.cast(libs["parent"]._handle, ctypes.c_void_p).value != ctypes.cast(libs["change"]._handle, ctypes.c_void_p).value


def use(name):
    _lib._lib = libs[name]


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


torch.manual_seed(0)
vae = M.VQGanVAE(precision="bf16", dim=256, codebook_size=65536).cuda()
ids = torch.randint(0, 65536, (args.batch, args.latent, args.latent), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))

# record the decoder's convolutions (inputs cloned: the decoder reuses nothing, but a replay must not depend on later writes)
calls = []
conv2d, conv_t = ops.conv2d, ops.conv_transpose2d


def rec2d(x, w, out, B, H, W, Cin, Cout, kind, **kw):
    calls.append(("conv2d", (x.clone(), w, out, B, H, W, Cin, Cout, kind), kw))
    return conv2d(x, w, out, B, H, W, Cin, Cout, kind, **kw)


def rec_t(x, w, out, B, H, W, Cin, Cout, **kw):
    calls.append(("conv_t", (x.clone(), w, out, B, H, W, Cin, Cout), kw))
    return conv_t(x, w, out, B, H, W, Cin, Cout, **kw)


use("change")
ops.conv2d, ops.conv_transpose2d = rec2d, rec_t
vae.decode_from_ids(ids)
ops.conv2d, ops.conv_transpose2d = conv2d, conv_t
torch.cuda.synchronize()


def describe(op, a, kw):
    x, w, out, B, H, W, Cin, Cout = a[:8]
    if op == "conv2d":
        kind = a[8]
        taps = {0: 1, 1: 9, 2: 16, 3: 25}[kind]
        ho, wo = (H // 2, W // 2) if kind == 2 else (H, W)
        epi = {ops.EPI_GLU: "GLU", ops.EPI_RESIDUAL: "residual"}.get(kw.get("epilogue", ops.EPI_STORE), "store")
        name = f"conv{ {0: '1x1', 1: '3x3', 2: '4x4s2', 3: '5x5'}[kind]} {Cin}->{Cout} {epi} @{H}x{W}"
        return name, 2.0 * B * ho * wo * Cout * taps * Cin
    name = f"convT {Cin}->{Cout}{' + RGB' if kw.get('rgb_w') is not None else ''} @{H}x{W}"
    return name, 2.0 * 4 * B * H * W * Cout * 4 * Cin


def run(op, a, kw):
    return (conv2d if op == "conv2d" else conv_t)(*a, **kw)


card = smi()
print(f"# {card}", flush=True)
prods = []
for op, a, kw in calls:
    name, flop = describe(op, a, kw)
    outs = {}
    for b in ("parent", "change"):
        use(b)
        a[2].zero_()
        run(op, a, kw)
        torch.cuda.synchronize()
        outs[b] = a[2].clone()
    rgb = kw.get("rgb_w") is not None
    same = torch.equal(outs["parent"].view(torch.uint8), outs["change"].view(torch.uint8))
    maxd = float((outs["parent"].float() - outs["change"].float()).abs().max())
    prods.append(dict(name=name, gflop=flop / 1e9, rgb=rgb, bitwise_equal=bool(same), max_abs_diff=maxd, ms={"parent": [], "change": []}))
dec = {"parent": [], "change": []}
for r in range(args.rounds):
    for b in (("parent", "change") if r % 2 == 0 else ("change", "parent")):
        use(b)
        for (op, a, kw), pr in zip(calls, prods):
            pr["ms"][b].append(best_ms(lambda: run(op, a, kw), args.iters))
        dec[b].append(best_ms(lambda: vae.decode_from_ids(ids), max(3, args.iters // 4)))

print(f"{'product':44s} {'GFLOP':>8s} {'parent us':>10s} {'TFLOP/s':>8s} {'change us':>10s} {'TFLOP/s':>8s} {'speedup':>8s}  outputs")
for pr in prods:
    p, c = min(pr["ms"]["parent"]), min(pr["ms"]["change"])
    pr.update(parent_us=p * 1e3, change_us=c * 1e3, parent_tflops=pr["gflop"] / p, change_tflops=pr["gflop"] / c,
              speedup=p / c, parent_spread_us=(max(pr["ms"]["parent"]) - p) * 1e3, change_spread_us=(max(pr["ms"]["change"]) - c) * 1e3)
    eq = "bitwise equal" if pr["bitwise_equal"] else f"max |diff| {pr['max_abs_diff']:.3e}"
    print(f"{pr['name']:44s} {pr['gflop']:8.1f} {pr['parent_us']:10.1f} {pr['parent_tflops']:8.1f} {pr['change_us']:10.1f} {pr['change_tflops']:8.1f} "
          f"{pr['speedup']:8.2f}  {eq}")
print(f"decode_from_ids ({args.batch} x {args.latent}^2): parent {min(dec['parent']):.2f} ms {sorted(dec['parent'])}, "
      f"change {min(dec['change']):.2f} ms {sorted(dec['change'])}")
print(f"# {smi()}", flush=True)
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(dict(card=card, batch=args.batch, latent=args.latent, products=prods, decode_ms=dec), f, indent=1)

"""The bf16 wgmma attention calls of a generate() in this tree's libmmg.so against another build of the library (--parent-lib, e.g. a parent
revision built into a side directory), alternated in one process.

Shapes: the C3 self-attention (128 sequences = 64 images x CFG, 8 heads, 256 queries, 256 keys + the null key) and cross-attention (64 live
sequences, 32 text keys + the null key, per-sequence key mask), both single-pass as the model calls them (unit-norm q and k, logit bound
1.02, scale 8), and the C4 self-attention (64 sequences, 1024 queries, 1024 keys + null: 128-key blocks).  Per build and round: best of
--iters with an L2 flush before each call, TFLOP/s from 4 B H Tq Tk 64 and GB/s from the bytes of q, k, v, mask and out.  The outputs of the
two builds on the same seeded inputs are compared: how many elements are bitwise equal, and the largest difference in bf16 ulps.
The card's name, power limit and SM clocks are read in the same process.
usage: python scripts/attention_bench.py --parent-lib DIR/libmmg.so [--rounds 3] [--iters 20] [--out results.json]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from muse_maskgit_pytorch_b200 import _lib, ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--parent-lib", required=True, help="the other build of libmmg.so")
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--out", default="")
args = ap.parse_args()
assert torch.cuda.is_available(), "attention_bench.py measures on the GPU; there is no CPU fallback"
torch.set_grad_enabled(False)

HEADS, SCALE, BOUND = 8, 8.0, 1.02
# name, sequences, queries, keys including the null key, per-sequence key mask
SHAPES = [("C3 self   B=128 Tq=256 Tk=257", 128, 256, 257, False),
          ("C3 cross  B=64  Tq=256 Tk=33 masked", 64, 256, 33, True),
          ("C4 self   B=64  Tq=1024 Tk=1025", 64, 1024, 1025, False)]


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


def ordered(x):
    """bf16 bit patterns as integers in the order of the values they encode (adjacent bf16 values differ by 1)"""
    i = x.view(torch.int16).to(torch.int32)
    return torch.where(i < 0, -(i & 0x7FFF), i)


def case(B, Tq, Tk, masked, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    alloc = (Tk + 7) // 8 * 8
    q = F.normalize(torch.randn((B * HEADS, Tq, 64), device="cuda", generator=g), dim=-1).to(torch.bfloat16)
    k = torch.zeros((B * HEADS, alloc, 64), device="cuda", dtype=torch.bfloat16)
    k[:, :Tk] = F.normalize(torch.randn((B * HEADS, Tk, 64), device="cuda", generator=g), dim=-1).to(torch.bfloat16)
    v = torch.zeros_like(k)
    v[:, :Tk] = torch.randn((B * HEADS, Tk, 64), device="cuda", generator=g).to(torch.bfloat16)
    km = (torch.rand((B, Tk - 1), device="cuda", generator=g) > 0.2).to(torch.uint8) if masked else None
    if masked:
        km[0] = 0                                    # one fully masked sequence: its output is the null value
    out = torch.empty((B * Tq, HEADS * 64), device="cuda", dtype=torch.bfloat16)
    return q, k, v, km, out


card = smi()
print(f"# {card}", flush=True)
rows = []
for i, (name, B, Tq, Tk, masked) in enumerate(SHAPES):
    q, k, v, km, out = case(B, Tq, Tk, masked, 100 + i)
    def fn(q=q, k=k, v=v, km=km, out=out, B=B, Tk=Tk):
        ops.attention(q, k, v, out, B, HEADS, Tk, key_mask=km, scale=SCALE, logit_bound=BOUND)
    outs = {}
    for b in ("parent", "change"):
        use(b)
        out.fill_(float("nan"))
        fn()
        torch.cuda.synchronize()
        outs[b] = out.clone()
    eq = outs["parent"].view(torch.int16) == outs["change"].view(torch.int16)
    ulps = int((ordered(outs["parent"]) - ordered(outs["change"])).abs().max())
    flop = 4.0 * B * HEADS * Tq * Tk * 64
    nbytes = 2 * (q.numel() + 2 * B * HEADS * Tk * 64 + out.numel()) + (km.numel() if masked else 0)
    rows.append(dict(name=name, B=B, Tq=Tq, Tk=Tk, masked=masked, gflop=flop / 1e9, mbytes=nbytes / 1e6, elements=out.numel(),
                     bitwise_equal=int(eq.sum()), max_ulps=ulps, ms={"parent": [], "change": []}, fn=fn))
for r in range(args.rounds):
    for b in (("parent", "change") if r % 2 == 0 else ("change", "parent")):
        use(b)
        for row in rows:
            row["ms"][b].append(best_ms(row["fn"], args.iters))

print(f"{'call':38s} {'parent us':>10s} {'TFLOP/s':>8s} {'GB/s':>7s} {'change us':>10s} {'TFLOP/s':>8s} {'GB/s':>7s} {'speedup':>8s}  outputs")
for row in rows:
    del row["fn"]
    p, c = min(row["ms"]["parent"]), min(row["ms"]["change"])
    row.update(parent_us=p * 1e3, change_us=c * 1e3, speedup=p / c,
               parent_spread_us=(max(row["ms"]["parent"]) - p) * 1e3, change_spread_us=(max(row["ms"]["change"]) - c) * 1e3)
    diff = row["elements"] - row["bitwise_equal"]
    print(f"{row['name']:38s} {p * 1e3:10.1f} {row['gflop'] / p:8.1f} {row['mbytes'] / p:7.0f} {c * 1e3:10.1f} {row['gflop'] / c:8.1f} "
          f"{row['mbytes'] / c:7.0f} {p / c:8.2f}  {diff} of {row['elements']} differ, max {row['max_ulps']} bf16 ulp")
print(f"# {smi()}", flush=True)
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(dict(card=card, shapes=rows), f, indent=1)

"""The T5 text encoder's feed-forward products (mmg_linear with the GEGLU_TANH or STORE + ReLU epilogue, bf16) in this tree's libmmg.so
against another build of the library (--parent-lib, e.g. a parent revision built into a side directory), alternated in one process.

Each product runs at M = 64 * T rows (64 prompts of T tokens, T in --tokens) with seeded bf16 inputs: best of --iters with an L2 flush
before each, per build and round, and TFLOP/s from the shapes.  The two builds' outputs are compared byte for byte.  The card's name,
power limit and SM clocks are read in the same process.
usage: python scripts/t5_ff_bench.py --parent-lib DIR/libmmg.so [--rounds 3] [--iters 20] [--out results.json]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from muse_maskgit_pytorch_b200 import _lib, ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--parent-lib", required=True, help="the other build of libmmg.so")
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--tokens", type=int, nargs="+", default=[32, 128])
ap.add_argument("--out", default="")
args = ap.parse_args()
assert torch.cuda.is_available(), "t5_ff_bench.py measures on the GPU; there is no CPU fallback"
torch.set_grad_enabled(False)

# (name, epilogue, K, N): N counts the accumulator columns, so a GEGLU_TANH product writes N / 2 outputs per row
PRODUCTS = [
    ("t5-v1_1-base wi GEGLU_TANH", ops.EPI_GEGLU_TANH, 768, 4096),
    ("t5-v1_1-xl wi GEGLU_TANH", ops.EPI_GEGLU_TANH, 2048, 10240),
    ("t5-base wi ReLU", ops.EPI_STORE, 768, 3072),
    ("t5-small wi ReLU", ops.EPI_STORE, 512, 2048),
    ("ReLU, N % 128 == 64", ops.EPI_STORE, 512, 2112),
]


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


g = torch.Generator(device="cuda").manual_seed(0)
cases = []
for name, epi, K, N in PRODUCTS:
    w = (torch.randn((N, K), device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    for T in args.tokens:
        M = 64 * T
        x = torch.randn((M, K), device="cuda", generator=g).to(torch.bfloat16)     # RMS-normalised activations: unit scale
        out = torch.empty((M, N // 2 if epi == ops.EPI_GEGLU_TANH else N), device="cuda", dtype=torch.bfloat16)
        act = 2 if epi == ops.EPI_STORE else 0
        cases.append(dict(name=f"{name}, T {T}", M=M, K=K, N=N, gflop=2.0 * M * N * K / 1e9,
                          fn=lambda x=x, w=w, out=out, epi=epi, act=act: ops.linear(x, w, out, epi, act=act), out=out))

card = smi()
print(f"# {card}", flush=True)
for c in cases:
    outs = {}
    for b in ("parent", "change"):
        use(b)
        c["out"].fill_(float("nan"))
        c["fn"]()
        torch.cuda.synchronize()
        outs[b] = c["out"].clone()
    c["byte_equal"] = bool(torch.equal(outs["parent"].view(torch.int16), outs["change"].view(torch.int16)))
    c["ms"] = {"parent": [], "change": []}
for r in range(args.rounds):
    for b in (("parent", "change") if r % 2 == 0 else ("change", "parent")):
        use(b)
        for c in cases:
            c["ms"][b].append(best_ms(c["fn"], args.iters))

print(f"{'product':40s} {'M':>6s} {'K':>5s} {'N':>6s} {'parent us':>10s} {'spread':>7s} {'TFLOP/s':>8s} {'change us':>10s} {'spread':>7s} "
      f"{'TFLOP/s':>8s} {'speedup':>8s}  outputs")
rows = []
for c in cases:
    p, ch = min(c["ms"]["parent"]), min(c["ms"]["change"])
    row = dict(name=c["name"], M=c["M"], K=c["K"], N=c["N"], gflop=c["gflop"], byte_equal=c["byte_equal"], ms=c["ms"],
               parent_us=p * 1e3, change_us=ch * 1e3, parent_tflops=c["gflop"] / p, change_tflops=c["gflop"] / ch, speedup=p / ch,
               parent_spread_us=(max(c["ms"]["parent"]) - p) * 1e3, change_spread_us=(max(c["ms"]["change"]) - ch) * 1e3)
    rows.append(row)
    print(f"{row['name']:40s} {row['M']:6d} {row['K']:5d} {row['N']:6d} {row['parent_us']:10.1f} {row['parent_spread_us']:7.1f} "
          f"{row['parent_tflops']:8.1f} {row['change_us']:10.1f} {row['change_spread_us']:7.1f} {row['change_tflops']:8.1f} "
          f"{row['speedup']:8.3f}  {'byte-equal' if row['byte_equal'] else 'DIFFERENT'}")
print(f"# {smi()}", flush=True)
if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(dict(card=card, card_end=smi(), products=rows), f, indent=1)

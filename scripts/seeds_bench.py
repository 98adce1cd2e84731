"""Per-image seeds at the C3 workload of bench.py (256 x 256, top-k 0.9, 18 steps, B = 64, random weights, whole-call CUDA graphs).

Parts:
  generate   generate() without and with image_seeds (new seeds every call, one captured graph per arm), the two arms alternated over
             --rounds rounds of --calls calls each; images/s of every call, median and range per arm.
  critic     the token critic's per-row (seed, position) table of a C3 call: 64 * 256 = 16 384 rows of 16 bytes (256 KiB), expanded on the
             device from the uploaded [64] seeds (512 bytes); device time of the expansion by CUDA events over 200 repetitions.
The card, its power limit and SM clocks are read in the same run.
usage: python scripts/seeds_bench.py [--rounds 5] [--calls 3] [--out seeds_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def summary(ms, batch):
    ips = sorted(batch / (v / 1e3) for v in ms)
    return dict(images_per_s=[round(v, 1) for v in ips], median=round(ips[len(ips) // 2], 1), min=round(ips[0], 1), max=round(ips[-1], 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "seeds_bench.py measures on the GPU; there is no CPU fallback"
    import bench
    from muse_maskgit_pytorch_b200.muse_maskgit import _seed_bits
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, T = bench.GLOBAL_BATCH, bench.TIMESTEPS
    gpu = card()
    print(f"# {gpu}", flush=True)
    mg = bench.build_models(dev)
    mg.sampler_seed = 2
    te = bench.text_embeddings(B).to(dev)
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    texts = [""] * B
    gen = lambda seeds: mg.generate(texts, timesteps=T, topk_filter_thres=0.9, image_seeds=seeds)
    out = dict(gpu=gpu, batch=B, timesteps=T)

    # ---- generate without / with per-image seeds, alternated
    gen(None); gen(1)                                                # both graphs captured outside the timing
    graphs = len(mg._graphs)
    ms = {"without": [], "with": []}
    call = 0
    for _ in range(args.rounds):
        for arm in ("without", "with"):
            for _ in range(args.calls):
                call += 1
                ms[arm].append(timed(lambda: gen(None if arm == "without" else call * B)))
    assert len(mg._graphs) == graphs, "new seeds re-captured a graph"
    out["generate"] = {arm: summary(v, B) for arm, v in ms.items()}
    print(json.dumps(dict(part="generate", **out["generate"])), flush=True)

    # ---- the critic's per-row key table at C3
    n = bench.TR_CFG["seq_len"]
    seeds = _seed_bits(range(B)).to(dev)
    pos = torch.arange(n, device=dev)
    expand = lambda: torch.stack((seeds[:, None].expand(B, n), pos.expand(B, n)), dim=-1)
    for _ in range(10):
        expand()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 200
    e0.record()
    for _ in range(reps):
        expand()
    e1.record()
    torch.cuda.synchronize()
    out["critic_row_key"] = dict(rows=B * n, table_bytes=B * n * 16, uploaded_bytes=B * 8, us_per_expansion=round(e0.elapsed_time(e1) * 1e3 / reps, 2))
    print(json.dumps(dict(part="critic_row_key", **out["critic_row_key"])), flush=True)
    out["gpu_after"] = card()
    print(f"# {out['gpu_after']}  (after the timed parts)", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()

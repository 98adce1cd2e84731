"""Per-image sampling settings at the C3 workload of bench.py (256 x 256, top-k 0.9, 18 steps, B = 64, random weights, whole-call CUDA graphs).

Parts:
  sweep      cond_scale cycled over 2, 3, 4, 5, 6 twice.  Arm "cache_miss" clears MaskGit._graphs before every call (what a graph key holding
             the setting costs: an eager warm-up and a capture per new value); arm "replay" keeps the one graph.  ms per call, graphs held
             and torch.cuda.max_memory_reserved after each arm.
  mixed      one call of 64 images in four groups of 16 with different (cond_scale, temperature) against four calls of 16 (graphs warm).
  uniform    with --parent DIR (a checkout of another revision, built): `bench.py --gpus 1 --no-extras` of DIR and of this tree alternated,
             --rounds each, images/s of every run.
The card, its power limit and SM clocks are read in the same run.
usage: python scripts/settings_bench.py [--parent DIR] [--rounds 2] [--out settings_bench.json]"""
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


def bench_images_per_s(tree):
    tree = os.path.abspath(tree)
    r = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--no-extras"], capture_output=True, text=True, cwd=tree)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py in {tree} failed ({r.returncode}): {r.stderr[-2000:]}")
    return json.loads(lines[-1])["value"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "settings_bench.py measures on the GPU; there is no CPU fallback"
    import bench
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
    gen = lambda n=B, **s: mg.generate(texts[:n], timesteps=T, topk_filter_thres=0.9, **s)
    out = dict(gpu=gpu, batch=B, timesteps=T)

    # ---- sweep
    scales = [2, 3, 4, 5, 6] * 2
    sweep = {}
    for arm in ("cache_miss", "replay"):
        mg._graphs.clear()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        gen(cond_scale=scales[0])                                  # the replay arm's one capture happens here, outside the timing
        ms = []
        for s in scales:
            if arm == "cache_miss":
                mg._graphs.clear()
            ms.append(timed(lambda: gen(cond_scale=s)))
        sweep[arm] = dict(ms_per_call=[round(v, 1) for v in ms], mean_ms=round(sum(ms) / len(ms), 1), graphs_held=len(mg._graphs),
                          max_memory_reserved_gib=round(torch.cuda.max_memory_reserved() / 2 ** 30, 2))
        print(json.dumps(dict(part="sweep", arm=arm, **sweep[arm])), flush=True)
    out["sweep"] = sweep

    # ---- mixed batch of four groups against four calls of 16
    groups = [(2.0, 1.0), (3.0, 0.7), (4.5, 1.2), (6.0, 0.5)]
    g = B // len(groups)
    cs = [c for c, _ in groups for _ in range(g)]
    tp = [t for _, t in groups for _ in range(g)]
    mixed = lambda: gen(cond_scale=cs, temperature=tp)
    split = lambda: [gen(g, cond_scale=c, temperature=t) for c, t in groups]
    mixed(); split()
    rows = {"one_call_64": [], "four_calls_16": []}
    for _ in range(5):
        rows["one_call_64"].append(timed(mixed))
        rows["four_calls_16"].append(timed(split))
    out["mixed"] = {k: dict(ms=[round(v, 1) for v in vs], median_ms=round(sorted(vs)[len(vs) // 2], 1),
                            images_per_s=round(B / (sorted(vs)[len(vs) // 2] / 1e3), 1)) for k, vs in rows.items()}
    print(json.dumps(dict(part="mixed", **out["mixed"])), flush=True)
    del mg
    torch.cuda.empty_cache()

    # ---- uniform scalar call: the bench.py of another revision and of this tree, alternated
    if args.parent:
        runs = {"parent": [], "this": []}
        for _ in range(args.rounds):
            runs["parent"].append(bench_images_per_s(args.parent))
            runs["this"].append(bench_images_per_s(ROOT))
        out["uniform"] = runs
        print(json.dumps(dict(part="uniform", **runs)), flush=True)
    out["gpu_after"] = card()
    print(f"# {out['gpu_after']}  (after the timed parts)", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()

"""Per-image timesteps and top-k threshold at the C3 workload of bench.py (256 x 256, B = 64, random weights, whole-call CUDA graphs).

Arms, each timed as whole-call graph replays (every arm runs on its own MaskGit view of the same weights, so its graphs stay resident:
one MaskGit keeps 4, and the arms need 7), alternated over --rounds after one warm-up call per arm; the script asserts that no timed call
captured a graph:
  mixed      one call of 64 images mixing timesteps in {8, 12, 18} and topk_filter_thres in {0.9, 0.95, 0.98} (nine groups)
  separate   the same requests issued as one uniform call per (timesteps, threshold) group (nine calls; 4 graphs, the threshold is data)
  uniform    64 images, 18 steps, threshold 0.9
  one_0_85   the same with one image at topk_filter_thres = 0.85: its k (9831 of 65536) does not fit the fused tail's candidate lists, so
             the whole call runs on materialised logits and the row-walking kernel
With --parent DIR (a checkout of another revision, built): `bench.py --gpus 1 --no-extras` of DIR and of this tree alternated.
The card, its power limit and SM clocks are read in the same run.
usage: python scripts/mixed_batch_bench.py [--parent DIR] [--rounds 5] [--out mixed_batch_bench.json]"""
import argparse
import copy
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from settings_bench import bench_images_per_s, card, timed  # noqa: E402

STEPS = (8, 12, 18)
THRES = (0.9, 0.95, 0.98)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mixed_batch_bench.py measures on the GPU; there is no CPU fallback"
    import bench
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = bench.GLOBAL_BATCH
    print(f"# {card()}", flush=True)
    mg = bench.build_models(dev)
    te = bench.text_embeddings(B).to(dev)
    texts = [""] * B
    groups = [(T, th) for T in STEPS for th in THRES]
    assign = [groups[i % len(groups)] for i in range(B)]
    seeds = list(range(B))
    steps, thres = [a[0] for a in assign], [a[1] for a in assign]
    mg_of = [mg]                                            # the MaskGit view of the arm being run

    def mixed():
        mg_of[0].transformer.encode_text = lambda t: te[:len(t)]
        mg_of[0].generate(texts, timesteps=steps, topk_filter_thres=thres, cond_scale=bench.COND_SCALE, image_seeds=seeds)

    def separate():
        for g in groups:
            idx = [i for i, a in enumerate(assign) if a == g]
            mg_of[0].transformer.encode_text = lambda t, idx=idx: te[idx]
            mg_of[0].generate([""] * len(idx), timesteps=g[0], topk_filter_thres=g[1], cond_scale=bench.COND_SCALE, image_seeds=[seeds[i] for i in idx])

    def uniform():
        mg_of[0].transformer.encode_text = lambda t: te[:len(t)]
        mg_of[0].generate(texts, timesteps=18, topk_filter_thres=0.9, cond_scale=bench.COND_SCALE, image_seeds=seeds)

    def one_wide():
        mg_of[0].transformer.encode_text = lambda t: te[:len(t)]
        mg_of[0].generate(texts, timesteps=18, topk_filter_thres=[0.85] + [0.9] * (B - 1), cond_scale=bench.COND_SCALE, image_seeds=seeds)

    arms = dict(mixed=mixed, separate=separate, uniform=uniform, one_0_85=one_wide)
    views = {name: copy.copy(mg) for name in arms}          # shallow: shared weights and packs, one graph cache per arm
    for v in views.values():
        v._graphs = {}
    for name, fn in arms.items():
        mg_of[0] = views[name]
        fn()                                                # warm-up: captures the arm's graphs
    graphs = {name: {id(e.graph) for e in v._graphs.values()} for name, v in views.items()}
    res = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            mg_of[0] = views[name]
            res[name].append(timed(fn))
    for name, v in views.items():                           # every timed call was a replay of a graph captured in the warm-up
        assert {id(e.graph) for e in v._graphs.values()} == graphs[name], f"{name}: a timed call captured a graph"
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    out = dict(card=card(), batch=B, ms=res, median_ms=med, graphs={k: len(v) for k, v in graphs.items()})
    print(f"mixed call {med['mixed']:.1f} ms vs {len(groups)} separate calls {med['separate']:.1f} ms")
    print(f"18 steps, thres 0.9: {med['uniform']:.1f} ms; one image at 0.85 (materialised route): {med['one_0_85']:.1f} ms")
    if args.parent:
        ips = {"parent": [], "this": []}
        for _ in range(args.rounds):
            ips["parent"].append(bench_images_per_s(args.parent))
            ips["this"].append(bench_images_per_s(ROOT))
        out["bench_images_per_s"] = ips
        print(f"bench.py images/s parent {ips['parent']} this {ips['this']}")
    out["card_after"] = card()
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

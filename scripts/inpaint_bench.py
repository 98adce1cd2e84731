"""Time MaskGit.inpaint against MaskGit.generate at the C3 workload of bench.py (256 x 256, 18 steps, cond_scale 3, top-k 0.9, B = 64, random
weights, whole-call CUDA graphs): masks regenerating 100 %, 50 % and 25 % of the 16 x 16 tokens of every image, and a ragged per-image mix
(0 to 100 %, one image fully masked).  The block stack costs what it costs in generate() (every token attends); only the sampling tail scales
with the sampled rows, so this measures how much a small mask saves.

The arms alternate within each round (generate, then each mask), CUDA events around --calls back-to-back calls per arm and round, median over
--rounds rounds.  Also reports libmmg launches per call from one eager call per arm, checks that the 100 % mask gives generate()'s tokens,
and prints the card, its power limit and SM clocks with the numbers.
usage: python scripts/inpaint_bench.py [--rounds 5] [--calls 3] [--out inpaint_bench.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def masks(b, f, seed=0):
    """token masks (b, f, f), True = regenerate"""
    full = torch.ones((b, f, f), dtype=torch.bool)
    half = torch.zeros((b, f, f), dtype=torch.bool); half[:, :, : f // 2] = True
    quarter = torch.zeros((b, f, f), dtype=torch.bool); quarter[:, f // 4: 3 * f // 4, f // 4: 3 * f // 4] = True
    g = torch.Generator().manual_seed(seed)
    frac = torch.rand((b,), generator=g)
    frac[0], frac[1] = 1.0, 0.0
    ragged = torch.rand((b, f, f), generator=g) < frac[:, None, None]
    ragged[0] = True
    return {"mask_100": full, "mask_50": half, "mask_25": quarter, "mask_ragged": ragged}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "inpaint_bench.py measures on the GPU; there is no CPU fallback"
    import bench
    from muse_maskgit_pytorch_b200 import _lib
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, T = bench.GLOBAL_BATCH, bench.TIMESTEPS
    mg = bench.build_models(dev)
    mg.sampler_seed = 2
    te = bench.text_embeddings(B).to(dev)
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    texts = [""] * B
    kw = dict(timesteps=T, cond_scale=bench.COND_SCALE, temperature=1., topk_filter_thres=0.9)
    images = torch.rand((B, 3, bench.IMAGE, bench.IMAGE), generator=torch.Generator().manual_seed(3)).to(dev)
    f = mg.vae.get_encoded_fmap_size(bench.IMAGE)
    ms_ = {k: v.to(dev) for k, v in masks(B, f).items()}
    arms = {"generate": lambda: mg.generate(texts, return_ids=True, **kw)}
    for name, m in ms_.items():
        arms[name] = (lambda m: lambda: mg.inpaint(texts, images, m, return_ids=True, **kw))(m)
    gpu = card()
    print(f"# {gpu}", flush=True)

    launches = {}
    mg.use_cuda_graph = False
    for name, fn in arms.items():
        fn()
        torch.cuda.synchronize()
        l0 = _lib.launch_count()
        fn()
        torch.cuda.synchronize()
        launches[name] = _lib.launch_count() - l0
    mg.use_cuda_graph = True
    outs = {name: fn() for name, fn in arms.items()}             # capture + warm-up of every graph
    same = bool(torch.equal(outs["generate"][1], outs["mask_100"][1]) and torch.equal(outs["generate"][0], outs["mask_100"][0]))
    torch.cuda.synchronize()

    times = {name: [] for name in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.calls):
                fn()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b) / args.calls)
    rows = []
    for name in arms:
        ms = statistics.median(times[name])
        n_regen = B * f * f if name == "generate" else int(ms_[name].sum())
        r = dict(arm=name, B=B, timesteps=T, ms_per_call=round(ms, 2), images_per_s=round(B / ms * 1e3, 1),
                 ms_spread=[round(min(times[name]), 2), round(max(times[name]), 2)], regenerated_token_share=round(n_regen / (B * f * f), 3),
                 libmmg_launches_per_call=launches[name], gpu=gpu)
        rows.append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps(dict(full_mask_equals_generate=same)), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(rows=rows, full_mask_equals_generate=same, gpu=gpu), fh, indent=1)
    print(f"# {card()}  (after the timed rounds)", flush=True)


if __name__ == "__main__":
    main()

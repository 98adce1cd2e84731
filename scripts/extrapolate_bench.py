"""Time MaskGit.extrapolate (image extrapolation) against the chain of inpaint() calls a user writes without it, at the C3 workload of
bench.py (256 x 256 frame, 16 x 16 tokens, CFG 3, top-k 0.9, B = 64, random weights, precomputed text embeddings, whole-call CUDA graphs),
with extrapolate's defaults (stride f // 2 = 8 tokens, 18 steps per window).

Workloads: 256 x 256 -> 256 x 512 ("right", K = 2 windows), -> 256 x 1024 ("right", K = 6), -> 512 x 256 ("down", K = 2).
Arms:
  extrapolate  one extrapolate() call: K windows on the device-resident token canvas, one VAE decode of the whole canvas;
  chain        per window, inpaint() of the 256 x 256 crop whose far `stride` token columns (rows) are new and masked, the rest the last
               pixels of the panorama so far; then the crop's new strip of pixels is pasted onto the panorama (K encodes and decodes).
The arms alternate within each round, CUDA events around --calls back-to-back calls per arm and round; the median and range over --rounds
rounds.  Also reports libmmg launches per eager call, the peak memory of each arm, the growth of mmg_simt_launch_count over an eager
extrapolate() call (CUDA-core matrix-product / attention launches), the chain's drift (known-context tokens of a round whose re-encoded id
differs from the id the previous round produced at that position) and the card, its power limit and SM clocks read in the same run.
usage: python scripts/extrapolate_bench.py [--rounds 5] [--calls 1] [--out extrapolate_bench.json]"""
import argparse
import inspect
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = (("256x512", "right", 256), ("256x1024", "right", 768), ("512x256", "down", 256))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def chain(mg, texts, images, direction, amount, stride, kw, drift=None):
    """The inpaint chain for "right" / "down": returns (panorama, ids of each round); drift (list) receives each round's changed context."""
    p = mg.vae.dim_divisor
    f = mg.vae.get_encoded_fmap_size(mg.image_size)
    S, sp = mg.image_size, stride * p
    down = direction == "down"
    pano = images
    mask = torch.zeros((images.shape[0], f, f), dtype=torch.bool, device=images.device)
    if down:
        mask[:, f - stride:, :] = True
    else:
        mask[:, :, f - stride:] = True
    prev, rounds = mg.vae.encode_ids(images), []
    for _ in range(amount // sp):
        ctx = pano[:, :, -(S - sp):, :] if down else pano[:, :, :, -(S - sp):]
        crop = torch.cat((ctx, torch.zeros_like(ctx[:, :, :sp] if down else ctx[..., :sp])), dim=2 if down else 3)
        out, ids = mg.inpaint(texts, crop, mask, return_ids=True, **kw)
        if drift is not None:         # context of this round vs the ids at those positions in the previous round's output
            now = ids[:, :f - stride] if down else ids[:, :, :f - stride]
            was = prev[:, -(f - stride):] if down else prev[:, :, -(f - stride):]
            drift.append(int((now != was).sum()))
        strip = out[:, :, -sp:] if down else out[..., -sp:]
        pano = torch.cat((pano, strip), dim=2 if down else 3)
        prev = ids
        rounds.append(ids)
    return pano, rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "extrapolate_bench.py measures on the GPU; there is no CPU fallback"
    import bench
    from muse_maskgit_pytorch_b200 import _lib
    from muse_maskgit_pytorch_b200.muse_maskgit import MaskGit
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = bench.GLOBAL_BATCH
    timesteps = inspect.signature(MaskGit.extrapolate).parameters["timesteps"].default
    mg = bench.build_models(dev)
    mg.sampler_seed = 2
    te = bench.text_embeddings(B).to(dev)
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    texts = [""] * B
    kw = dict(cond_scale=bench.COND_SCALE, temperature=1., topk_filter_thres=0.9, timesteps=timesteps)
    images = torch.rand((B, 3, bench.IMAGE, bench.IMAGE), generator=torch.Generator().manual_seed(3)).to(dev)
    f = mg.vae.get_encoded_fmap_size(bench.IMAGE)
    stride = f // 2
    gpu = card()
    print(f"# {gpu}", flush=True)
    rows, extra = [], {}
    for name, direction, amount in WORKLOADS:
        arms = {"extrapolate": lambda: mg.extrapolate(texts, images, direction=direction, amount=amount, return_ids=True, **kw),
                "chain": lambda: chain(mg, texts, images, direction, amount, stride, kw)}
        info = dict(windows=amount // (stride * mg.vae.dim_divisor), stride=stride, timesteps=timesteps)
        mg.use_cuda_graph = False
        launches = {}
        for arm, fn in arms.items():
            fn()
            torch.cuda.synchronize()
            l0, s0 = _lib.launch_count(), _lib.simt_launch_count()
            fn()
            torch.cuda.synchronize()
            launches[arm] = _lib.launch_count() - l0
            if arm == "extrapolate":
                info["simt_launches_per_eager_extrapolate"] = _lib.simt_launch_count() - s0
        mg.use_cuda_graph = True
        peak = {}
        for arm, fn in arms.items():                       # capture + warm-up of every graph, then the arm's peak memory
            fn()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            peak[arm] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        drift = []
        chain(mg, texts, images, direction, amount, stride, kw, drift)
        info.update(chain_drift_per_round=drift, context_tokens_per_round=B * f * (f - stride))
        times = {arm: [] for arm in arms}
        for _ in range(args.rounds):
            for arm, fn in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.calls):
                    fn()
                b.record()
                b.synchronize()
                times[arm].append(a.elapsed_time(b) / args.calls)
        for arm in arms:
            ms = statistics.median(times[arm])
            row = dict(workload=name, direction=direction, arm=arm, B=B, ms_per_call=round(ms, 1), panoramas_per_s=round(B / ms * 1e3, 1),
                       ms_range=[round(min(times[arm]), 1), round(max(times[arm]), 1)], libmmg_launches_per_eager_call=launches[arm],
                       peak_memory_gib=peak[arm], gpu=gpu)
            rows.append(row)
            print(json.dumps(row), flush=True)
        extra[name] = info
        print(json.dumps(dict(workload=name, **info)), flush=True)
        mg._graphs.clear()
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(rows=rows, workloads=extra, gpu=gpu), fh, indent=1)
    print(f"# {card()}  (after the timed rounds)", flush=True)


if __name__ == "__main__":
    main()

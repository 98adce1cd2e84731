"""Time the sharded editing entry points and the sharded cascade over the GPUs of one node, one JSON line per workload:
  inpaint_sharded  C3 (256 x 256, 18 steps, cond_scale 3, top-k 0.9, global batch 64), a left-half mask and a ragged per-image mask;
  edit_sharded     C3 with edit's defaults (8 iterations x 4 steps on 10 % of the tokens), global batch 64;
  muse_sharded     the C3 base model -> the C4 super-resolution model (512 x 512 conditioned on 256 x 256), 18 + 18 steps, global batch 32.
Random weights, whole-call CUDA graphs, text embeddings resident on the device.  Every shape is warmed up (graph capture included)
before its timed window: barrier + synchronize, CUDA events around --calls back-to-back calls, the slowest rank's time.  The card's
name and power limit are read in the same run.

usage: python -m torch.distributed.run --nproc-per-node N scripts/sharded_bench.py [--calls 3] [--warmup 2] [--out DIR/sharded.json]
(N = 1 gives the one-GPU rows.)"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(index):
    q = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(index)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sharded_bench.py measures on the GPU; there is no CPU fallback"
    import bench
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import parallel
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    from inpaint_bench import masks
    dist, rank, world, local, device = bench.dist_setup()
    gpu = card(local)
    B, T, cs = bench.GLOBAL_BATCH, bench.TIMESTEPS, bench.COND_SCALE
    kw = dict(timesteps=T, cond_scale=cs, temperature=1., topk_filter_thres=0.9)
    mg = bench.build_models(device)
    te = bench.text_embeddings(B).to(device)
    texts = [""] * B
    images = torch.rand((B, 3, bench.IMAGE, bench.IMAGE), generator=torch.Generator().manual_seed(3)).to(device)
    f = mg.vae.get_encoded_fmap_size(bench.IMAGE)
    ms_ = {k: v.to(device) for k, v in masks(B, f).items()}
    sr = bench.build_models(device, superres=True)
    muse = M.Muse(base=mg, superres=sr)
    Bm = 32
    arms = {
        "inpaint_sharded C3, left-half mask": (B, lambda: parallel.inpaint_sharded(mg, texts, images, ms_["mask_50"], text_embeds=te, seed=2, **kw)),
        "inpaint_sharded C3, ragged mask": (B, lambda: parallel.inpaint_sharded(mg, texts, images, ms_["mask_ragged"], text_embeds=te, seed=2, **kw)),
        "edit_sharded C3, 8 x 4 steps on 10 %": (B, lambda: parallel.edit_sharded(mg, texts, images, text_embeds=te, seed=2, cond_scale=cs)),
        "muse_sharded C3 -> C4, 18 + 18 steps": (Bm, lambda: parallel.muse_sharded(muse, texts[:Bm], text_embeds=te[:Bm], cond_scale=cs,
                                                                                  timesteps=T, return_pil_images=False)),
    }
    mg.sampler_seed = sr.sampler_seed = 2
    rows = []
    for name, (batch, fn) in arms.items():
        for _ in range(max(args.warmup, 1)):
            fn()
        ms, _ = bench.timed_loop(dist, world, device, fn, args.calls)
        row = dict(workload=name, n_gpus=world, global_batch=batch, ms_per_call=round(ms, 2), images_per_s=round(batch / ms * 1e3, 2),
                   calls=args.calls, gpu=gpu)
        rows.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
    if rank == 0:
        print(f"# {card(local)}  (after the timed rounds)", flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as fh:
                json.dump(dict(rows=rows, gpu=gpu), fh, indent=1)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    with torch.no_grad():
        main()

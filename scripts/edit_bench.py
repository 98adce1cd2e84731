"""Time MaskGit.edit (mask-free editing) against MaskGit.generate and against the pixel-chained equivalent at the C3 workload of bench.py
(256 x 256, CFG 3, top-k 0.9, B = 64, random weights, whole-call CUDA graphs), with edit's default iterations / fraction / timesteps.

Arms:
  generate   generate() with bench.py's 18 steps;
  edit       edit(images) with the defaults (8 iterations of 4 steps on r_b = int(0.1 * 256) = 25 tokens per image);
  chained    `iterations` calls of inpaint(timesteps=4), each on the previous call's decoded images, each with a random token mask of
             r_b tokens per image (the pixel round trip a user has without edit).
The arms alternate within each round, CUDA events around --calls back-to-back calls per arm and round; the median and range over --rounds
rounds.  Also reports the chained arm's drift (tokens outside a round's mask whose id differs from the previous round's output: the VQGAN
round trip is not idempotent; edit keeps every unselected token by construction), libmmg launches per eager call of generate(), a full-mask
inpaint() at 18 steps and edit, and the card, its power limit and SM clocks read in the same run.
usage: python scripts/edit_bench.py [--rounds 5] [--calls 3] [--out edit_bench.json]"""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def random_masks(iterations, b, f, r, seed=0):
    """[iterations] (b, f, f) token masks with exactly r tokens per image, drawn uniformly."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(iterations):
        m = torch.zeros((b, f * f), dtype=torch.bool)
        m.scatter_(1, torch.rand((b, f * f), generator=g).argsort(dim=1)[:, :r], True)
        out.append(m.reshape(b, f, f))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "edit_bench.py measures on the GPU; there is no CPU fallback"
    import bench
    from muse_maskgit_pytorch_b200 import _lib
    from muse_maskgit_pytorch_b200.muse_maskgit import MaskGit
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, T = bench.GLOBAL_BATCH, bench.TIMESTEPS
    defaults = {k: v.default for k, v in inspect.signature(MaskGit.edit).parameters.items() if k in ("iterations", "fraction", "timesteps")}
    its, frac, te_steps = defaults["iterations"], defaults["fraction"], defaults["timesteps"]
    mg = bench.build_models(dev)
    mg.sampler_seed = 2
    te = bench.text_embeddings(B).to(dev)
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    texts = [""] * B
    kw = dict(cond_scale=bench.COND_SCALE, temperature=1., topk_filter_thres=0.9)
    images = torch.rand((B, 3, bench.IMAGE, bench.IMAGE), generator=torch.Generator().manual_seed(3)).to(dev)
    f = mg.vae.get_encoded_fmap_size(bench.IMAGE)
    r = max(int(frac * f * f), 1)
    chain_masks = [m.to(dev) for m in random_masks(its, B, f, r)]

    def chained():
        img, outs = images, []
        for m in chain_masks:
            img, ids = mg.inpaint(texts, img, m, timesteps=te_steps, return_ids=True, **kw)
            outs.append(ids)
        return img, outs

    arms = {"generate": lambda: mg.generate(texts, timesteps=T, return_ids=True, **kw),
            "edit": lambda: mg.edit(texts, images, return_ids=True, **kw),
            "chained_inpaint": chained}
    gpu = card()
    print(f"# {gpu}", flush=True)

    launch_calls = {"generate": arms["generate"], "inpaint_full_mask_18_steps":
                    lambda: mg.inpaint(texts, images, torch.ones((B, f, f), dtype=torch.bool, device=dev), timesteps=T, return_ids=True, **kw),
                    "edit": arms["edit"]}
    launches = {}
    mg.use_cuda_graph = False
    for name, fn in launch_calls.items():
        fn()
        torch.cuda.synchronize()
        l0 = _lib.launch_count()
        fn()
        torch.cuda.synchronize()
        launches[name] = _lib.launch_count() - l0
    mg.use_cuda_graph = True
    outs = {name: fn() for name, fn in arms.items()}             # capture + warm-up of every graph
    torch.cuda.synchronize()

    # drift of the chained arm: round j starts from encode_ids(decode(round j-1's ids)); tokens outside its mask should equal those ids
    ids0 = mg.vae.encode_ids(images)
    prev, drift = ids0, []
    for m, ids in zip(chain_masks, outs["chained_inpaint"][1]):
        drift.append(int(((ids != prev) & ~m).sum()))
        prev = ids
    ever = torch.stack(chain_masks).any(dim=0)
    drift_never_selected = int(((outs["chained_inpaint"][1][-1] != ids0) & ~ever).sum())
    edit_changed = int((outs["edit"][1] != ids0).sum())

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
        row = dict(arm=name, B=B, ms_per_call=round(ms, 2), images_per_s=round(B / ms * 1e3, 1),
                   ms_range=[round(min(times[name]), 2), round(max(times[name]), 2)], gpu=gpu)
        if name == "generate":
            row.update(timesteps=T)
        else:
            row.update(iterations=its, fraction=frac, timesteps=te_steps, tokens_per_round=r)
        rows.append(row)
        print(json.dumps(row), flush=True)
    extra = dict(libmmg_launches_per_eager_call=launches, chained_drift_per_round=drift, chained_drift_total=sum(drift),
                 chained_drift_never_selected=drift_never_selected, edit_tokens_changed=edit_changed, tokens=B * f * f)
    print(json.dumps(extra), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(rows=rows, gpu=gpu, **extra), fh, indent=1)
    print(f"# {card()}  (after the timed rounds)", flush=True)


if __name__ == "__main__":
    main()

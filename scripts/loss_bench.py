"""Time MaskGit.forward (the training loss, evaluated without gradients) at the C3 workload of bench.py: 256 x 256 images as 16 x 16 tokens,
dim 512, depth 8, heads 8, V = 65536, B = 64, random weights, 32 text tokens, fed as token ids.

Arms, alternating within each round, each call seeded the same way within a round (same masks, same labelled rows):
  fused         the default: to_logits + cross-entropy in mmg_logits_xent, no [rows, V] logits buffer
  materialised  use_fused_tail = False: mmg_linear writes the fp32 logits rows, mmg_logits_xent_rows reduces them
  self_critic   a self-token-critic model over the same weights: the critic branch materialises the labelled rows once, samples them over the
                full vocabulary and runs the critic stack
CUDA events around each call, median over --rounds rounds.  Then, per arm, torch.cuda.max_memory_allocated growth of one call, and in a separate
torch.profiler run the time of the mmg_logits_xent kernels (GEMM + merge) with its rate 2 R V K / time against the 989 TFLOP/s dense bf16 figure
of the H100 SXM data sheet.  Prints the card, its power limit and clocks with the numbers, and checks that the fused and materialised losses agree.
usage: python scripts/loss_bench.py [--rounds 7] [--out loss_bench.json]"""
import argparse
import json
import math
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "loss_bench.py measures on the GPU; there is no CPU fallback"
    import bench
    import muse_maskgit_pytorch_b200 as M
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = bench.GLOBAL_BATCH
    mg = bench.build_models(dev)
    te = bench.text_embeddings(B).to(dev)
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    mg_sc = M.MaskGit(image_size=bench.IMAGE, transformer=mg.transformer, vae=mg.vae, self_token_critic=True).to(dev)
    mg_sc.sampler_seed = 5
    tr = mg.transformer
    V, K = tr.num_tokens, tr.dim
    n = mg.vae.get_encoded_fmap_size(bench.IMAGE) ** 2
    ids = torch.randint(0, V, (B, n), generator=torch.Generator().manual_seed(1)).to(dev)
    texts = [""] * B

    def call(arm, seed):
        torch.manual_seed(seed)
        mg.use_fused_tail = arm != "materialised"
        return (mg_sc if arm == "self_critic" else mg)(ids, texts=texts)

    def labelled_rows(seed):          # the call's first draw is the per-sequence mask ratio; cosine schedule, rounded, at least 1
        torch.manual_seed(seed)
        return int((n * torch.cos(torch.zeros((B,), device=dev).uniform_(0, 1) * math.pi * 0.5)).round().clamp(min=1).sum())

    arms = ["fused", "materialised", "self_critic"]
    for arm in arms:                                                    # warm-up: packing, workspaces, cuBLAS-free first launches
        call(arm, 0)
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    rows = []
    agree = []
    for r in range(args.rounds):
        seed = 100 + r
        rows.append(labelled_rows(seed))
        losses = {}
        for arm in arms:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            losses[arm] = call(arm, seed)
            e.record()
            torch.cuda.synchronize()
            times[arm].append(s.elapsed_time(e))
        agree.append(abs(float(losses["fused"]) - float(losses["materialised"])) / abs(float(losses["materialised"])))
    mem = {}
    for arm in arms:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        call(arm, 100)
        torch.cuda.synchronize()
        mem[arm] = torch.cuda.max_memory_allocated() - base
    R = labelled_rows(100)
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call("fused", 100)
        torch.cuda.synchronize()
    us = {}
    for ev in prof.key_averages():
        if "tc_logits_kernel<true>" in ev.key or "logits_xent_merge_kernel" in ev.key:
            us[ev.key] = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    xent_ms = sum(us.values()) / 1e3
    tflops = 2 * R * V * K / (xent_ms * 1e-3) / 1e12 if xent_ms else float("nan")
    out = dict(card=card(), workload=f"MaskGit.forward at C3: B={B}, n={n}, V={V}, dim={K}, depth {len(tr.transformer_blocks.layers)}",
               rounds=args.rounds, labelled_rows_per_call=dict(median=statistics.median(rows), min=min(rows), max=max(rows)),
               ms_per_call={a: round(statistics.median(t), 3) for a, t in times.items()},
               ms_per_call_spread={a: [round(min(t), 3), round(max(t), 3)] for a, t in times.items()},
               peak_memory_growth_MiB={a: round(v / 2 ** 20, 1) for a, v in mem.items()},
               logits_bytes_of_R_rows_MiB=round(R * V * 4 / 2 ** 20, 1), profiled_rows=R,
               mmg_logits_xent_kernels_ms=round(xent_ms, 3), mmg_logits_xent_kernels=us,
               mmg_logits_xent_TFLOPs=round(tflops, 1), share_of_989_TFLOPs_bf16_datasheet=round(tflops / 989, 3),
               fused_vs_materialised_max_rel_loss_gap=max(agree))
    print(json.dumps(out, indent=1))
    assert max(agree) <= 1e-4, "fused and materialised losses disagree"
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

"""Per-kernel device time of the fused logits + sampling tail inside one eager generate() at C3 (bench.py's models, 256 x 256, 18 steps,
CFG 3, batch 64), from a torch.profiler capture of its own: tc_logits_kernel, the finisher, the threshold kernels and the wgmma GEMM
instantiations (the sample GEMM among them), with tc_logits_kernel's rate over the call's logits FLOPs.
usage: python scripts/logits_profile.py [--out DIR]   (DIR gets the kernel table as JSON)"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from muse_maskgit_pytorch_b200 import parallel  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", default="")
args = ap.parse_args()

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"# {torch.cuda.get_device_name()}  nvidia-smi name, power.limit, clocks.max.sm, clocks.sm: {smi}", flush=True)
dev = torch.device("cuda")
mg = bench.build_models(dev)
mg.use_cuda_graph = False
b = bench.GLOBAL_BATCH
te = bench.text_embeddings(b).to(dev)
kw = dict(timesteps=bench.TIMESTEPS, cond_scale=bench.COND_SCALE, temperature=1., topk_filter_thres=0.9)
run = lambda: parallel.generate_sharded(mg, [""] * b, text_embeds_shard=te, seed=2, **kw)
run(); run()
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    run()
    torch.cuda.synchronize()
tot = {a.key: [a.self_device_time_total / 1e3, a.count] for a in prof.key_averages() if a.self_device_time_total > 0}
all_ms = sum(v[0] for v in tot.values())
# rows sampled per call: max(int(cos(pi/2 * i / (T - 1)) * 256), 1) masked positions per image at step i (the guided embedding is formed
# before to_logits, so the null pass adds no logits rows)
rows = b * sum(max(int(math.cos(math.pi / 2 * i / (bench.TIMESTEPS - 1)) * 256), 1) for i in range(bench.TIMESTEPS))
flop = 2.0 * rows * 65536 * 512
table = {}
print(f"kernel time in one eager generate(): {all_ms:.1f} ms; logits FLOPs {flop / 1e12:.2f} TFLOP over {rows} rows")
for name, (ms, n) in sorted(tot.items(), key=lambda kv: -kv[1][0]):
    if any(s in name for s in ("tc_logits_kernel", "logits_finish", "logits_threshold", "tc_gemm_kernel", "logits_sample")):
        line = f"{ms:9.2f} ms {100 * ms / all_ms:5.1f} %  x{n:5d}  {name[:110]}"
        if "tc_logits_kernel" in name:
            line += f"   {flop / (ms * 1e-3) / 1e12:.0f} TFLOP/s"
        print(line, flush=True)
        table[name] = {"ms": round(ms, 3), "launches": n}
if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "logits_profile.json"), "w") as f:
        json.dump({"device": smi, "total_ms": all_ms, "logits_tflop": flop / 1e12, "kernels": table}, f, indent=1)

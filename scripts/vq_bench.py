"""VQ codebook lookup (LFQ, bf16 tokens, wgmma route) at the C5 per-GPU size and 8x that: the bench.py `hbm_kernels` measurement alone.
usage: python scripts/vq_bench.py        (MMG_PDL=1 to overlap consecutive launches' prologues)"""
import json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
with torch.no_grad():
    mg = bench.build_models(torch.device("cuda", 0))
    pk = bench.peaks()
    print(json.dumps(bench.hbm_kernels(mg, pk)))

"""Time the T5 text encoder: libmmg's T5Encoder (bf16, fp32; bf16 also replayed as a CUDA graph) against HF's eager T5EncoderModel (fp32 and
model.bfloat16()), on random-weight encoders with the t5-v1_1-base and t5-v1_1-xl shapes at B = 64 and T in {32, 128} (ragged padding).

CUDA events around each call, median of --iters calls after --warmup; FLOP counted from the shapes (the matrix products and the two attention
products); relative L2 error of every arm against HF fp32 on the live rows.  Prints one JSON line per (shape, T, arm) and writes them to --out.
usage: python scripts/t5_bench.py [--iters 20] [--warmup 5] [--out t5_bench.json]"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {
    "t5-v1_1-base": dict(d_model=768, num_heads=12, d_ff=2048, num_layers=12),
    "t5-v1_1-xl": dict(d_model=2048, num_heads=32, d_ff=5120, num_layers=24),
}


def flops(c, B, T):
    d, inner, ff, L = c["d_model"], c["num_heads"] * 64, c["d_ff"], c["num_layers"]
    R = B * T
    per_layer = 2 * R * d * 3 * inner + 2 * R * inner * d + 2 * R * d * 2 * ff + 2 * R * ff * d + 2 * 2 * B * c["num_heads"] * T * T * 64
    return L * per_layer


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--T", default="32,128")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "t5_bench.py measures on the GPU; there is no CPU fallback"
    from transformers import T5Config, T5EncoderModel
    from muse_maskgit_pytorch_b200 import T5Encoder
    gpu = card()
    print(f"# {gpu}", flush=True)
    rows = []
    B = 64
    for name in args.shapes.split(","):
        s = SHAPES[name]
        cfg = T5Config(vocab_size=32128, d_kv=64, feed_forward_proj="gated-gelu", dropout_rate=0.0, **s)
        torch.manual_seed(0)
        with torch.device("cuda"):
            hf32 = T5EncoderModel(cfg).eval()
        for T in (int(t) for t in args.T.split(",")):
            g = torch.Generator().manual_seed(T)
            ids = torch.randint(0, 32128, (B, T), generator=g).cuda()
            lens = torch.randint(T // 2, T + 1, (B,), generator=g); lens[0] = T
            mask = (torch.arange(T)[None, :] < lens[:, None]).long().cuda()
            live = mask.bool()
            fl = flops(s, B, T)

            def hf_call(m):
                with torch.no_grad():
                    return m(input_ids=ids, attention_mask=mask).last_hidden_state.float().masked_fill(~live[..., None], 0)
            ref = hf_call(hf32)

            def add(arm, fn):
                out = fn()
                ms = time_ms(fn, args.iters, args.warmup)
                err = float((out[live].double() - ref[live].double()).norm() / ref[live].double().norm())
                r = dict(shape=name, B=B, T=T, arm=arm, ms=round(ms, 3), tflops=round(fl / ms / 1e9, 1), rel_l2_vs_hf_fp32=float(f"{err:.3e}"), gpu=gpu)
                rows.append(r)
                print(json.dumps(r), flush=True)

            add("hf_fp32_eager", lambda: hf_call(hf32))
            hf16 = copy.deepcopy(hf32).bfloat16()
            add("hf_bf16_eager", lambda: hf_call(hf16))
            del hf16
            for prec in ("bf16", "fp32"):
                enc = T5Encoder(cfg, precision=prec, init_weights=False).cuda()
                enc.load_state_dict(hf32.state_dict(), strict=True)
                add(f"native_{prec}", lambda: enc(ids, mask))
                if prec == "bf16":
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        g_out = enc(ids, mask)
                    add("native_bf16_graph", lambda: (graph.replay(), g_out)[1])
                    del graph, g_out
                del enc
                torch.cuda.empty_cache()
        del hf32
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()

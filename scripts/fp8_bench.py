"""precision="fp8" against "bf16" on one GPU: the three e4m3 products at C3 shapes, C3 generate() images/s, and the fp8 teacher-forced
flip rate against the fp32 oracle.  The card's name, power limit and SM clocks are read in the same process.
usage: python scripts/fp8_bench.py [--rounds 5] [--calls 3] [--iters 10] [--no-flip] [--out results/fp8_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from muse_maskgit_pytorch_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--calls", type=int, default=3)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--no-flip", action="store_true")
ap.add_argument("--out", default="")
args = ap.parse_args()
assert torch.cuda.is_available(), "fp8_bench.py measures on the GPU; there is no CPU fallback"
torch.set_grad_enabled(False)
bf, E4 = torch.bfloat16, torch.float8_e4m3fn
TR_CFG = dict(num_tokens=65536, seq_len=256, dim=512, depth=8, dim_head=64, heads=8, ff_mult=4)     # bench.py's C3 model
VAE_CFG = dict(dim=256, codebook_size=65536)
B, STEPS = 64, 18


def smi():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def kernel_ms(fn, iters):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[0], ts[len(ts) // 2]


def products():
    """(name, M, N, K, bf16 fn, fp8 fn) at C3: B = 64, 2 CFG branches, 256 tokens, dim 512, 8 heads, FF inner 1365 -> 1408"""
    out = []
    g = torch.Generator(device="cuda").manual_seed(0)
    heads, tokens = 8, 256
    for name, Mr, N, K, kind in (("self QKV <256, QKV>", 2 * B * tokens, 3 * heads * 64, 512, "qkv"),
                                 ("cross q <128, QKV>", B * tokens, heads * 64, 512, "q"),
                                 ("FF1 GEGLU <256, GEGLU>", 2 * B * tokens, 2816, 512, "geglu")):
        a32 = torch.randn((Mr, K), device="cuda", generator=g)
        w32 = torch.randn((N, K), device="cuda", generator=g) * K ** -0.5
        a, w = a32.to(bf), w32.to(bf)
        sa, sw = a32.abs().amax(1) / 448, w32.abs().amax(1) / 448
        a8, w8 = (a32 / sa[:, None]).clamp(-448, 448).to(E4), (w32 / sw[:, None]).clamp(-448, 448).to(E4)
        bs = Mr // tokens
        qsc = torch.ones((64,), device="cuda")
        if kind == "geglu":
            h = torch.empty((Mr, N // 2), device="cuda", dtype=bf)
            st = torch.empty((Mr, N // 64, 2), device="cuda")
            f16 = lambda a=a, w=w, h=h, st=st: ops.linear(a, w, h, epilogue=ops.EPI_GEGLU, row_stats=st)
            f8 = lambda h=h, st=st, a8=a8, w8=w8, sa=sa, sw=sw: ops.linear_fp8(a8, sa, w8, sw, h, epilogue=ops.EPI_GEGLU, row_stats=st)
        else:
            q = torch.empty((bs * heads, tokens, 64), device="cuda", dtype=bf)
            if kind == "qkv":
                k = torch.zeros((bs * heads, tokens + 8, 64), device="cuda", dtype=bf)
                v = torch.zeros_like(k)
                epi = ops.qkv_epilogue(bf, heads, tokens, q=q, k=k, v=v, q_scale=qsc, k_scale=qsc, key_off=1)
            else:
                epi = ops.qkv_epilogue(bf, heads, tokens, q=q, q_scale=qsc)
            f16 = lambda a=a, w=w, epi=epi: ops.linear(a, w, None, epilogue=ops.EPI_QKV, epi=epi)
            f8 = lambda a8=a8, w8=w8, sa=sa, sw=sw, epi=epi: ops.linear_fp8(a8, sa, w8, sw, None, epilogue=ops.EPI_QKV, epi=epi)
        out.append((name, Mr, N, K, f16, f8))
    return out


def build(precision):
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-512"] = {"d_model": 512}
    torch.manual_seed(0)
    vae = M.VQGanVAE(precision="bf16", **VAE_CFG)
    tr = M.MaskGitTransformer(t5_name="synth-512", precision=precision, **TR_CFG)
    mg = M.MaskGit(image_size=256, transformer=tr, vae=vae).cuda()
    te = torch.randn((B, 32, 512), generator=torch.Generator().manual_seed(1)).cuda()
    te[1::2, 24:] = 0.
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    mg.sampler_seed = 2
    return mg


def main():
    res = dict(gpu_before=smi())
    print("GPU:", res["gpu_before"], flush=True)
    rows = []
    for name, Mr, N, K, f16, f8 in products():
        flop = 2.0 * Mr * N * K
        b16, b8 = kernel_ms(f16, args.iters), kernel_ms(f8, args.iters)
        r = dict(product=name, M=Mr, N=N, K=K, bf16_best_us=b16[0] * 1e3, bf16_median_us=b16[1] * 1e3, fp8_best_us=b8[0] * 1e3,
                 fp8_median_us=b8[1] * 1e3, bf16_tflops=flop / b16[0] / 1e9, fp8_tflops=flop / b8[0] / 1e9)
        rows.append(r)
        print(f"{name:26s} {Mr}x{N}x{K}: bf16 {r['bf16_best_us']:.1f} us ({r['bf16_tflops']:.0f} TFLOP/s), fp8 {r['fp8_best_us']:.1f} us "
              f"({r['fp8_tflops']:.0f} TFLOP/s), speed-up {r['bf16_best_us'] / r['fp8_best_us']:.2f}x  (best of {args.iters}, L2 flushed; "
              f"medians {r['bf16_median_us']:.1f} / {r['fp8_median_us']:.1f} us)", flush=True)
    res["products"] = rows

    texts = ["a"] * B
    models = {p: build(p) for p in ("bf16", "fp8")}
    for p, mg in models.items():                       # warm-up: packing, workspaces, graph capture
        mg.generate(texts, timesteps=STEPS, cond_scale=3)
        mg.generate(texts, timesteps=STEPS, cond_scale=3)
    torch.cuda.synchronize()
    times = {p: [] for p in models}
    for rnd in range(args.rounds):
        for p in (("bf16", "fp8") if rnd % 2 == 0 else ("fp8", "bf16")):
            mg = models[p]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.calls):
                mg.generate(texts, timesteps=STEPS, cond_scale=3)
            torch.cuda.synchronize()
            times[p].append((time.perf_counter() - t0) / args.calls * 1e3)
    res["generate"] = {}
    for p, ts in times.items():
        s = sorted(ts)
        res["generate"][p] = dict(ms_per_call_median=s[len(s) // 2], ms_min=s[0], ms_max=s[-1], images_per_s=B / s[len(s) // 2] * 1e3)
        print(f"C3 generate() {p}: {s[len(s) // 2]:.1f} ms per call ({s[0]:.1f}-{s[-1]:.1f}), {B / s[len(s) // 2] * 1e3:.1f} images/s "
              f"(median of {args.rounds} alternated rounds of {args.calls} calls, CUDA graphs)", flush=True)
    torch.manual_seed(5)
    ids = {p: models[p].generate(texts[:8], timesteps=STEPS, cond_scale=3, return_ids=True)[1] for p in models}
    res["fp8_vs_bf16_id_agreement"] = float((ids["fp8"] == ids["bf16"]).float().mean())
    del models
    torch.cuda.empty_cache()
    res["gpu_after"] = smi()
    print("GPU after:", res["gpu_after"], flush=True)

    if not args.no_flip:
        from tests import test_gpu_full_config as FC
        import muse_maskgit_pytorch_b200 as M
        bf_tr, _ = FC.base_transformer()
        torch.manual_seed(0)
        tr = M.MaskGitTransformer(t5_name="synth-512", precision="fp8", **FC.TR_BASE)
        tr.load_state_dict(bf_tr.state_dict())
        vae_cls = M.VQGanVAE                             # the token loop does not touch the VAE
        M.VQGanVAE = lambda *a, precision=None, **k: vae_cls(*a, precision="bf16", **k)
        try:
            flips, total, per_step, worst = FC._c3_teacher_forced(tr.cuda())
            flips_bf, total_bf, _, _ = FC._c3_teacher_forced(bf_tr)
        finally:
            M.VQGanVAE = vae_cls
        res["flip_rate"] = dict(fp8=flips / total, fp8_flips=flips, tokens=total, bf16=flips_bf / total_bf, per_step_fp8=per_step)
        print(f"C3 teacher-forced flip rate vs the fp32 oracle: fp8 {flips}/{total} = {flips / total:.4f}, bf16 {flips_bf}/{total_bf} = "
              f"{flips_bf / total_bf:.4f}", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""GPU: MaskGit.forward (the training loss, evaluated without gradients) and its kernels.

  mmg_logits_xent / mmg_logits_xent_rows against fp64 torch on the same bf16 operands (split plans, ragged row counts, label columns at
  chunk edges, constant / peaked / large-magnitude rows), their agreement, run-to-run bitwise equality and the unsupported-shape rule;
  MaskGit.forward against the unmodified reference's losses (tests/golden/loss_small.npz) with the reference's draws injected, in fp32 and
  bf16; the ATen noise stream against a replay of the reference's CUDA draws; the fused path's memory; the call's errors and side effects.
"""
import math
import random

import pytest
import torch

from oracle import fused_tail as FT
from tests import util, loss_oracle as LO

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def M():
    import muse_maskgit_pytorch_b200 as m
    from muse_maskgit_pytorch_b200 import t5
    for d in (128, 512):
        t5.T5_CONFIGS[f"synth-{d}"] = {"d_model": d}
    return m


def ops():
    from muse_maskgit_pytorch_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ kernels
def fp64_nll(e, w, labels):
    lg = e.double() @ w.double().t()
    return torch.logsumexp(lg, dim=-1) - lg.gather(1, labels.long()[:, None])[:, 0], lg.abs().amax(dim=-1)


def run_fused(e, w, labels):
    o = ops()
    nbytes = o.logits_xent_workspace_bytes(e.shape[0], w.shape[0], w.shape[1])
    assert nbytes > 0
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    nll = torch.empty((e.shape[0],), device="cuda")
    return o.logits_xent(e, w, labels, nll, ws)


def run_rows(e, w, labels):
    o = ops()
    lg = torch.empty((e.shape[0], w.shape[0]), device="cuda")
    o.linear(e, w, lg)
    return o.logits_xent_rows(lg, labels, torch.empty((e.shape[0],), device="cuda"))


def operands(R, V, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    e = torch.randn((R, K), device="cuda", generator=g).bfloat16()
    w = (torch.randn((V, K), device="cuda", generator=g) * (3.0 / math.sqrt(K))).bfloat16()
    edges = torch.tensor([0, 63, 64, 127, 128, V - 1], device="cuda", dtype=torch.int32)
    labels = torch.randint(0, V, (R,), device="cuda", generator=g, dtype=torch.int32)
    labels[:min(R, 6)] = edges[:min(R, 6)]
    return e, w, labels


def check(e, w, labels, tag):
    """|nll - fp64| <= 1e-4 + 4 fp32 ulps of the row's largest logit (the fp32 sum M + log(sum) - x_label cannot resolve less on a
    row of logits ~1e3); fused vs rows within 2e-5 on the same scale; two fused calls bitwise equal."""
    ref, mag = fp64_nll(e, w, labels)
    tol = 1e-4 + 4.8e-7 * mag
    a, b, rows = run_fused(e, w, labels), run_fused(e, w, labels), run_rows(e, w, labels)
    assert torch.isfinite(a).all() and torch.isfinite(rows).all(), tag
    assert torch.equal(a, b), tag
    err = (a.double() - ref).abs()
    assert (err <= tol).all(), (tag, float(err.max()), int(err.argmax()))
    assert ((rows.double() - ref).abs() <= tol).all(), tag
    assert ((a - rows).abs().double() <= 2e-5 + 4.8e-7 * mag).all(), (tag, float((a - rows).abs().max()))
    return float(err.max())


@pytest.mark.parametrize("V", [1024, 1280, 8192, 65536])
@pytest.mark.parametrize("K", [64, 128, 512])
def test_xent_kernels_vs_fp64(V, K):
    worst = 0.
    for R in (1, 77, 300):
        worst = max(worst, check(*operands(R, V, K, seed=R + V + K), f"R={R} V={V} K={K}"))
    print(f"V={V} K={K}: max |nll - fp64| = {worst:.2e}")


def test_xent_every_split_plan():
    """Row counts that reach every split plan of the shared work split at V = 65536, each with a ragged last M-tile."""
    units = torch.cuda.get_device_properties(0).multi_processor_count
    plans = {S: FT.rows_for_plan(65536, S, units) for S in (1, 2, 4, 8, 16, 32, 64)}
    plans = {S: R for S, R in plans.items() if R is not None}
    assert 1 in plans and 2 in plans
    for S, R in plans.items():
        err = check(*operands(R, 65536, 512, seed=S), f"S={S} R={R}")
        print(f"S={S} R={R}: max |nll - fp64| = {err:.2e}")


def test_xent_constant_peaked_and_large_rows():
    V, K = 8192, 128
    e, w, labels = operands(8, V, K, seed=5)
    e[0] = 0                                                            # constant row: nll = log V
    w[:, 0] = 0
    w[1234, 0] = 1.
    e[1] = 0; e[1, 0] = 80.                                             # one logit 80 above the rest, label on it and off it
    e[2] = 0; e[2, 0] = 80.
    labels[1], labels[2] = 1234, 7
    w[:, 1] = (torch.rand(V, device="cuda") * 2 - 1).bfloat16()
    e[3] = 0; e[3, 1] = 1024.                                           # logits of magnitude ~1e3 (exact products)
    e[4] = 0; e[4, 1] = -1024.
    check(e, w, labels, "special rows")
    nll = run_fused(e, w, labels)
    assert abs(float(nll[0]) - math.log(V)) < 1e-5
    assert float(nll[1]) < 1e-5 and abs(float(nll[2]) - 80.) < 1e-4


def test_xent_unsupported_shapes_rejected():
    o = ops()
    from muse_maskgit_pytorch_b200 import _lib
    for V, K in ((1000, 64), (1024, 96), (1024, 32), (64, 64)):
        assert o.logits_xent_workspace_bytes(100, V, K) == 0
    e, w, labels = operands(10, 1024, 64, seed=1)
    n0 = _lib.launch_count()
    with pytest.raises(_lib.MMGError):
        o.logits_xent(e[:, :32].contiguous(), w[:, :32].contiguous(), labels, torch.empty(10, device="cuda"), torch.empty(1024, dtype=torch.uint8, device="cuda"))
    assert _lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------ MaskGit.forward vs the reference
def load(module, sd):
    full = module.state_dict()
    for k, v in sd.items():
        full[k] = v
    module.load_state_dict(full)
    return module


def make_model(name, precision, **model_kw):
    """The G4-G8 models of tests/golden/make_golden.py as MaskGit instances."""
    m = M()
    sd, cfg, critic, vae_sd, seq_len = LO.model_weights(name)
    vae = load(m.VQGanVAE(dim=16, layers=2, codebook_size=1024, precision="fp32"), vae_sd)     # exact tokens: the gap is the transformer's
    tr = load(m.MaskGitTransformer(num_tokens=1024, dim=128, seq_len=seq_len, depth=2, heads=2, t5_name="synth-128",
                                   self_cond=cfg["self_cond"], precision=precision), sd)
    te = util.text_embeds("g4.te", 3, 8, 128, 14).cuda()
    tr.encode_text = lambda texts: te[:len(texts)]
    kw = dict(image_size=16, transformer=tr, vae=vae)
    if name == "g5":
        kw.update(image_size=32, cond_image_size=16)
    if name == "g7":
        kw["token_critic"] = load(m.TokenCritic(num_tokens=1024, dim=128, seq_len=16, depth=1, heads=2, t5_name="synth-128", precision=precision),
                                  critic["sd"])
    if name == "g8":
        kw["self_token_critic"] = True
    mg = m.MaskGit(**kw, **model_kw)
    if name == "g8":
        mg.token_critic.to_pred.weight.data.copy_(critic["w_pred"]); mg.token_critic.to_pred.bias.data.copy_(critic["b_pred"])
    return mg.cuda()


def golden_forward(name, c, precision, monkeypatch):
    mg = make_model(c["model"], precision, **c["model_kw"])
    mg.sampler_noise_fn = util.torch_noise_fn(c["seed"])
    draws = iter(c["py_draws"])
    monkeypatch.setattr(random, "random", lambda: next(draws))
    kw = dict(c["kw"])
    if c["cond_images"] is not None:
        kw["cond_images"] = c["cond_images"].cuda()
    loss = mg(c["input"].cuda(), texts=["a"] * c["input"].shape[0], **kw)
    assert next(draws, None) is None, "forward made fewer python random() draws than the reference"
    assert loss.shape == () and loss.dtype == torch.float32 and loss.is_cuda
    return float(loss)


@pytest.mark.parametrize("name", sorted(LO.golden_cases()))
def test_forward_fp32_matches_reference(name, monkeypatch):
    c = LO.golden_cases()[name]
    loss = golden_forward(name, c, "fp32", monkeypatch)
    print(f"{name}: fp32 {loss:.7f} reference {c['loss']:.7f}")
    assert abs(loss - c["loss"]) <= 1e-4


@pytest.mark.parametrize("name", sorted(LO.golden_cases()))
def test_forward_bf16_relative_gap(name, monkeypatch):
    c = LO.golden_cases()[name]
    loss = golden_forward(name, c, "bf16", monkeypatch)
    gap = abs(loss - c["loss"]) / abs(c["loss"])
    print(f"{name}: bf16 {loss:.6f} reference {c['loss']:.6f} relative gap {gap:.2e}")
    assert gap <= 5e-3


def test_forward_aten_noise_matches_replayed_cuda_draws(monkeypatch):
    """sampler_rng = "aten": the critic branch's gumbel noise is the reference's own zeros_like(logits).uniform_() stream on the CUDA
    generator; a CPU oracle fed the same draws made with torch on the GPU gives the same loss, and the generator ends where the replay ends."""
    c = LO.golden_cases()["token_critic"]
    mg = make_model("g7", "fp32")
    mg.sampler_rng = "aten"
    monkeypatch.setattr(random, "random", lambda: 0.57)
    gen = torch.cuda.default_generators[0]
    torch.cuda.manual_seed(1234)
    loss = float(mg(c["input"].cuda(), texts=["a"] * 3))
    end = gen.get_offset()
    torch.cuda.manual_seed(1234)
    ref = LO.golden_case_loss(c, lambda shape: torch.zeros(shape, device="cuda").uniform_(0, 1).cpu(), lambda: 0.57)
    print(f"aten: {loss:.7f} replay {float(ref):.7f}")
    assert abs(loss - float(ref)) <= 1e-4
    assert gen.get_offset() == end


# ------------------------------------------------------------------------------------------------ fused path memory, behaviour
def c3_like_model(b=8):
    m = M()
    torch.manual_seed(0)
    tr = m.MaskGitTransformer(num_tokens=65536, dim=512, seq_len=256, depth=2, heads=8, t5_name="synth-512")
    vae = m.VQGanVAE(dim=16, layers=4, codebook_size=65536)
    te = torch.randn((b, 32, 512), device="cuda")
    tr.encode_text = lambda texts: te[:len(texts)]
    return m.MaskGit(image_size=256, transformer=tr, vae=vae).cuda()


def test_fused_forward_holds_no_logits_buffer():
    b, n, V = 8, 256, 65536
    mg = c3_like_model(b)
    ids = torch.randint(0, V, (b, n), device="cuda")
    run = lambda: (torch.manual_seed(7), float(mg(ids, texts=["a"] * b)))[1]
    run()                                                                # packs weights, allocates the block workspace
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fused = run()
    grow = torch.cuda.max_memory_allocated() - base
    mg.use_fused_tail = False
    unfused = run()
    torch.manual_seed(7)                                                 # the call's first draw: the mask ratio of each sequence
    nm = (n * torch.cos(torch.zeros((b,), device="cuda").uniform_(0, 1) * math.pi * 0.5)).round().clamp(min=1)
    R = int(nm.sum())
    print(f"R = {R} labelled rows: fused peak growth {grow / 2**20:.1f} MiB vs R*V*4 = {R * V * 4 / 2**20:.1f} MiB; "
          f"loss fused {fused:.6f} materialised {unfused:.6f}")
    assert grow < R * V * 4 / 4
    assert abs(fused - unfused) <= 1e-4 * abs(unfused)


def test_forward_errors_and_side_effects():
    from muse_maskgit_pytorch_b200 import _lib
    mg = make_model("g4", "bf16")
    ids = torch.randint(0, 1024, (3, 16), device="cuda")
    with torch.enable_grad(), pytest.raises(RuntimeError, match="torch.no_grad"):
        mg(ids, texts=["a"] * 3)
    bad = ids.clone(); bad[1, 3] = mg.mask_id
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        mg(bad, texts=["a"] * 3)
    with pytest.raises(ValueError):
        mg(-ids - 1, texts=["a"] * 3)
    assert _lib.launch_count() == n0
    run = lambda: (torch.manual_seed(3), random.seed(3), float(mg(ids, texts=["a"] * 3)))[2]
    assert run() == run()
    mg.sampler_seed = 11
    before = mg.generate(texts=["a"] * 3, timesteps=6, return_ids=True)[1].clone()
    for training in (True, False):
        mg.train(training)
        run()
        assert mg.training == training and mg.transformer.training == training
    after = mg.generate(texts=["a"] * 3, timesteps=6, return_ids=True)[1]
    assert torch.equal(before, after)

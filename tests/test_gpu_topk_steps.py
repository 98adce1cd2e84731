"""GPU: per-image top-k threshold and step count (`topk_filter_thres` / `timesteps` per image).

Kernels: with a per-image k table, each image's rows of mmg_logits_sample (candidate-list and row-walking kernels, noise modes 0 /
injected / ATen) and of mmg_logits_fused (its finishing kernel, its materialised fallback leg, the exact threshold at V <= 4096) equal a
launch with that image's k as the scalar; rows with k = 1 inside a call the largest k routes to the row-walking kernel keep their token.

Models: with image_seeds, each image of a mixed batch (timesteps, topk_filter_thres, cond_scale, temperature) equals its lone scalar call,
for generate and ragged inpaint, bf16 and fp32, with and without a token critic, with self-conditioning, on virtual ranks of world 2 and 3
and through Muse.forward; with injected noise a mixed fp32 call equals the CPU oracle image by image; one captured graph replays for new
thresholds on the same route and for a permuted assignment of step counts; uniform calls launch what they launched before; bad
arguments raise before any launch."""
import math

import pytest
import torch

from muse_maskgit_pytorch_b200 import _lib
from oracle import muse_oracle as O
from tests import util
from tests.test_gpu_fused_tail import _case, _fp64_check
from tests.test_gpu_image_seeds import SEEDS, _bits, _model, _report, _te_bank
from tests.test_gpu_inpaint import _images, _ragged_tokens
from tests.test_gpu_models import M, make_branch_maskgit, make_maskgit
from tests.test_gpu_sharded_entry_points import _virtual_ranks

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
bf = torch.bfloat16

STEPS = [6, 4, 8, 6, 3, 8, 5]
THRES = [0.9, 0.95, 0.8, 0.98, 0.9, 0.85, 0.7]
TEMPS = [1.0, 0.5, 2.0, 1.0, 0.0, 1.5, 0.8]
SCALES = [3.0, 1.0, 2.0, 5.0, 3.0, 4.0, 1.5]
NOISE = [0.7, 0.2, 1.0, 0.5, 0.0, 0.9, 0.3]
FRACS = [1, 0.3, 0.6, 0, 0.5, 0.8, 0.2]


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _kdev(ks):
    return torch.tensor(ks, dtype=torch.int32, device="cuda")


# ------------------------------------------------------------------------------------------------ kernels
def _sample_case(B, nm, V, seed):
    g = torch.Generator().manual_seed(seed)
    n = nm + 3
    mp = torch.stack([torch.sort(torch.randperm(n, generator=g)[:nm]).values for _ in range(B)]).int().cuda().contiguous()
    logits = (torch.randn((B * nm, V), generator=g) * 2).cuda()
    return n, mp, logits


def _run_sample(logits, mp, n, nm, k, **kw):
    B = mp.shape[0]
    ids = torch.full((B, n), -1, dtype=torch.long, device="cuda")
    scores = torch.zeros((B, n), device="cuda")
    ops().logits_sample(logits, mp, ids, scores, nm, k, 0.9, step=3, seed=11, **kw)
    return ids, scores


def _noise_kw(mode, B, n, V):
    if mode == "philox":
        return dict(image_seed=_bits(SEEDS[:B]))
    if mode == "injected":
        return dict(u=torch.rand((B, n, V), generator=torch.Generator().manual_seed(5)).cuda())
    from muse_maskgit_pytorch_b200.muse_maskgit import _aten_uniform_geometry
    stride, _ = _aten_uniform_geometry(torch.device("cuda"), B * n * V)
    return dict(aten=(16, torch.zeros((1,), dtype=torch.int64, device="cuda"), stride))


@pytest.mark.parametrize("mode", ["philox", "injected", "aten"])
@pytest.mark.parametrize("V,ks", [(4096, [410, 1, 205, 4096]), (16384, [12000, 1, 1639, 9300])], ids=["list", "row_walking"])
def test_logits_sample_per_image_k_equals_scalar(V, ks, mode):
    """Each image's rows under k_dev equal the scalar launch at its own k: bitwise on the candidate-list kernel; on the row-walking
    kernel (the largest k > 9216 routes every row there) the token is the same and the score differs only in the softmax sum's order."""
    B, nm = len(ks), 5
    n, mp, logits = _sample_case(B, nm, V, V)
    kw = _noise_kw(mode, B, n, V)
    ids, scores = _run_sample(logits, mp, n, nm, max(ks), k_dev=_kdev(ks), **kw)
    for b, k in enumerate(ks):
        want_ids, want_sc = _run_sample(logits, mp, n, nm, k, **kw)
        assert torch.equal(ids[b], want_ids[b]), (b, k)
        if max(ks) <= ops().SAMPLE_LIST_CAP or k > ops().SAMPLE_LIST_CAP:
            assert torch.equal(scores[b], want_sc[b]), (b, k)
        else:
            assert torch.allclose(scores[b], want_sc[b], rtol=0, atol=2e-6), (b, k)
    # k = 1 keeps the largest logit: the token is the row's argmax whatever the noise
    top = logits.view(B, nm, V).argmax(dim=-1)
    assert torch.equal(ids[1].gather(0, mp[1].long()), top[1])


@pytest.mark.parametrize("R,V,K,ks", [(96, 1024, 64, [103, 1, 300]), (300, 65536, 512, [6554, 1, 3277]), (24, 4096, 128, [410, 1, 2000])],
                         ids=["V1024_exact", "V65536", "V4096_exact"])
def test_logits_fused_per_image_k_equals_scalar_and_fp64(R, V, K, ks):
    """The fused tail with k_dev: each image's rows equal the scalar fused call at its own k bitwise, and the fp64 oracle on injected
    noise wherever the perturbed top-2 margin is clear."""
    o = ops()
    e, w, b, n, nm, mp = _case(R, V, K, seed=R + V, b=len(ks))
    u = torch.rand((b, n, V), generator=torch.Generator().manual_seed(R)).cuda()

    def run(k, k_dev=None):
        ws = torch.empty((o.logits_fused_workspace_bytes(R, V, K, max(ks)),), dtype=torch.uint8, device="cuda")
        status = torch.zeros((2,), dtype=torch.int32, device="cuda")
        ids = torch.full((b, n), -1, dtype=torch.long, device="cuda")
        sc = torch.zeros((b, n), device="cuda")
        o.logits_fused(e, w, mp, ids, sc, nm, k, 1.0, ws, status, u=u, k_dev=k_dev)
        assert int(status[1]) == 0
        return ids, sc

    ids, sc = run(max(ks), _kdev(ks))
    for i, k in enumerate(ks):
        want_ids, want_sc = run(k)
        assert torch.equal(ids[i], want_ids[i]) and torch.equal(sc[i], want_sc[i]), (i, k)
        rows = list(range(i * nm, (i + 1) * nm))
        bi = torch.tensor([r // nm for r in rows])
        pi = mp.cpu().long().reshape(-1)[rows]
        _fp64_check(e, w, (bi, pi), ids, sc, rows, k, 1.0, u.cpu()[bi, pi], 1e-3)


def test_logits_fused_fallback_leg_per_image_k():
    """All-equal logits overflow every candidate list, so every row goes through the materialised leg, where sampled row r is row_index[i]:
    each image's ids and scores equal the scalar launch at its own k on the same leg bitwise, and image b keeps the lowest k_b indices
    (with k_b = 1 its token is index 0)."""
    o = ops()
    B, n, nm, V, K = 3, 20, 6, 1024, 64
    ks = [103, 1, 2]
    g = torch.Generator().manual_seed(4)
    mp = torch.stack([torch.sort(torch.randperm(n, generator=g)[:nm]).values for _ in range(B)]).int().cuda().contiguous()
    e = torch.zeros((B * nm, K), device="cuda", dtype=bf)
    w = torch.randn((V, K), device="cuda").to(bf)

    def run(k, k_dev=None):
        ws = torch.empty((o.logits_fused_workspace_bytes(B * nm, V, K, max(ks)),), dtype=torch.uint8, device="cuda")
        status = torch.zeros((2,), dtype=torch.int32, device="cuda")
        ids = torch.full((B, n), -1, dtype=torch.long, device="cuda")
        scores = torch.zeros((B, n), device="cuda")
        o.logits_fused(e, w, mp, ids, scores, nm, k, 1.0, ws, status, seed=5, step=2, image_seed=_bits(SEEDS[:B]), k_dev=k_dev)
        assert int(status[0]) == B * nm and int(status[1]) == 0      # every row took the fallback leg
        return ids, scores

    ids, scores = run(max(ks), _kdev(ks))
    for bi, k in enumerate(ks):
        want_ids, want_sc = run(k)
        assert torch.equal(ids[bi], want_ids[bi]) and torch.equal(scores[bi], want_sc[bi]), (bi, k)
        got = ids[bi].gather(0, mp[bi].long())
        assert bool(((got >= 0) & (got < k)).all()), (bi, k, got)
    assert bool((ids[1].gather(0, mp[1].long()) == 0).all())


# ------------------------------------------------------------------------------------------------ models
def _call(mg, method, idx, critic, per_image=True):
    """method over the images idx of the 7-image bank; per_image=False passes image idx[0]'s timesteps / threshold as scalars."""
    pick = lambda v: [v[i] for i in idx]
    steps, thres = (pick(STEPS), pick(THRES)) if per_image else (STEPS[idx[0]], THRES[idx[0]])
    kw = dict(temperature=pick(TEMPS), cond_scale=pick(SCALES), image_seeds=pick(SEEDS), return_ids=True, timesteps=steps,
              topk_filter_thres=thres)
    if critic:
        kw["critic_noise_scale"] = pick(NOISE)
    texts = [str(i) for i in idx]
    if method == "generate":
        return mg.generate(texts, **kw)
    return mg.inpaint(texts, _images(7, 16)[idx], _ragged_tokens(7, 4, 8, FRACS)[idx].cuda(), **kw)


def _selfcond_model(precision):
    mg, _, _ = make_branch_maskgit("gen_selfcond_small", precision)
    te = _te_bank()
    mg.transformer.encode_text = lambda texts: torch.stack([te[int(t)] for t in texts])
    mg.use_cuda_graph = False
    return mg


@pytest.mark.parametrize("variant", ["plain", "token_critic", "self_cond"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("method", ["generate", "inpaint"])
def test_mixed_image_equals_its_lone_scalar_call(method, precision, variant):
    critic = variant == "token_critic"
    mg = _selfcond_model(precision) if variant == "self_cond" else _model(precision, critic)
    img, ids = _call(mg, method, list(range(7)), critic)
    for i in range(7):
        a_img, a_ids = _call(mg, method, [i], critic, per_image=False)
        _report(f"{method} {precision} {variant} image {i} (T={STEPS[i]}, thres={THRES[i]}) alone", ids[i:i + 1], a_ids, img[i:i + 1], a_img)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("method", ["generate", "inpaint"])
def test_mixed_virtual_ranks_equal_the_unsharded_call(method, world):
    mg = _model("bf16", True)
    img, ids = _call(mg, method, list(range(7)), True)
    kw = dict(temperature=TEMPS, cond_scale=SCALES, critic_noise_scale=NOISE, image_seeds=SEEDS, return_ids=True, timesteps=STEPS,
              topk_filter_thres=THRES)
    args = {} if method == "generate" else dict(images=_images(7, 16), mask=_ragged_tokens(7, 4, 8, FRACS).cuda())
    s_img, s_ids = _virtual_ranks(getattr(mg, method), (mg,), [str(i) for i in range(7)], world, 5, text_embeds=_te_bank(), **args, **kw)
    _report(f"{method} world {world}", ids, s_ids, img, s_img)


def test_muse_per_image_steps_equal_lone_stages():
    from muse_maskgit_pytorch_b200.muse_maskgit import splitmix64
    base, sup = make_maskgit("bf16"), make_maskgit("bf16", superres=True)
    te = _te_bank()[:5]
    for m in (base, sup):
        m.transformer.encode_text = lambda texts: te[:len(texts)]
    muse = M().Muse(base=base, superres=sup)
    steps, sr_steps = STEPS[:5], [3, 5, 4, 4, 6]
    hi, lo = muse(["a"] * 5, cond_scale=SCALES[:5], timesteps=steps, superres_timesteps=sr_steps, return_lowres=True,
                  return_pil_images=False, image_seeds=41)
    for i in range(5):
        base.transformer.encode_text = sup.transformer.encode_text = lambda texts, i=i: te[i:i + 1]
        want_lo = base.generate(["a"], cond_scale=SCALES[i], timesteps=steps[i], image_seeds=[41 + i])
        want_hi = sup.generate(["a"], cond_scale=SCALES[i], timesteps=sr_steps[i], cond_images=want_lo, image_seeds=[splitmix64(41 + i)])
        assert torch.equal(lo[i:i + 1], want_lo) and torch.equal(hi[i:i + 1], want_hi), i


def test_mixed_fp32_injected_noise_equals_the_oracle_per_image():
    """sampler_noise_fn supplies (b, n, V) per step; image b's slice of it, run through the CPU oracle with that image's own timesteps,
    threshold and temperature, gives its tokens."""
    from muse_maskgit_pytorch_b200 import t5
    Mm = M()
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    tr = Mm.MaskGitTransformer(num_tokens=1024, dim=128, seq_len=16, depth=2, heads=2, t5_name="synth-128", precision="fp32")
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    full = tr.state_dict(); full.update(sd); tr.load_state_dict(full)
    vae = Mm.VQGanVAE(dim=16, layers=2, codebook_size=1024, precision="fp32")
    vsd = util.vae_sd(16, 2, 1024, seed=12)
    full = vae.state_dict(); full.update(vsd); vae.load_state_dict(full)
    mg = Mm.MaskGit(image_size=16, transformer=tr.cuda(), vae=vae.cuda()).cuda()
    te = util.text_embeds("g4.te", 3, 8, 128, 14)
    tr.encode_text = lambda texts: te[:len(texts)]
    mg.use_cuda_graph = False
    noise, drawn = util.torch_noise_fn(777), {}

    def record(step, shape):                      # the noise function draws a stream: keep what the call consumed, per step
        drawn[step] = noise(step, shape)
        return drawn[step]
    mg.sampler_noise_fn = record
    steps, thres, temps = [6, 3, 5], [0.9, 0.95, 0.8], [1.0, 0.7, 1.3]
    _, ids = mg.generate(["a"] * 3, timesteps=steps, topk_filter_thres=thres, temperature=temps, return_ids=True)
    for i in range(3):
        sliced = lambda step, shape, i=i: drawn[step][i:i + 1]
        _, ref_ids = O.generate(sd, dict(heads=2, depth=2), vsd, 10, te[i:i + 1], 4, sliced, timesteps=steps[i], topk_thres=thres[i],
                                temperature=temps[i])
        assert torch.equal(ids[i].cpu().view(1, -1), ref_ids), i


def test_graph_replays_for_new_thresholds_and_permuted_steps():
    mg = _model("bf16", True)
    mg.use_cuda_graph = True
    texts = [str(i) for i in range(7)]
    run = lambda steps, thres: mg.generate(texts, timesteps=steps, topk_filter_thres=thres, cond_scale=SCALES, critic_noise_scale=NOISE,
                                           image_seeds=SEEDS, return_ids=True)
    cases = [(STEPS, THRES), (STEPS, [0.92, 0.9, 0.97, 0.8, 0.99, 0.9, 0.75]), (STEPS[::-1], THRES)]
    got = [run(*cases[0])]
    n_graphs = len(mg._graphs)
    got += [run(*c) for c in cases[1:]]
    assert len(mg._graphs) == n_graphs
    mg.use_cuda_graph = False
    for (steps, thres), g in zip(cases, got):
        want = run(steps, thres)
        _report(f"graph vs eager T={steps} thres={thres}", want[1], g[1], want[0], g[0])


@pytest.mark.parametrize("method", ["generate", "inpaint", "edit"])
def test_uniform_launch_count_unchanged(method):
    """A per-image list of equal values is the scalar call: the same launches."""
    mg = _model("bf16", True)
    mg.sampler_seed = 3
    counts = []
    img, mask = _images(7, 16), _ragged_tokens(7, 4, 8, FRACS).cuda()
    texts = [str(i) for i in range(7)]
    for T, thres in ((6, 0.9), ([6] * 7, [0.9] * 7)):
        l0 = _lib.launch_count()
        if method == "generate":
            mg.generate(texts, timesteps=T, topk_filter_thres=thres)
        elif method == "inpaint":
            mg.inpaint(texts, img, mask, timesteps=T, topk_filter_thres=thres)
        else:
            mg.edit(texts, img, mask=mask, iterations=2, fraction=0.5, timesteps=3, topk_filter_thres=thres)
        torch.cuda.synchronize()
        counts.append(_lib.launch_count() - l0)
    assert counts[0] == counts[1], counts


def test_bad_arguments_raise_before_any_launch():
    mg = _model("bf16", False)
    img, mask = _images(3, 16), _ragged_tokens(3, 4, 8, [1, 0.5, 0.2]).cuda()
    texts = ["0", "1", "2"]
    bad = [("generate", dict(timesteps=[6, 0, 3])), ("generate", dict(timesteps=[6, 3])), ("generate", dict(timesteps=[6, 3.0, 2])),
           ("generate", dict(topk_filter_thres=[0.9, 1.0, 0.9])), ("generate", dict(topk_filter_thres=[0.9, -0.1, 0.9])),
           ("generate", dict(topk_filter_thres=[0.9, 0.9])), ("inpaint", dict(timesteps=[6, 4, 0])),
           ("edit", dict(timesteps=[3, 3, 2])), ("extrapolate", dict(timesteps=torch.tensor([3, 3, 3])))]
    for method, kw in bad:
        l0 = _lib.launch_count()
        with pytest.raises(ValueError):
            if method == "generate":
                mg.generate(texts, **kw)
            elif method == "inpaint":
                mg.inpaint(texts, img, mask, **kw)
            elif method == "edit":
                mg.edit(texts, img, mask=mask, **kw)
            else:
                mg.extrapolate(texts, torch.cat([img, img], dim=3), amount=16, stride=2, **kw)
        assert _lib.launch_count() == l0, (method, kw)
    mg.sampler_rng = "aten"
    l0 = _lib.launch_count()
    with pytest.raises(ValueError):
        mg.generate(texts, timesteps=[6, 4, 4])
    assert _lib.launch_count() == l0

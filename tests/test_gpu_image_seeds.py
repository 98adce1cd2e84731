"""GPU: per-image sampling seeds (`image_seeds`).

Kernels, against oracle/philox.py on the host: with an image_seed table, image b's gumbel noise (mmg_logits_sample small-k and big-k,
mmg_logits_fused with its finishing kernel and its materialised fallback leg), critic noise (mmg_critic_score row_key) and edit keys
(mmg_edit_select) are Philox under image_seeds[b] with the image-local position as the row counter; without it, the (seed, global row)
stream of before.

Models: image b of a batch equals image b called alone with its seed and image b of the permuted batch (ids identical, images bitwise
equal), for generate, inpaint (ragged masks), edit and extrapolate, bf16 and fp32, with and without a token critic, with per-image
cond_scale / temperature; virtual ranks of world 2 and 3 equal the unsharded call; Muse.forward equals its two stages called with the
documented seeds; a captured graph replays for new seeds; the launch count does not change with seeds.  Two caveats are measured and
printed: a batch whose fused-tail split count S differs from a lone image's, and a companion whose longer prompt moves the batch to the
next 32-token context bucket."""
import math

import numpy as np
import pytest
import torch

from muse_maskgit_pytorch_b200 import _lib
from muse_maskgit_pytorch_b200.muse_maskgit import splitmix64
from oracle import philox
from tests import edit_oracle as EO
from tests import util
from tests.test_gpu_fused_tail import _case, _fp64_check, _run_both
from tests.test_gpu_inpaint import _images, _ragged_tokens
from tests.test_gpu_models import M, make_branch_maskgit, make_maskgit
from tests.test_gpu_sharded_entry_points import _virtual_ranks

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
bf = torch.bfloat16
U64 = 1 << 64
SEEDS = [2 ** 64 - 1, 7, 2 ** 63 + 5, 12345, 0, 2 ** 40 + 3, 99]


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _bits(seeds):
    return torch.tensor([s - U64 if s >= 1 << 63 else s for s in seeds], dtype=torch.int64, device="cuda")


def _check_token(got, seed, step, row, V, k):
    """Token of a row whose logits are all equal: the kept set is the lowest k indices and the perturbed value -log(-log u) grows with u,
    so the token is the argmax of u over them.  The kernel takes its logs with fast approximations (absolute error ~2^-21), which may
    order two u closer than 1e-5; then either of the two is accepted."""
    u = philox.uniform(seed, step, row, V)[:k].astype(np.float64)
    order = np.argsort(-u, kind="stable")
    best, second = int(order[0]), int(order[1])
    assert got == best or (u[best] - u[second] < 1e-5 and got == second), (got, best, second, u[best] - u[second])


# ------------------------------------------------------------------------------------------------ kernels
def _ragged_pos(B, n, nm, g):
    """masked_pos [B, nm]: image 0 lists nm distinct positions, the others fewer, padded by repeating a position (the pad rows of
    mmg_remask_frozen compute the same value as the row they repeat)."""
    rows = []
    for b in range(B):
        c = nm - b
        p = torch.sort(torch.randperm(n, generator=g)[:c]).values
        rows.append(torch.cat([p, p[:1].repeat(nm - c)]))
    return torch.stack(rows).int().cuda().contiguous()


@pytest.mark.parametrize("V,k", [(1024, 103), (16384, 10000)], ids=["small_k", "big_k"])
def test_logits_sample_equal_logits_vs_oracle(V, k):
    o = ops()
    B, n, nm, step = 3, 20, 6, 5
    mp = _ragged_pos(B, n, nm, torch.Generator().manual_seed(V))
    logits = torch.zeros((B * nm, V), device="cuda")
    seeds = SEEDS[:B]
    seed_dev = torch.tensor([77], dtype=torch.int64, device="cuda")
    for image_seed in (_bits(seeds), None):
        ids = torch.full((B, n), -1, dtype=torch.long, device="cuda")
        scores = torch.zeros((B, n), device="cuda")
        o.logits_sample(logits, mp, ids, scores, nm, k, 1.0, seed=1000, step=step, row_offset=3 * n, seed_dev=seed_dev, image_seed=image_seed)
        for b in range(B):
            for p in mp[b].tolist():
                if image_seed is not None:
                    _check_token(int(ids[b, p]), seeds[b], step, p, V, k)
                else:
                    _check_token(int(ids[b, p]), 1077, step, 3 * n + b * n + p, V, k)
        assert torch.allclose(scores[ids >= 0], torch.full_like(scores[ids >= 0], 1 - 1 / V))


def test_logits_fused_fallback_leg_equal_logits_vs_oracle():
    """All-equal logits overflow every candidate list, so every row is redone on the materialised leg (row_index)."""
    o = ops()
    B, n, nm, V, K, step = 3, 20, 6, 1024, 64, 2
    k = math.ceil(0.1 * V)
    mp = _ragged_pos(B, n, nm, torch.Generator().manual_seed(4))
    e = torch.zeros((B * nm, K), device="cuda", dtype=bf)
    w = torch.randn((V, K), device="cuda").to(bf)
    ws = torch.empty((o.logits_fused_workspace_bytes(B * nm, V, K, k),), dtype=torch.uint8, device="cuda")
    status = torch.zeros((2,), dtype=torch.int32, device="cuda")
    ids = torch.full((B, n), -1, dtype=torch.long, device="cuda")
    scores = torch.zeros((B, n), device="cuda")
    o.logits_fused(e, w, mp, ids, scores, nm, k, 1.0, ws, status, seed=5, step=step, row_offset=11, image_seed=_bits(SEEDS[:B]))
    assert int(status[0]) == B * nm and int(status[1]) == 0
    for b in range(B):
        for p in mp[b].tolist():
            _check_token(int(ids[b, p]), SEEDS[b], step, p, V, k)


@pytest.mark.parametrize("R,V,K,b", [(96, 1024, 64, 3), (300, 65536, 512, 3)])
def test_logits_fused_finish_vs_materialised_and_fp64_oracle(R, V, K, b):
    """Random rows through the candidate lists: the fused path equals the materialised one, and both equal the fp64 oracle on
    Philox(image_seeds[b], position) wherever the perturbed top-2 margin is clear."""
    e, w, b, n, nm, mp = _case(R, V, K, seed=R + V, b=b)
    k = math.ceil(0.1 * V)
    step, seeds = 3, SEEDS[:b]
    ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, 1.0, seed=9, step=step, row_offset=4 * n, image_seed=_bits(seeds))
    assert torch.equal(ids_a, ids_b), int((ids_a != ids_b).sum())
    assert float((sc_a - sc_b).abs().max()) < 2e-6 and int(status[1]) == 0
    rows = list(range(R))
    bi = torch.tensor([r // nm for r in rows])
    pi = mp.cpu().long().reshape(-1)[rows]
    u = torch.stack([torch.from_numpy(philox.uniform(seeds[int(bb)], step, int(p), V)) for bb, p in zip(bi, pi)])
    checked = _fp64_check(e, w, (bi, pi), ids_b, sc_b, rows, k, 1.0, u, 1e-3)
    print(f"fused R={R} V={V}: fallback rows {int(status[0])}, fp64 oracle on {checked} of {R} rows")


def test_critic_score_row_key_vs_oracle():
    """A zero head scores s = 0, so scores = (u - 0.5) * noise_mul gives back the critic stream's u."""
    o = ops()
    B, n, dim, step = 3, 24, 128, 4
    rows = B * n
    xc = torch.randn((rows, dim), device="cuda")
    gamma, w = torch.ones((dim,), device="cuda"), torch.zeros((dim,), device="cuda")
    seeds = SEEDS[:B]
    key = torch.stack((_bits(seeds)[:, None].expand(B, n), torch.arange(n, device="cuda").expand(B, n)), dim=-1).contiguous()
    seed_dev = torch.tensor([5], dtype=torch.int64, device="cuda")
    for row_key in (key, None):
        scores = torch.empty((rows,), device="cuda")
        o.critic_score(xc, None, gamma, w, 0., 1., 1., scores, seed=40, step=step, row_offset=7, seed_dev=seed_dev, row_key=row_key)
        got = (scores + 0.5).cpu().numpy()
        for r in range(rows):
            want = (philox.uniform_at(seeds[r // n], step, r % n, 0xFFFFFFFF) if row_key is not None
                    else philox.uniform_at(45, step, 7 + r, 0xFFFFFFFF))
            assert got[r] == want, (row_key is not None, r)


def test_edit_select_image_seed_vs_oracle():
    o = ops()
    B, n, it = 4, 64, 3
    g = torch.Generator().manual_seed(8)
    keep = (torch.rand((B, n), generator=g) < 0.3).to(torch.uint8)
    counts = [5, 0, 17, 40]
    seeds = SEEDS[:B]
    seed_dev = torch.tensor([123], dtype=torch.int64, device="cuda")
    for image_seed in (_bits(seeds), None):
        ids = torch.zeros((B, n), dtype=torch.long, device="cuda")
        scores = torch.ones((B, n), device="cuda")
        frozen = torch.empty((B, n), dtype=torch.uint8, device="cuda")
        o.edit_select(ids, scores, frozen, keep.cuda(), torch.tensor(counts, dtype=torch.int32, device="cuda"), 999, it, seed=1,
                      seed_dev=seed_dev, row_offset=2 * n, image_seed=image_seed)
        if image_seed is not None:
            keys = torch.cat([EO.philox_keys(s, it, 1, n) for s in seeds])
        else:
            keys = EO.philox_keys(124, it, B, n, row_offset=2)
        sel = EO.select(keys, keep == 0, counts)
        assert torch.equal(frozen.cpu() == 0, sel)
        assert torch.equal(ids.cpu() == 999, sel)


# ------------------------------------------------------------------------------------------------ models
TEMPS = [1.0, 0.5, 2.0, 1.0, 0.0, 1.5, 0.8]
SCALES = [3.0, 1.0, 2.0, 5.0, 3.0, 4.0, 1.5]
NOISE = [0.7, 0.2, 1.0, 0.5, 0.0, 0.9, 0.3]
FRACS = [1, 0.3, 0.6, 0, 0.5, 0.8, 0.2]


def _te_bank():
    return util.text_embeds("g4.te", 3, 8, 128, 14).cuda().repeat(3, 1, 1)[:7].contiguous()


def _model(precision, critic):
    if critic:
        mg, _, _ = make_branch_maskgit("gen_critic_small", precision)
    else:
        mg = make_maskgit(precision)
    te = _te_bank()
    mg.transformer.encode_text = lambda texts: torch.stack([te[int(t)] for t in texts])
    mg.use_cuda_graph = False
    return mg


def _call(mg, method, idx, critic, extra_kw=None):
    """method over the images idx (a list of indices into the 7-image bank), every per-image input taken for those images."""
    b = len(idx)
    pick = lambda v: [v[i] for i in idx]
    kw = dict(temperature=pick(TEMPS), cond_scale=pick(SCALES), image_seeds=pick(SEEDS), return_ids=True)
    if critic:
        kw["critic_noise_scale"] = pick(NOISE)
    img = _images(7, 16)[idx]
    mask = _ragged_tokens(7, 4, 8, FRACS)[idx].cuda()
    texts = [str(i) for i in idx]
    if method == "generate":
        return mg.generate(texts, timesteps=6, **kw)
    if method == "inpaint":
        return mg.inpaint(texts, img, mask, timesteps=6, **kw)
    if method == "edit":
        return mg.edit(texts, img, mask=mask, iterations=2, fraction=0.5, timesteps=3, **kw)
    wide = torch.cat([img, _images(7, 16, tag="seeds.wide")[idx]], dim=3)
    return mg.extrapolate(texts, wide, direction="right", amount=16, stride=2, timesteps=3, **kw)


def _report(name, want_ids, got_ids, want_img, got_img):
    n_diff = int((want_ids != got_ids).sum())
    same = torch.equal(want_img, got_img)
    print(f"{name}: {n_diff} of {want_ids.numel()} ids differ; images bitwise equal: {same} "
          f"(max |diff| {float((want_img - got_img).abs().max()):.3e})")
    assert n_diff == 0 and same, name


@pytest.mark.parametrize("critic", [False, True], ids=["no_critic", "token_critic"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("method", ["generate", "inpaint", "edit", "extrapolate"])
def test_image_equals_its_lone_call_and_the_permuted_batch(method, precision, critic):
    mg = _model(precision, critic)
    full = list(range(7))
    img, ids = _call(mg, method, full, critic)
    perm = [3, 6, 0, 5, 1, 4, 2]
    p_img, p_ids = _call(mg, method, perm, critic)
    _report(f"{method} {precision} critic={critic} permuted", ids[perm], p_ids, img[perm], p_img)
    for i in full:
        a_img, a_ids = _call(mg, method, [i], critic)
        _report(f"{method} {precision} critic={critic} image {i} alone", ids[i:i + 1], a_ids, img[i:i + 1], a_img)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("method", ["generate", "inpaint", "edit", "extrapolate"])
def test_virtual_ranks_equal_the_unsharded_call(method, world):
    mg = _model("bf16", True)
    full = list(range(7))
    img, ids = _call(mg, method, full, True)
    te = _te_bank()
    texts = [str(i) for i in full]
    kw = dict(temperature=TEMPS, cond_scale=SCALES, critic_noise_scale=NOISE, image_seeds=SEEDS, return_ids=True)
    args = dict(images=_images(7, 16), mask=_ragged_tokens(7, 4, 8, FRACS).cuda())
    if method == "generate":
        kw.update(timesteps=6)
        args = {}
    elif method == "inpaint":
        kw.update(timesteps=6)
    elif method == "edit":
        kw.update(iterations=2, fraction=0.5, timesteps=3)
    else:
        kw.update(direction="right", amount=16, stride=2, timesteps=3)
        args = dict(images=torch.cat([_images(7, 16), _images(7, 16, tag="seeds.wide")], dim=3))
    # each virtual rank draws a different call seed first: with per-image seeds no rank reads one
    s_img, s_ids = _virtual_ranks(getattr(mg, method), (mg,), texts, world, 5, text_embeds=te, **args, **kw)
    _report(f"{method} world {world}", ids, s_ids, img, s_img)


def test_muse_equals_its_stages_with_derived_seeds():
    base, sup = make_maskgit("bf16"), make_maskgit("bf16", superres=True)
    te = _te_bank()[:5]
    for m in (base, sup):
        m.transformer.encode_text = lambda texts: te[:len(texts)]
    muse = M().Muse(base=base, superres=sup)
    texts = ["a"] * 5
    hi, lo = muse(texts, cond_scale=SCALES[:5], timesteps=6, return_lowres=True, return_pil_images=False, image_seeds=41)
    want_lo = base.generate(texts, cond_scale=SCALES[:5], timesteps=6, image_seeds=[41 + i for i in range(5)])
    want_hi = sup.generate(texts, cond_scale=SCALES[:5], timesteps=6, cond_images=want_lo,
                           image_seeds=[splitmix64(41 + i) for i in range(5)])
    assert torch.equal(lo, want_lo) and torch.equal(hi, want_hi)


def test_graph_replays_for_new_seeds_and_equals_eager():
    mg = _model("bf16", True)
    mg.use_cuda_graph = True
    texts = [str(i) for i in range(7)]
    run = lambda seeds: mg.generate(texts, timesteps=6, cond_scale=SCALES, critic_noise_scale=NOISE, image_seeds=seeds, return_ids=True)
    g1 = run(SEEDS)
    n_graphs = len(mg._graphs)
    g2 = run(torch.tensor([s + 1000 for s in range(7)], device="cuda"))
    assert len(mg._graphs) == n_graphs
    mg.use_cuda_graph = False
    for got, seeds in ((g1, SEEDS), (g2, [s + 1000 for s in range(7)])):
        want = run(seeds)
        _report("graph vs eager", want[1], got[1], want[0], got[0])
    assert not torch.equal(g1[1], g2[1])


@pytest.mark.parametrize("method", ["generate", "inpaint", "edit", "extrapolate"])
def test_launch_count_unchanged_by_seeds(method):
    mg = _model("bf16", True)
    mg.sampler_seed = 3
    counts = []
    for seeds in (None, SEEDS):
        l0 = _lib.launch_count()
        kw = {} if seeds is None else {"image_seeds": seeds}
        b = 7
        img, mask = _images(b, 16), _ragged_tokens(b, 4, 8, FRACS).cuda()
        texts = [str(i) for i in range(b)]
        if method == "generate":
            mg.generate(texts, timesteps=6, **kw)
        elif method == "inpaint":
            mg.inpaint(texts, img, mask, timesteps=6, **kw)
        elif method == "edit":
            mg.edit(texts, img, mask=mask, iterations=2, fraction=0.5, timesteps=3, **kw)
        else:
            mg.extrapolate(texts, torch.cat([img, img], dim=3), amount=16, stride=2, timesteps=3, **kw)
        torch.cuda.synchronize()
        counts.append(_lib.launch_count() - l0)
    print(f"{method}: {counts[0]} libmmg launches without image_seeds, {counts[1]} with")
    assert counts[0] == counts[1]


def test_fused_tail_overflow_rerun_keeps_the_seeds():
    """Every logit ties, so the first step overflows the fused tail's fallback and the call is repeated on the materialised path; the
    rerun samples with the same per-image seeds, so the result equals asking for the materialised path directly."""
    from tests.test_gpu_fused_tail import _degenerate_maskgit
    mg, b = _degenerate_maskgit()
    mg.use_cuda_graph = False
    seeds = [500 + 3 * i for i in range(b)]
    img, ids = mg.generate(["a"] * b, timesteps=4, image_seeds=seeds, return_ids=True)
    assert mg.last_fused_fallback_rows > 128                    # the fused attempt overflowed and was repeated
    mg.use_fused_tail = False
    want_img, want_ids = mg.generate(["a"] * b, timesteps=4, image_seeds=seeds, return_ids=True)
    _report("overflow rerun vs the materialised path", want_ids, ids, want_img, img)


def test_seeded_call_draws_no_host_seed():
    mg = _model("bf16", False)
    torch.manual_seed(0)
    state = torch.get_rng_state()
    mg.generate(["0", "1"], timesteps=4, image_seeds=[1, 2])
    assert torch.equal(torch.get_rng_state(), state)


# ------------------------------------------------------------------------------------------------ the two caveats
def test_split_count_caveat():
    """300 images: the whole batch and a lone image run the fused tail with different column splits S.  The split can move the
    confidence score's last bits; the ids and images of the probed images are compared and any difference is reported as a count."""
    from oracle import fused_tail as FT
    units = torch.cuda.get_device_properties(0).multi_processor_count
    b = 300
    s_full, s_one = FT.lf_plan(b * 16, 1024, units)["S"], FT.lf_plan(16, 1024, units)["S"]
    print(f"fused-tail split count at step 0: batch of {b} S = {s_full}, one image S = {s_one} ({units} SMs)")
    assert s_full != s_one
    mg = make_maskgit("bf16")
    mg.use_cuda_graph = False
    te = util.text_embeds("g4.te", 3, 8, 128, 14).cuda()
    mg.transformer.encode_text = lambda texts: te[[int(t) % 3 for t in texts]]
    seeds = [1000 + 17 * i for i in range(b)]
    img, ids = mg.generate([str(i) for i in range(b)], timesteps=8, image_seeds=seeds, return_ids=True)
    for i in (0, 1, 150, 299):
        a_img, a_ids = mg.generate([str(i)], timesteps=8, image_seeds=[seeds[i]], return_ids=True)
        _report(f"split count: image {i} of {b} vs alone", ids[i:i + 1], a_ids, img[i:i + 1], a_img)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_context_padding_caveat(graph):
    """Image 0's 8-token prompt alone, and next to a companion whose 40-token prompt pads the batch's context to 40 tokens (eager) or
    from the 32-token bucket to the 64-token one (graph); padded text rows are zero, which masks their keys."""
    mg = make_maskgit("bf16")
    mg.use_cuda_graph = graph
    te = util.text_embeds("g4.te", 3, 8, 128, 14).cuda()
    long = torch.from_numpy(np.random.default_rng(3).standard_normal((40, 128)).astype(np.float32)).cuda()
    padded = torch.zeros((2, 40, 128), device="cuda")
    padded[0, :8] = te[0]
    padded[1] = long
    kw = dict(timesteps=6, image_seeds=[77], cond_scale=[3.0], return_ids=True)
    mg.transformer.encode_text = lambda texts: te[:1]
    a_img, a_ids = mg.generate(["0"], **kw)
    mg.transformer.encode_text = lambda texts: padded
    img, ids = mg.generate(["0", "1"], timesteps=6, image_seeds=[77, 78], cond_scale=[3.0, 3.0], return_ids=True)
    _report(f"context padding {'graph' if graph else 'eager'}: 8-token prompt alone vs next to a 40-token one", a_ids, ids[:1], a_img, img[:1])

"""GPU tests of MaskGit.inpaint: the frozen-position re-mask kernel (mmg_remask_frozen) against a torch restatement, the two anchors
(everything masked == generate(), nothing masked == the encoded image), token parity with the CPU oracle (tests/inpaint_oracle.py) in fp32
with injected noise, the bf16 teacher-forced flip rate, CUDA-graph replay and determinism, batch sharding, and the fused tail's overflow
rerun."""
import pytest
import torch

from oracle import synth
from tests import inpaint_oracle as IO, util
from tests.test_gpu_models import CFG, make_branch_maskgit, make_maskgit

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
MASK_ID = 1024


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _images(b, size, tag="inp.img"):
    return torch.from_numpy(synth.uniform(tag, (b, 3, size, size), 31)).cuda()


def _ragged_tokens(b, f, seed, fracs):
    """(b, f, f) bool token masks, image i regenerating about fracs[i] of its tokens (0 -> none, 1 -> all)."""
    g = torch.Generator().manual_seed(seed)
    m = torch.stack([torch.rand((f, f), generator=g) < fr if 0 < fr < 1 else torch.full((f, f), fr >= 1) for fr in fracs])
    return m


# ------------------------------------------------------------------------------------------------ kernel
def _ref_remask_frozen(ids, scores, frozen, counts, rows, mask_id):
    B, n = ids.shape
    ids = ids.clone()
    mp = torch.empty((B, rows), dtype=torch.int32)
    for b in range(B):
        free = (frozen[b] == 0).nonzero().flatten()
        order = free[torch.argsort(-scores[b, free], stable=True)]              # ties: lowest position first
        c = min(int(counts[b]), rows, len(free))
        sel = torch.sort(order[:c]).values
        ids[b, sel] = mask_id
        fz = frozen[b].nonzero().flatten()
        mp[b, :c] = sel.int()
        mp[b, c:] = int(fz[0]) if len(fz) else 0
    return ids, torch.full_like(scores, -1e5), mp


@pytest.mark.parametrize("n", [16, 256, 1024])
def test_remask_frozen_kernel_vs_torch(n):
    B = 6
    g = torch.Generator().manual_seed(n)
    frozen = (torch.rand((B, n), generator=g) < 0.5).to(torch.uint8)
    frozen[3] = 0                                 # no frozen position: its count is all rows
    frozen[5] = 1                                 # everything frozen
    frozen[0, 0] = 0; frozen[0, -1] = 1           # a pad position that is not position 0
    free = [int(f) for f in (frozen == 0).sum(1)]
    scores = torch.rand((B, n), generator=g)
    scores[::2] = torch.randint(0, 4, (3, n), generator=g).float()          # heavily tied rows
    ids = torch.randint(0, MASK_ID, (B, n), generator=g)
    for rows in (n, n // 2 + 1):
        # counts 0, 1, every non-frozen position, all rows (the image without frozen positions), about half, 0 (all frozen)
        counts = torch.tensor([0, 1, min(free[2], rows), rows, min(max(free[4] // 2, 1), rows), 0], dtype=torch.int32)
        idd, sd = ids.clone().cuda(), scores.clone().cuda()
        mp = torch.full((B, rows), -7, dtype=torch.int32, device="cuda")
        ops().remask_frozen(idd, sd, mp, frozen.cuda(), counts.cuda(), rows, MASK_ID)
        want_ids, want_sc, want_mp = _ref_remask_frozen(ids, scores, frozen, counts, rows, MASK_ID)
        assert torch.equal(idd.cpu(), want_ids)
        assert torch.equal(sd.cpu(), want_sc)
        assert torch.equal(mp.cpu(), want_mp)
        assert torch.equal(idd.cpu()[frozen.bool()], ids[frozen.bool()])


def test_remask_frozen_without_frozen_positions_equals_remask():
    """Nothing frozen and every count equal to num_masked: byte-identical to mmg_remask."""
    B, n, nm = 4, 256, 97
    g = torch.Generator().manual_seed(4)
    scores = torch.randint(0, 8, (B, n), generator=g).float().cuda()
    ids = torch.randint(0, MASK_ID, (B, n), generator=g).cuda()
    i1, s1, m1 = ids.clone(), scores.clone(), torch.zeros((B, n), dtype=torch.int32, device="cuda")
    i2, s2, m2 = ids.clone(), scores.clone(), torch.zeros((B, n), dtype=torch.int32, device="cuda")
    ops().remask(i1, s1, m1, nm, MASK_ID)
    ops().remask_frozen(i2, s2, m2, torch.zeros((B, n), dtype=torch.uint8, device="cuda"), torch.full((B,), nm, dtype=torch.int32, device="cuda"),
                        nm, MASK_ID)
    assert torch.equal(i1, i2) and torch.equal(s1, s2) and torch.equal(m1, m2)


# ------------------------------------------------------------------------------------------------ anchors
def _te():
    return util.text_embeds("g4.te", 3, 8, 128, 14).cuda()


def _setup(mg, te):
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    return mg


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("rng", ["mmg", "aten"])
def test_full_mask_equals_generate_bf16(graph, rng):
    mg = _setup(make_maskgit("bf16"), _te())
    mg.use_cuda_graph, mg.sampler_rng, mg.sampler_seed = graph, rng, 42
    img = _images(3, 16)
    torch.manual_seed(3)
    gi, gids = mg.generate(["a"] * 3, timesteps=8, return_ids=True)
    torch.manual_seed(3)
    ii, iids = mg.inpaint(["a"] * 3, img, torch.ones((3, 16, 16), dtype=torch.bool), timesteps=8, return_ids=True)
    assert torch.equal(iids, gids) and torch.equal(ii, gi)


@pytest.mark.parametrize("name", ["gen_selfcond_small", "gen_critic_small", "gen_selfcritic_small", "gen_remask_prev_small"])
def test_full_mask_equals_generate_optional_branches(name):
    """bf16 Philox under the CUDA graph, with self-conditioning, a TokenCritic, the SelfCritic and can_remask_prev_masked."""
    mg, kw, _ = make_branch_maskgit(name, "bf16")
    _setup(mg, _te())
    mg.sampler_seed = 5
    gi, gids = mg.generate(["a"] * 3, timesteps=8, return_ids=True, **kw)
    ii, iids = mg.inpaint(["a"] * 3, _images(3, 16), torch.ones((3, 4, 4), dtype=torch.bool), timesteps=8, return_ids=True, **kw)
    assert torch.equal(iids, gids) and torch.equal(ii, gi)


def test_full_mask_equals_generate_fp32_injected_noise():
    mg = _setup(make_maskgit("fp32"), _te())
    mg.sampler_noise_fn = util.torch_noise_fn(777)
    gi, gids = mg.generate(["a"] * 3, timesteps=8, return_ids=True)
    mg.sampler_noise_fn = util.torch_noise_fn(777)
    ii, iids = mg.inpaint(["a"] * 3, _images(3, 16), torch.ones((3, 1, 16, 16)), timesteps=8, return_ids=True)
    assert torch.equal(iids, gids) and torch.equal(ii, gi)


@pytest.mark.parametrize("precision,graph", [("bf16", True), ("bf16", False), ("fp32", False)])
def test_empty_mask_returns_the_encoded_image(precision, graph):
    mg = _setup(make_maskgit(precision), _te())
    mg.use_cuda_graph, mg.sampler_seed = graph, 9
    img = _images(3, 16)
    out, ids = mg.inpaint(["a"] * 3, img, torch.zeros((3, 16, 16), dtype=torch.bool), timesteps=6, return_ids=True)
    known = mg.vae.encode_ids(img)
    assert torch.equal(ids, known)
    assert torch.equal(out, mg.vae.decode_from_ids(known))


# ------------------------------------------------------------------------------------------------ parity with the oracle
def _oracle_check(mg, sd, cfg, te, img, regen_tok, T, cond=None, **kw):
    b = img.shape[0]
    mg.sampler_noise_fn = util.torch_noise_fn(901)
    _, ids = mg.inpaint(["a"] * b, img, regen_tok.cuda(), cond_images=cond, timesteps=T, return_ids=True, **kw)
    known = mg.vae.encode_ids(img).reshape(b, -1).cpu()
    cond_ids = None if cond is None else mg.cond_vae.encode_ids(cond).cpu()
    okw = {}
    if "critic_noise_scale" in kw:
        okw = dict(critic=dict(kind="token", sd=util.critic_sd(1024, 128, 16, 1, 2, seed=22, text_dim=128), cfg=dict(heads=2, depth=1)),
                   critic_noise_scale=kw["critic_noise_scale"])
    want = IO.inpaint_ids(sd, cfg, te.cpu(), known, regen_tok.reshape(b, -1), MASK_ID, util.torch_noise_fn(901), cond_ids=cond_ids,
                          timesteps=T, **okw)
    got = ids.reshape(b, -1).cpu()
    assert torch.equal(got, want), int((got != want).sum())
    frozen = ~regen_tok.reshape(b, -1)
    assert torch.equal(got[frozen], known[frozen])
    return want


def test_fp32_ragged_masks_token_identical_to_oracle():
    mg = _setup(make_maskgit("fp32"), _te())
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    _oracle_check(mg, sd, CFG, _te(), _images(3, 16), _ragged_tokens(3, 4, 1, [0, 1, 0.5]), 8)


def test_fp32_superres_token_identical_to_oracle():
    """superres: 32 x 32 images (8 x 8 tokens) conditioned on 16 x 16 images; pixel masks (a centre box and a border: outpainting)."""
    mg = make_maskgit("fp32", superres=True)
    te = _te()[:2]
    _setup(mg, te)
    sd = util.transformer_sd(1024, 128, 64, 2, 2, seed=15, text_dim=128)
    pm = torch.zeros((2, 32, 32), dtype=torch.bool)
    pm[0, 9:22, 5:19] = True
    pm[1] = True; pm[1, 8:24, 8:24] = False
    from muse_maskgit_pytorch_b200.muse_maskgit import regen_tokens
    regen = regen_tokens(pm, 2, 32, 8)
    assert 0 < int(regen[0].sum()) < int(regen[1].sum()) < 64
    want = _oracle_check(mg, sd, CFG, te, _images(2, 32), regen, 8, cond=_images(2, 16, "inp.cond"))
    mg.sampler_noise_fn = util.torch_noise_fn(901)
    _, ids_px = mg.inpaint(["a"] * 2, _images(2, 32), pm.cuda(), cond_images=_images(2, 16, "inp.cond"), timesteps=8, return_ids=True)
    assert torch.equal(ids_px.reshape(2, -1).cpu(), want)                 # the pixel mask pools to the same tokens


def test_fp32_token_critic_token_identical_to_oracle():
    mg, kw, _ = make_branch_maskgit("gen_critic_small", "fp32")
    _setup(mg, _te())
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    _oracle_check(mg, sd, CFG, _te(), _images(3, 16), _ragged_tokens(3, 4, 2, [0.3, 1, 0.7]), 8, **kw)


def test_bf16_teacher_forced_flip_rate():
    """bf16 tail fed the oracle's ids and noise at every step (the pad rows built as mmg_remask_frozen builds them): sampled-token flips
    on the regenerated positions below the 8 % bound of generate(); frozen ids never change."""
    mg = make_maskgit("bf16")
    tr = mg.transformer
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    te = util.text_embeds("g4.te", 3, 8, 128, 14)
    regen = _ragged_tokens(3, 4, 3, [1, 0.5, 0.25]).reshape(3, -1)
    known = mg.vae.encode_ids(_images(3, 16)).reshape(3, -1).cpu()
    trace = []
    IO.inpaint_ids(sd, CFG, te, known, regen, MASK_ID, util.torch_noise_fn(777), timesteps=18, trace=trace)
    ctx = tr._prepare_context(te.cuda(), None, [False, True])
    P = tr._packed()
    flips = total = 0
    b, n = known.shape
    for st in trace:
        rows = max(max(st["num_masked"]), 1)
        mp = torch.empty((b, rows), dtype=torch.int32)
        for i in range(b):
            pos = (st["ids_in"][i] == MASK_ID).nonzero().flatten()
            fz = (~regen[i]).nonzero().flatten()
            mp[i, :len(pos)] = pos.int()
            mp[i, len(pos):] = int(fz[0]) if len(fz) else 0
        ids_in = st["ids_in"].cuda()
        x = tr._run_blocks(ids_in, ctx, 2)
        e = torch.empty((b * rows, 128), device="cuda", dtype=P["adt"])
        mpd = mp.cuda().contiguous()
        ops().final_embed(x[:b * n], x[b * n:], P["gf"], mpd, e, b, n, rows, 3.0)
        lg = torch.empty((b * rows, 1024), device="cuda")
        ops().linear(e, P["wlog"], lg)
        ids = ids_in.clone(); sc = torch.full((b, n), -1e5, device="cuda")
        ops().logits_sample(lg, mpd, ids, sc, rows, 103, float(st["temperature"]), u=st["u"].cuda().contiguous(), only_masked_id=MASK_ID)
        ids = ids.cpu()
        is_mask = st["ids_in"] == MASK_ID
        assert torch.equal(ids[~is_mask], st["ids_in"][~is_mask])
        flips += int((ids[is_mask] != st["ids_out"][is_mask]).sum()); total += int(is_mask.sum())
    print(f"bf16 inpaint teacher-forced flip rate {flips}/{total}")
    assert total > 150 and flips / total < 0.08


# ------------------------------------------------------------------------------------------------ graph, determinism, sharding
def test_graph_replay_determinism_and_repack():
    mg = _setup(make_maskgit("bf16"), _te())
    mg.sampler_seed = 5
    img = _images(3, 16)
    m1 = _ragged_tokens(3, 4, 5, [0.5, 1, 0])
    m2 = m1.clone(); m2[0] = torch.flip(m1[0], dims=(0, 1)); m2[2, 0, 0] = True         # other positions, same N_max (16)
    run = lambda m: mg.inpaint(["a"] * 3, img, m.cuda(), timesteps=8, return_ids=True)
    a, ida = run(m1)
    keys = list(mg._graphs)
    graph_obj = mg._graphs[keys[-1]].graph
    a2, ida2 = run(m1)
    c, idc = run(m2)                                           # same N_max: the captured graph replays with the new mask
    assert list(mg._graphs) == keys and mg._graphs[keys[-1]].graph is graph_obj
    assert keys[-1][-1] == ("inpaint", 16)
    mg.use_cuda_graph = False
    b_, idb = run(m1)
    d, idd = run(m2)
    assert torch.equal(ida, ida2) and torch.equal(a, a2) and torch.equal(ida, idb) and torch.equal(a, b_)
    assert torch.equal(idc, idd) and torch.equal(c, d) and not torch.equal(ida, idc)
    # load_state_dict: the graphs are dropped and the new weights are packed before the next call
    mg.use_cuda_graph = True
    sd = {k: v.clone() for k, v in mg.state_dict().items()}
    sd["transformer.to_logits.weight"] *= 1.5
    pack0 = mg.transformer._pack
    mg.load_state_dict(sd)
    e, ide = run(m1)
    assert mg.transformer._pack is not None and mg.transformer._pack is not pack0
    mg.use_cuda_graph = False
    f_, idf = run(m1)
    assert torch.equal(ide, idf) and torch.equal(e, f_)


def test_row_offset_shard_reproduces_its_rows():
    mg = _setup(make_maskgit("bf16"), _te())
    te = _te()
    mg.sampler_seed = 11
    img = _images(3, 16)
    m = _ragged_tokens(3, 4, 6, [1, 0.4, 0.7])
    _, ida = mg.inpaint(["a"] * 3, img, m.cuda(), timesteps=8, return_ids=True)
    mg.row_offset = 1
    mg.transformer.encode_text = lambda texts: te[1:1 + len(texts)]
    _, idc = mg.inpaint(["a"] * 2, img[1:], m[1:].cuda(), timesteps=8, return_ids=True)
    assert torch.equal(idc, ida[1:])


def test_fused_tail_overflow_reruns_as_inpaint():
    """Constant logits (zero to_logits, V = 65536): every sampled row, pad rows included, falls back and the first step overflows the fused
    tail's fallback; the materialised rerun is an inpaint call (frozen ids kept) equal to asking for the materialised tail directly."""
    from tests.test_gpu_fused_tail import _degenerate_maskgit
    mg, b = _degenerate_maskgit()
    mg.sampler_seed = 42
    img = _images(b, 16)
    m = torch.rand((b, 4, 4), generator=torch.Generator().manual_seed(7)) < 0.6
    m[0] = True
    known = mg.vae.encode_ids(img)
    mg.use_fused_tail, mg.last_fused_fallback_rows = True, 0
    img_f, ids_f = mg.inpaint(["a"] * b, img, m.cuda(), timesteps=4, return_ids=True)
    assert mg.last_fused_fallback_rows > 128
    mg.use_fused_tail = False
    img_m, ids_m = mg.inpaint(["a"] * b, img, m.cuda(), timesteps=4, return_ids=True)
    assert torch.equal(ids_f, ids_m) and torch.equal(img_f, img_m)
    assert torch.equal(ids_f[~m.cuda()], known[~m.cuda()])

"""GPU tests of MaskGit.edit (mask-free editing): the selection kernel (mmg_edit_select) against a torch restatement with injected and Philox
keys, the anchors (one full-fraction iteration == generate() / inpaint(), zero iterations == the encoded image), token parity with the CPU
oracle (tests/edit_oracle.py) in fp32 with injected noise, kept tokens in bf16 and fp8, CUDA-graph replay and determinism, batch sharding,
the fused tail's overflow rerun and the argument checks."""
import pytest
import torch

from oracle import synth
from tests import edit_oracle as EO, util
from tests.test_gpu_models import CFG, make_branch_maskgit, make_maskgit

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
MASK_ID = 1024


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _images(b, size, tag="edit.img"):
    return torch.from_numpy(synth.uniform(tag, (b, 3, size, size), 31)).cuda()


def _ragged_tokens(b, f, seed, fracs):
    """(b, f, f) bool token masks, image i editable on about fracs[i] of its tokens (0 -> none, 1 -> all)."""
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.rand((f, f), generator=g) < fr if 0 < fr < 1 else torch.full((f, f), fr >= 1) for fr in fracs])


def _te():
    return util.text_embeds("g4.te", 3, 8, 128, 14).cuda()


def _setup(mg, te):
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    return mg


# ------------------------------------------------------------------------------------------------ kernel
def _kernel_case(n, seed):
    B = 7
    g = torch.Generator().manual_seed(seed)
    keep = (torch.rand((B, n), generator=g) < torch.rand((B, 1), generator=g)).to(torch.uint8)       # ragged keep maps
    keep[3] = 0                                   # everything editable
    keep[5] = 1                                   # nothing editable
    free = [int(f) for f in (keep == 0).sum(1)]
    # counts 0, 1, every editable position, n (nothing kept), about half, 0 (nothing editable), more than the editable positions
    counts = torch.tensor([0, 1, free[2], n, max(free[4] // 2, 1), 0, n], dtype=torch.int32)
    ids = torch.randint(0, MASK_ID, (B, n), generator=g)
    return keep, counts, ids


def _check_select(keys, keep, counts, ids, u, seed_dev, iteration, row_offset):
    B, n = ids.shape
    idd, sd = ids.clone().cuda(), torch.rand((B, n), device="cuda")
    fz = torch.full((B, n), 7, dtype=torch.uint8, device="cuda")
    ops().edit_select(idd, sd, fz, keep.cuda(), counts.cuda(), MASK_ID, iteration, u=u, seed_dev=seed_dev, row_offset=row_offset)
    sel = EO.select(keys, keep == 0, [int(c) for c in counts])
    want_ids = ids.clone(); want_ids[sel] = MASK_ID
    assert torch.equal(fz.cpu(), (~sel).to(torch.uint8))
    assert torch.equal(idd.cpu(), want_ids)
    assert torch.equal(sd.cpu(), torch.zeros((B, n)))
    assert [int(c) for c in sel.sum(1)] == [min(int(c), int(f)) for c, f in zip(counts, (keep == 0).sum(1))]


@pytest.mark.parametrize("n", [16, 256, 1024])
def test_edit_select_injected_keys_vs_torch(n):
    keep, counts, ids = _kernel_case(n, n)
    g = torch.Generator().manual_seed(n + 1)
    keys = torch.rand((7, n), generator=g)
    keys[::2] = torch.randint(0, 4, (4, n), generator=g).float() / 4          # forced ties
    _check_select(keys, keep, counts, ids, keys.cuda().contiguous(), None, 0, 0)


@pytest.mark.parametrize("n", [16, 256, 1024])
def test_edit_select_philox_keys_vs_oracle(n):
    keep, counts, ids = _kernel_case(n, n + 2)
    seed = (3 << 50) + 977
    seed_dev = torch.tensor([seed], dtype=torch.int64, device="cuda")
    for iteration, row_offset in ((0, 0), (5, 3)):
        keys = EO.philox_keys(seed, iteration, 7, n, row_offset=row_offset)
        _check_select(keys, keep, counts, ids, None, seed_dev, iteration, row_offset * n)


# ------------------------------------------------------------------------------------------------ anchors
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_one_full_iteration_equals_generate_and_inpaint_bf16(graph):
    mg = _setup(make_maskgit("bf16"), _te())
    mg.use_cuda_graph, mg.sampler_seed = graph, 42
    img = _images(3, 16)
    gi, gids = mg.generate(["a"] * 3, timesteps=8, return_ids=True)
    ei, eids = mg.edit(["a"] * 3, img, iterations=1, fraction=1.0, timesteps=8, return_ids=True)
    assert torch.equal(eids, gids) and torch.equal(ei, gi)
    m = _ragged_tokens(3, 4, 1, [0.3, 1, 0.6]).cuda()
    ii, iids = mg.inpaint(["a"] * 3, img, m, timesteps=8, return_ids=True)
    ei, eids = mg.edit(["a"] * 3, img, mask=m, iterations=1, fraction=1.0, timesteps=8, return_ids=True)
    assert torch.equal(eids, iids) and torch.equal(ei, ii)
    known = mg.vae.encode_ids(img)
    assert torch.equal(eids[~m], known[~m]) and not (eids[m] == known[m]).all()


@pytest.mark.parametrize("precision,graph", [("bf16", True), ("bf16", False), ("fp32", False)])
def test_zero_iterations_return_the_encoded_image(precision, graph):
    mg = _setup(make_maskgit(precision), _te())
    mg.use_cuda_graph, mg.sampler_seed = graph, 9
    img = _images(3, 16)
    out, ids = mg.edit(["a"] * 3, img, iterations=0, return_ids=True)
    known = mg.vae.encode_ids(img)
    assert torch.equal(ids, known)
    assert torch.equal(out, mg.vae.decode_from_ids(known))


# ------------------------------------------------------------------------------------------------ parity with the oracle
def _oracle_check(mg, sd, te, img, editable_tok, iterations, fraction, T, cond=None, **kw):
    b = img.shape[0]
    mg.sampler_noise_fn = util.torch_noise_fn(901)
    mask = None if editable_tok is None else editable_tok.cuda()
    _, ids = mg.edit(["a"] * b, img, mask=mask, iterations=iterations, fraction=fraction, timesteps=T, cond_images=cond, return_ids=True, **kw)
    known = mg.vae.encode_ids(img).reshape(b, -1).cpu()
    n = known.shape[1]
    editable = torch.ones((b, n), dtype=torch.bool) if editable_tok is None else editable_tok.reshape(b, -1)
    cond_ids = None if cond is None else mg.cond_vae.encode_ids(cond).cpu()
    okw = {}
    if "critic_noise_scale" in kw:
        okw = dict(critic=dict(kind="token", sd=util.critic_sd(1024, 128, 16, 1, 2, seed=22, text_dim=128), cfg=dict(heads=2, depth=1)),
                   critic_noise_scale=kw["critic_noise_scale"])
    trace = []
    want = EO.edit_ids(sd, CFG, te.cpu(), known, editable, MASK_ID, util.torch_noise_fn(901), iterations=iterations, fraction=fraction,
                       timesteps=T, cond_ids=cond_ids, trace=trace, **okw)
    got = ids.reshape(b, -1).cpu()
    assert torch.equal(got, want), int((got != want).sum())
    assert torch.equal(got[~editable], known[~editable])
    assert sum(bool((t["ids"] != (known if i == 0 else trace[i - 1]["ids"])).any()) for i, t in enumerate(trace)) > 0
    return want


@pytest.mark.parametrize("fracs", [None, [0, 1, 0.5]], ids=["no_mask", "ragged"])
def test_fp32_token_identical_to_oracle(fracs):
    mg = _setup(make_maskgit("fp32"), _te())
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    tok = None if fracs is None else _ragged_tokens(3, 4, 1, fracs)
    _oracle_check(mg, sd, _te(), _images(3, 16), tok, 3, 0.4, 3)


def test_fp32_token_critic_token_identical_to_oracle():
    mg, kw, _ = make_branch_maskgit("gen_critic_small", "fp32")
    _setup(mg, _te())
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    _oracle_check(mg, sd, _te(), _images(3, 16), _ragged_tokens(3, 4, 2, [0.3, 1, 0.7]), 2, 0.5, 4, **kw)


def test_fp32_superres_token_identical_to_oracle():
    """superres: 32 x 32 images (8 x 8 tokens) conditioned on 16 x 16 images, a ragged pixel mask pooled to tokens."""
    from muse_maskgit_pytorch_b200.muse_maskgit import regen_tokens
    mg = make_maskgit("fp32", superres=True)
    te = _te()[:2]
    _setup(mg, te)
    sd = util.transformer_sd(1024, 128, 64, 2, 2, seed=15, text_dim=128)
    pm = torch.zeros((2, 32, 32), dtype=torch.bool)
    pm[0, 9:22, 5:19] = True
    pm[1] = True; pm[1, 8:24, 8:24] = False
    want = _oracle_check(mg, sd, te, _images(2, 32), regen_tokens(pm, 2, 32, 8), 3, 0.3, 3, cond=_images(2, 16, "edit.cond"))
    mg.sampler_noise_fn = util.torch_noise_fn(901)
    _, ids_px = mg.edit(["a"] * 2, _images(2, 32), mask=pm.cuda(), iterations=3, fraction=0.3, timesteps=3, cond_images=_images(2, 16, "edit.cond"),
                        return_ids=True)
    assert torch.equal(ids_px.reshape(2, -1).cpu(), want)                 # the pixel mask pools to the same tokens


# ------------------------------------------------------------------------------------------------ kept tokens in bf16 / fp8
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_tokens_outside_the_mask_are_kept(precision):
    from tests.test_gpu_fp8 import small_maskgit
    mg = small_maskgit(precision)                               # 64 x 64 images, 16 x 16 tokens
    mg.sampler_seed = 23
    img = _images(3, 64)
    known = mg.vae.encode_ids(img)
    m = _ragged_tokens(3, 16, 4, [0.2, 0.9, 0.5]).cuda()
    _, ids = mg.edit(["a"] * 3, img, mask=m, iterations=4, fraction=0.25, timesteps=3, return_ids=True)
    assert torch.equal(ids[~m], known[~m]) and not torch.equal(ids, known)
    _, ids1 = mg.edit(["a"] * 3, img, iterations=1, fraction=0.1, timesteps=3, return_ids=True)
    changed = (ids1 != known).reshape(3, -1).sum(1)
    assert (changed <= int(0.1 * 256)).all() and int(changed.sum()) > 0, changed.tolist()


# ------------------------------------------------------------------------------------------------ graph, determinism, sharding
def test_graph_replay_determinism_and_weight_edit():
    mg = _setup(make_maskgit("bf16"), _te())
    mg.sampler_seed = 5
    img = _images(3, 16)
    m = _ragged_tokens(3, 4, 5, [0.5, 1, 0]).cuda()
    run = lambda: mg.edit(["a"] * 3, img, mask=m, iterations=3, fraction=0.5, timesteps=4, return_ids=True)
    a, ida = run()
    key = list(mg._graphs)[-1]
    graph_obj = mg._graphs[key].graph
    a2, ida2 = run()
    assert mg._graphs[key].graph is graph_obj and key[-1] == ("edit", 3, 8)
    mg.use_cuda_graph = False
    b_, idb = run()
    assert torch.equal(ida, ida2) and torch.equal(a, a2) and torch.equal(ida, idb) and torch.equal(a, b_)
    # an in-place weight edit drops the packed weights and the captured graph
    mg.use_cuda_graph = True
    mg.transformer.to_logits.weight.mul_(1.5)
    c, idc = run()
    assert mg._graphs[key].graph is not graph_obj
    mg.use_cuda_graph = False
    d, idd = run()
    assert torch.equal(idc, idd) and torch.equal(c, d) and not torch.equal(idc, ida)


def test_row_offset_shard_reproduces_its_rows():
    mg = _setup(make_maskgit("bf16"), _te())
    te = _te()
    mg.sampler_seed = 11
    img = _images(3, 16)
    m = _ragged_tokens(3, 4, 6, [1, 0.4, 0.7])
    _, ida = mg.edit(["a"] * 3, img, mask=m.cuda(), iterations=3, fraction=0.5, timesteps=4, return_ids=True)
    mg.row_offset = 1
    mg.transformer.encode_text = lambda texts: te[1:1 + len(texts)]
    _, idc = mg.edit(["a"] * 2, img[1:], mask=m[1:].cuda(), iterations=3, fraction=0.5, timesteps=4, return_ids=True)
    assert torch.equal(idc, ida[1:])


def test_fused_tail_overflow_reruns_as_edit():
    """Constant logits (zero to_logits, V = 65536): every sampled row falls back and the first step (16 images x 9 rows) overflows the fused
    tail's fallback; the materialised rerun is an edit call equal to asking for the materialised tail directly, with the kept tokens kept."""
    from tests.test_gpu_fused_tail import _degenerate_maskgit
    mg, b = _degenerate_maskgit()
    mg.sampler_seed = 42
    img = _images(b, 16)
    m = torch.rand((b, 4, 4), generator=torch.Generator().manual_seed(7)) < 0.6
    m[0] = True
    known = mg.vae.encode_ids(img)
    mg.use_fused_tail, mg.last_fused_fallback_rows = True, 0
    img_f, ids_f = mg.edit(["a"] * b, img, mask=m.cuda(), iterations=2, fraction=0.6, timesteps=3, return_ids=True)
    assert mg.last_fused_fallback_rows > 128
    mg.use_fused_tail = False
    img_m, ids_m = mg.edit(["a"] * b, img, mask=m.cuda(), iterations=2, fraction=0.6, timesteps=3, return_ids=True)
    assert torch.equal(ids_f, ids_m) and torch.equal(img_f, img_m)
    assert torch.equal(ids_f[~m.cuda()], known[~m.cuda()])


# ------------------------------------------------------------------------------------------------ arguments
def test_argument_errors():
    mg = _setup(make_maskgit("bf16"), _te())
    img = _images(3, 16)
    for kw in (dict(fraction=0), dict(fraction=1.5), dict(fraction=-0.1), dict(iterations=-1), dict(iterations=1.5), dict(timesteps=0)):
        with pytest.raises(ValueError):
            mg.edit(["a"] * 3, img, **kw)
    mg.sampler_rng = "aten"
    with pytest.raises(ValueError, match="aten"):
        mg.edit(["a"] * 3, img)
    mg.sampler_rng = "mmg"
    with pytest.raises(ValueError):
        mg.edit(["a"] * 3, img[:2])

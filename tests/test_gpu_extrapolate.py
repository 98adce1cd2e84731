"""GPU tests of MaskGit.extrapolate (image extrapolation): the window kernel (mmg_extrapolate_window) against torch slicing, token parity with
the CPU oracle (tests/extrapolate_oracle.py) in fp32 with injected noise, the anchors (one full-width window == generate(), input tokens ==
vae.encode_ids, pixels == vae.decode_from_ids of the canvas), CUDA-graph replay and determinism, batch sharding, the fused tail's overflow
rerun and the argument checks."""
import pytest
import torch

from muse_maskgit_pytorch_b200 import parallel
from oracle import synth
from tests import extrapolate_oracle as XO, util
from tests.test_gpu_models import CFG, M, make_branch_maskgit, make_maskgit, small_transformer

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
MASK_ID = 1024
F, P = 4, 4                    # the small models: 16 x 16 images, 4 x 4 tokens of 4 x 4 pixels


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _images(b, h=16, w=16, tag="extrap.img"):
    return torch.from_numpy(synth.uniform(tag, (b, 3, h, w), 33)).cuda()


def _input(b, direction, extra=0):
    """(b, 3, H, W) images whose long side along `direction` is extra tokens past the 16-pixel frame."""
    return _images(b, 16 + 4 * extra, 16) if direction in ("down", "up") else _images(b, 16, 16 + 4 * extra)


def _te():
    return util.text_embeds("g4.te", 3, 8, 128, 14).cuda()


def _setup(mg, te):
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    return mg


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("direction", XO.DIRECTIONS)
@pytest.mark.parametrize("stride,extra", [(1, 0), (2, 3), (4, 1)])
def test_window_kernel_vs_torch(direction, stride, extra):
    B, K = 7, 3
    vertical = direction in ("down", "up")
    in_h, in_w = (F + extra, F) if vertical else (F, F + extra)
    (H, W), _, corners = XO.plan(direction, in_h, in_w, F, stride, K)
    strip = XO.strip(direction, F, stride)
    g = torch.Generator().manual_seed(stride * 10 + extra)
    for corner in (corners[0], corners[-1]):
        r, c = corner
        canvas = torch.randint(0, MASK_ID + 1, (B, H, W), generator=g)
        ids = torch.randint(0, MASK_ID, (B, F * F), generator=g)
        cv, idd, sd = canvas.cuda(), ids.cuda(), torch.rand((B, F * F), device="cuda")
        ops().extrapolate_window(cv, idd, sd, corner, direction, stride, MASK_ID)
        want = canvas[:, r:r + F, c:c + F].clone()
        want[:, strip] = MASK_ID
        assert torch.equal(idd.cpu(), want.reshape(B, -1)) and torch.equal(sd.cpu(), torch.zeros((B, F * F)))
        assert torch.equal(cv.cpu(), canvas)                                     # a load leaves the canvas alone
        # store: only the strip of the window moves into the canvas
        ids2 = torch.randint(0, MASK_ID, (B, F * F), generator=g)
        idd.copy_(ids2.cuda())
        sd.fill_(0.5)
        ops().extrapolate_window(cv, idd, sd, corner, direction, stride, MASK_ID, store=True)
        want = canvas.clone()
        block = want[:, r:r + F, c:c + F]
        block[:, strip] = ids2.reshape(B, F, F)[:, strip]
        assert torch.equal(cv.cpu(), want)
        assert torch.equal(idd.cpu(), ids2) and bool((sd == 0.5).all())


def test_window_kernel_rejects_a_window_outside_the_canvas():
    from muse_maskgit_pytorch_b200 import _lib
    cv = torch.zeros((2, 4, 8), dtype=torch.long, device="cuda")
    idd, sd = torch.zeros((2, 16), dtype=torch.long, device="cuda"), torch.zeros((2, 16), device="cuda")
    with pytest.raises(_lib.MMGError, match="outside"):
        ops().extrapolate_window(cv, idd, sd, (0, 5), "right", 2, MASK_ID)


# ------------------------------------------------------------------------------------------------ parity with the oracle
def _oracle_check(mg, sd, cfg, te, img, direction, K, stride, T, okw=None, cond_scale=3, **kw):
    """fp32 extrapolate() with injected noise against the oracle; a per-image cond_scale is checked row by row against oracle runs at each
    image's value (the oracle takes one scale per call; images are independent under the same noise)."""
    b = img.shape[0]
    mg.sampler_noise_fn = util.torch_noise_fn(901)
    out, canvas = mg.extrapolate(["a"] * b, img, direction=direction, amount=K * stride * P, stride=stride, timesteps=T, cond_scale=cond_scale,
                                 return_ids=True, **kw)
    known = mg.vae.encode_ids(img).cpu()
    scales = cond_scale if isinstance(cond_scale, (list, tuple)) else [cond_scale] * b
    want = torch.empty_like(canvas.cpu())
    for s in sorted(set(scales)):
        rows = [i for i, v in enumerate(scales) if v == s]
        full = XO.extrapolate_ids(sd, cfg, te.cpu()[:b], known, direction, K, stride, MASK_ID, util.torch_noise_fn(901), timesteps=T,
                                  cond_scale=float(s), **(okw or {}))
        want[rows] = full[rows]
    got = canvas.cpu()
    assert got.shape == want.shape and torch.equal(got, want), int((got != want).sum())
    (H, W), (r, c), _ = XO.plan(direction, known.shape[1], known.shape[2], F, stride, K)
    assert torch.equal(got[:, r:r + known.shape[1], c:c + known.shape[2]], known)
    assert out.shape == (b, 3, H * P, W * P)
    return got


@pytest.mark.parametrize("direction", XO.DIRECTIONS)
@pytest.mark.parametrize("K,stride,extra", [(1, 2, 0), (3, 1, 0), (3, 2, 2)])
def test_fp32_token_identical_to_oracle(direction, K, stride, extra):
    mg = _setup(make_maskgit("fp32"), _te())
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    _oracle_check(mg, sd, CFG, _te(), _input(3, direction, extra), direction, K, stride, 3)


@pytest.mark.parametrize("name", ["gen_critic_small", "gen_selfcritic_small"])
def test_fp32_critic_branches_token_identical_to_oracle(name):
    from tests.test_oracle_golden import _branch_case
    mg, kw, _ = make_branch_maskgit(name, "fp32")
    _setup(mg, _te())
    sd, cfg, okw, _ = _branch_case(name)
    _oracle_check(mg, sd, cfg, _te(), _input(3, "left", 1), "left", 2, 2, 3, okw=okw, **kw)


def test_fp32_per_image_cond_scale_token_identical_to_oracle():
    mg = _setup(make_maskgit("fp32"), _te())
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    _oracle_check(mg, sd, CFG, _te(), _input(3, "down"), "down", 2, 2, 3, cond_scale=[3.0, 1.0, 2.0])


# ------------------------------------------------------------------------------------------------ anchors
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_one_full_width_window_equals_generate_bf16(graph):
    mg = _setup(make_maskgit("bf16"), _te())
    mg.use_cuda_graph, mg.sampler_seed = graph, 42
    img = _images(3)
    _, gids = mg.generate(["a"] * 3, timesteps=8, return_ids=True)
    out, canvas = mg.extrapolate(["a"] * 3, img, amount=16, stride=F, timesteps=8, return_ids=True)
    assert canvas.shape == (3, F, 2 * F) and out.shape == (3, 3, 16, 32)
    assert torch.equal(canvas[:, :, F:], gids)
    assert torch.equal(canvas[:, :, :F], mg.vae.encode_ids(img))
    assert torch.equal(out, mg.vae.decode_from_ids(canvas))


@pytest.mark.parametrize("precision", ["bf16", "fp32", "fp8"])
def test_input_tokens_kept_and_pixels_are_the_canvas_decode(precision):
    if precision == "fp8":
        from tests.test_gpu_fp8 import small_maskgit
        mg, size, f = small_maskgit("fp8"), 64, 16              # 64 x 64 images, 16 x 16 tokens
    else:
        mg, size, f = _setup(make_maskgit(precision), _te()), 16, F
    mg.sampler_seed = 23
    for direction in XO.DIRECTIONS:
        vertical = direction in ("down", "up")
        img = _images(3, size + 8 if vertical else size, size if vertical else size + 8, tag="extrap.keep")
        stride = f // 2
        out, canvas = mg.extrapolate(["a"] * 3, img, direction=direction, amount=2 * stride * P, timesteps=3, return_ids=True)
        known = mg.vae.encode_ids(img)
        (H, W), (r, c), _ = XO.plan(direction, known.shape[1], known.shape[2], f, stride, 2)
        assert canvas.shape == (3, H, W) and out.shape == (3, 3, H * P, W * P)
        assert torch.equal(canvas[:, r:r + known.shape[1], c:c + known.shape[2]], known)
        assert int(canvas.max()) < mg.transformer.num_tokens and int(canvas.min()) >= 0          # every new token generated
        assert torch.equal(out, mg.vae.decode_from_ids(canvas))


# ------------------------------------------------------------------------------------------------ graph, determinism, sharding
def test_graph_replay_determinism_and_weight_edit():
    mg = _setup(make_maskgit("bf16"), _te())
    mg.sampler_seed = 5
    img = _input(3, "right", 1)
    run = lambda: mg.extrapolate(["a"] * 3, img, amount=24, stride=2, timesteps=4, return_ids=True)
    a, ida = run()
    key = list(mg._graphs)[-1]
    graph_obj = mg._graphs[key].graph
    a2, ida2 = run()
    assert mg._graphs[key].graph is graph_obj and key[-1] == ("extrapolate", "right", 3, 2, (F, 5 + 6))
    mg.use_cuda_graph = False
    b_, idb = run()
    assert torch.equal(ida, ida2) and torch.equal(a, a2) and torch.equal(ida, idb) and torch.equal(a, b_)
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
    img = _images(3)
    _, ida = mg.extrapolate(["a"] * 3, img, direction="up", amount=24, stride=2, timesteps=4, return_ids=True)
    mg.row_offset = 1
    mg.transformer.encode_text = lambda texts: te[1:1 + len(texts)]
    _, idc = mg.extrapolate(["a"] * 2, img[1:], direction="up", amount=24, stride=2, timesteps=4, return_ids=True)
    assert torch.equal(idc, ida[1:])


@pytest.mark.parametrize("world", [2, 3])
def test_virtual_ranks_equal_the_unsharded_call(world):
    from tests.test_gpu_sharded_entry_points import SCALES, _compare, _te as _te_b, _unsharded, _virtual_ranks
    mg = make_maskgit("bf16")
    b = len(SCALES)
    texts, te, img = ["a"] * b, _te_b(b), _images(b, 16, 20)
    kw = dict(direction="right", amount=16, stride=2, timesteps=3, cond_scale=SCALES, temperature=torch.linspace(0.5, 1.5, b), return_ids=True)
    full_img, full_ids = _unsharded(mg.extrapolate, (mg,), texts, te, 25, images=img, **kw)
    img_s, ids_s = _virtual_ranks(mg.extrapolate, (mg,), texts, world, 25, text_embeds=te, images=img, **kw)
    _compare(f"extrapolate world {world}", full_ids, ids_s, [full_img], [img_s])
    # the public entry point in a single process, and what a rank without rows contributes
    mg.transformer.encode_text = lambda t: te
    torch.manual_seed(25)
    got = parallel.extrapolate_sharded(mg, texts, img, "right", 16, text_embeds=te, **{k: v for k, v in kw.items() if k not in ("direction", "amount")})
    assert all(torch.equal(x, y) for x, y in zip(got, (full_img, full_ids)))
    e_img, e_ids = parallel._empty_result(mg, True, image_hw=tuple(full_img.shape[2:]))
    assert e_img.shape == (0, 3, 16, 36) and e_ids.shape == (0, 4, 9) and e_ids.dtype == torch.int64
    assert parallel._empty_result(mg, True)[1].shape == (0, 4, 4)


def test_fused_tail_overflow_reruns_as_extrapolate():
    """Constant logits (zero to_logits, V = 65536): step 0 of each window samples 16 images x 16 rows, more than the fused tail's fallback
    holds; the materialised rerun is an extrapolation equal to asking for the materialised tail directly, with the input tokens kept."""
    from tests.test_gpu_fused_tail import _degenerate_maskgit
    mg, b = _degenerate_maskgit()
    mg.sampler_seed = 42
    img = _images(b)
    known = mg.vae.encode_ids(img)
    mg.use_fused_tail, mg.last_fused_fallback_rows = True, 0
    img_f, ids_f = mg.extrapolate(["a"] * b, img, direction="left", amount=32, stride=F, timesteps=3, return_ids=True)
    assert mg.last_fused_fallback_rows > 128
    mg.use_fused_tail = False
    img_m, ids_m = mg.extrapolate(["a"] * b, img, direction="left", amount=32, stride=F, timesteps=3, return_ids=True)
    assert ids_f.shape == (b, F, 3 * F) and img_f.shape == (b, 3, 16, 48)
    assert torch.equal(ids_f, ids_m) and torch.equal(img_f, img_m)
    assert torch.equal(ids_f[:, :, 2 * F:], known)


# ------------------------------------------------------------------------------------------------ arguments
def test_argument_errors_launch_nothing():
    from muse_maskgit_pytorch_b200 import _lib
    mg = _setup(make_maskgit("bf16"), _te())
    img = _images(3)
    calls = [(img, dict(direction="diagonal")), (img, dict(amount=0)), (img, dict(amount=12)), (img, dict(amount=8, stride=0)),
             (img, dict(amount=8, stride=5)), (img, dict(amount=8.5)), (img, dict(amount=8, timesteps=0)), (img[:2], dict(amount=8)),
             (_images(3, 16, 18), dict(amount=8)), (_images(3, 20, 16), dict(amount=8)), (_images(3, 16, 20), dict(direction="down", amount=8))]
    torch.cuda.synchronize()
    l0 = _lib.launch_count()
    for images, kw in calls:
        with pytest.raises(ValueError):
            mg.extrapolate(["a"] * 3, images, **kw)
    mg.sampler_rng = "aten"
    with pytest.raises(ValueError, match="aten"):
        mg.extrapolate(["a"] * 3, img, amount=8)
    with pytest.raises(ValueError, match="aten"):
        parallel.extrapolate_sharded(mg, ["a"] * 3, img, amount=8)
    mg.sampler_rng = "mmg"
    sup = make_maskgit("bf16", superres=True)
    with pytest.raises(ValueError, match="cond_image_size"):
        sup.extrapolate(["a"] * 2, _images(2, 32, 32), amount=16)
    vae8 = M().VQGanVAE(dim=128, layers=2, codebook_size=1024, precision="fp8")
    mg8 = M().MaskGit(image_size=16, transformer=small_transformer("bf16"), vae=vae8).cuda()
    with pytest.raises(ValueError, match="tile geometry"):
        mg8.extrapolate(["a"] * 3, img, amount=8)               # 16 x 24 pixels: the 8 x 12 map has no e4m3 conv tile
    assert _lib.launch_count() == l0

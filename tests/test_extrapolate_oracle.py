"""CPU: the image extrapolation oracle (tests/extrapolate_oracle.py) against its own definition and against inpaint_ids, and MaskGit's window
plan and argument checks (host-only, before any launch) against the oracle's."""
import pytest
import torch

from tests import extrapolate_oracle as XO, inpaint_oracle as IO, util

torch.set_grad_enabled(False)
CFG = dict(heads=2, depth=2)
V, F = 1024, 4


def _setup(seed=1, in_w=F, in_h=F):
    known = torch.randint(0, V, (3, in_h, in_w), generator=torch.Generator().manual_seed(seed))
    return util.transformer_sd(V, 128, F * F, 2, 2, seed=13, text_dim=128), util.text_embeds("g4.te", 3, 8, 128, 14), known


@pytest.mark.parametrize("direction", XO.DIRECTIONS)
@pytest.mark.parametrize("stride,K,extra", [(1, 3, 0), (2, 3, 2), (4, 1, 0), (3, 2, 1), (2, 1, 0)])
def test_windows_cover_every_new_token_once_and_no_input_token(direction, stride, K, extra):
    vertical = direction in ("down", "up")
    in_h, in_w = (F + extra, F) if vertical else (F, F + extra)
    (H, W), (r, c), corners = XO.plan(direction, in_h, in_w, F, stride, K)
    assert (H, W) == ((in_h + K * stride, F) if vertical else (F, in_w + K * stride))
    assert len(corners) == K
    cover = torch.zeros((H, W), dtype=torch.int32)
    s = XO.strip(direction, F, stride)
    assert int(s.sum()) == F * stride
    for w, (r0, c0) in enumerate(corners):
        assert 0 <= r0 and r0 + F <= H and 0 <= c0 and c0 + F <= W
        cover[r0:r0 + F, c0:c0 + F] += s.int()
        far = {"right": c0 + F, "left": c0, "down": r0 + F, "up": r0}[direction]
        edge = {"right": in_w, "left": K * stride, "down": in_h, "up": K * stride}[direction]
        assert abs(far - edge) == stride * (w + 1)          # the far edge lies stride * (w + 1) tokens past the input's edge
    is_input = torch.zeros((H, W), dtype=torch.bool)
    is_input[r:r + in_h, c:c + in_w] = True
    assert (cover[is_input] == 0).all() and (cover[~is_input] == 1).all()


@pytest.mark.parametrize("direction", XO.DIRECTIONS)
def test_input_tokens_kept_and_changes_stay_in_each_strip(direction):
    sd, te, known = _setup(2)
    trace = []
    got = XO.extrapolate_ids(sd, CFG, te, known, direction, 3, 1, V, util.torch_noise_fn(5), timesteps=3, trace=trace)
    (H, W), (r, c), corners = XO.plan(direction, F, F, F, 1, 3)
    assert got.shape == (3, H, W)
    assert torch.equal(got[:, r:r + F, c:c + F], known)
    assert int(got.max()) < V and int(got.min()) >= 0
    s = XO.strip(direction, F, 1).reshape(-1)
    for t in trace:
        assert (t["known"][:, s] == V).all()                # the strip starts masked, the context is the canvas
        assert not ((t["ids"] != t["known"]) & ~s).any()


@pytest.mark.parametrize("critic", [False, True])
def test_one_full_window_equals_inpaint_of_every_token(critic):
    sd, te, known = _setup(3)
    kw = dict(critic=dict(kind="token", sd=util.critic_sd(V, 128, F * F, 1, 2, seed=22, text_dim=128), cfg=dict(heads=2, depth=1)),
              critic_noise_scale=0.7) if critic else {}
    got = XO.extrapolate_ids(sd, CFG, te, known, "right", 1, F, V, util.torch_noise_fn(9), timesteps=5, **kw)
    want = IO.inpaint_ids(sd, CFG, te, known.reshape(3, -1), torch.ones((3, F * F), dtype=torch.bool), V, util.torch_noise_fn(9), timesteps=5,
                          **kw)
    assert torch.equal(got[:, :, :F], known)
    assert torch.equal(got[:, :, F:].reshape(3, -1), want)


# ------------------------------------------------------------------------------------------------ MaskGit's host-side plan
def _maskgit():
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    tr = M.MaskGitTransformer(num_tokens=V, dim=128, seq_len=F * F, depth=1, heads=2, t5_name="synth-128")
    vae = M.VQGanVAE(dim=16, layers=2, codebook_size=V)
    return M.MaskGit(image_size=16, transformer=tr, vae=vae)


@pytest.mark.parametrize("direction", XO.DIRECTIONS)
@pytest.mark.parametrize("stride,K,extra", [(1, 3, 0), (2, 3, 2), (4, 1, 0)])
def test_maskgit_window_plan_equals_the_oracle(direction, stride, K, extra):
    mg = _maskgit()
    vertical = direction in ("down", "up")
    in_h, in_w = (F + extra, F) if vertical else (F, F + extra)
    images = torch.zeros((2, 3, 4 * in_h, 4 * in_w))
    w = mg._extrapolate_plan(images, 2, direction, K * stride * 4, stride)
    canvas, at, corners = XO.plan(direction, in_h, in_w, F, stride, K)
    assert (w.canvas, w.input_at, list(w.corners), w.stride) == (canvas, at, corners, stride)
    assert torch.equal(mg._window_strip(direction, F, stride), XO.strip(direction, F, stride))
    assert w.key == ("extrapolate", direction, K, stride, canvas)


def test_maskgit_argument_errors_on_the_host():
    mg = _maskgit()
    img = torch.zeros((2, 3, 16, 16))
    bad = [dict(direction="sideways"), dict(amount=0), dict(amount=-8), dict(amount=12), dict(amount=8.0), dict(stride=0), dict(stride=5),
           dict(stride=3, amount=16), dict(timesteps=0)]
    for kw in bad:
        with pytest.raises(ValueError):
            mg.extrapolate(["a"] * 2, img, **dict(dict(amount=8), **kw))
    for shape in ((2, 3, 16, 18), (2, 3, 12, 16), (3, 3, 16, 16), (2, 1, 16, 16), (2, 3, 16)):
        with pytest.raises(ValueError, match="images"):
            mg.extrapolate(["a"] * 2, torch.zeros(shape), amount=8)
    with pytest.raises(ValueError, match="images"):
        mg.extrapolate(["a"] * 2, torch.zeros((2, 3, 20, 16)), amount=8)          # "right" needs H = image_size
    with pytest.raises(ValueError, match="images"):
        mg.extrapolate(["a"] * 2, torch.zeros((2, 3, 16, 20)), direction="up", amount=8)
    mg.sampler_rng = "aten"
    with pytest.raises(ValueError, match="aten"):
        mg.extrapolate(["a"] * 2, img, amount=8)

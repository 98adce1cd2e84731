"""CPU: the inpainting oracle (tests/inpaint_oracle.py) against generate_ids and its own definition, and the pixel -> token mask pooling of
MaskGit.inpaint."""
import math

import pytest
import torch

from oracle import muse_oracle as O
from tests import inpaint_oracle as IO, util

torch.set_grad_enabled(False)
CFG = dict(heads=2, depth=2)
V, N = 1024, 16


def _setup():
    return util.transformer_sd(V, 128, N, 2, 2, seed=13, text_dim=128), util.text_embeds("g4.te", 3, 8, 128, 14)


def _critic(kind):
    if kind == "token":
        return dict(kind="token", sd=util.critic_sd(V, 128, N, 1, 2, seed=22, text_dim=128), cfg=dict(heads=2, depth=1))
    return None


@pytest.mark.parametrize("critic,remask_prev", [(None, False), ("token", False), (None, True)])
def test_full_mask_equals_generate_ids(critic, remask_prev):
    sd, te = _setup()
    known = torch.randint(0, V, (3, N), generator=torch.Generator().manual_seed(1))
    kw = dict(timesteps=6, critic=_critic(critic), critic_noise_scale=0.7, can_remask_prev_masked=remask_prev)
    want = O.generate_ids(sd, CFG, te, N, V, util.torch_noise_fn(777), **kw)
    got = IO.inpaint_ids(sd, CFG, te, known, torch.ones((3, N), dtype=torch.bool), V, util.torch_noise_fn(777), **kw)
    assert torch.equal(got, want)


def test_empty_mask_returns_known_ids():
    sd, te = _setup()
    known = torch.randint(0, V, (3, N), generator=torch.Generator().manual_seed(2))
    trace = []
    got = IO.inpaint_ids(sd, CFG, te, known, torch.zeros((3, N), dtype=torch.bool), V, util.torch_noise_fn(5), timesteps=4, trace=trace)
    assert torch.equal(got, known)
    assert all(st["num_masked"] == [0, 0, 0] for st in trace)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_ragged_masks_keep_frozen_ids_and_follow_the_schedule(seed):
    sd, te = _setup()
    g = torch.Generator().manual_seed(seed)
    known = torch.randint(0, V, (3, N), generator=g)
    regen = torch.rand((3, N), generator=g) < torch.tensor([[0.2], [0.6], [0.9]])
    if seed == 0:
        regen[0] = False                                        # one image with nothing to regenerate
    T = 7
    trace = []
    got = IO.inpaint_ids(sd, CFG, te, known, regen, V, util.torch_noise_fn(100 + seed), timesteps=T, trace=trace)
    assert torch.equal(got[~regen], known[~regen])
    assert (got[regen] != V).all() and int(got.max()) < V
    for step, st in enumerate(trace):
        t = torch.linspace(0, 1, T)[step]
        for i in range(3):
            nb = int(regen[i].sum())
            want = max(int((torch.cos(t * math.pi * 0.5) * nb).item()), 1) if nb else 0
            masked = st["ids_in"][i] == V
            assert int(masked.sum()) == want == st["num_masked"][i], (step, i)
            assert not (masked & ~regen[i]).any()
            assert torch.equal(st["ids_out"][i][~regen[i]], known[i][~regen[i]])
            assert not (st["ids_out"][i] == V).any()                # every position is decoded after each step


def test_mask_pooling_at_patch_edges():
    from muse_maskgit_pytorch_b200.muse_maskgit import regen_tokens
    size, f = 16, 4                                             # 4 x 4 pixel patches
    for r, c in [(0, 0), (3, 3), (3, 4), (4, 3), (4, 4), (7, 8), (12, 15), (15, 15), (15, 0)]:
        m = torch.zeros((2, size, size), dtype=torch.bool)
        m[1, r, c] = True
        want = torch.zeros((2, f, f), dtype=torch.bool)
        want[1, r // 4, c // 4] = True
        assert torch.equal(regen_tokens(m, 2, size, f), want), (r, c)
        assert torch.equal(regen_tokens(m[:, None].long(), 2, size, f), want), (r, c)        # (b, 1, H, W) and {0, 1} integers
    # a masked band ending exactly at a patch edge does not spill into the next token
    m = torch.zeros((1, size, size), dtype=torch.uint8)
    m[0, :, :8] = 1
    assert torch.equal(regen_tokens(m, 1, size, f)[0], torch.tensor([[True, True, False, False]] * 4))
    tok = torch.rand((2, f, f), generator=torch.Generator().manual_seed(3)) < 0.5
    assert torch.equal(regen_tokens(tok, 2, size, f), tok)                                   # token resolution passes through
    with pytest.raises(ValueError):
        regen_tokens(torch.zeros((2, 8, 8), dtype=torch.bool), 2, size, f)
    with pytest.raises(ValueError):
        regen_tokens(torch.zeros((3, size, size), dtype=torch.bool), 2, size, f)
    with pytest.raises(ValueError):
        regen_tokens(torch.full((2, size, size), 2), 2, size, f)
    with pytest.raises(ValueError):
        regen_tokens(torch.zeros((2, 2, size, size), dtype=torch.bool), 2, size, f)

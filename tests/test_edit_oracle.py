"""CPU: the mask-free editing oracle (tests/edit_oracle.py) against its own definition and against inpaint_ids, and its Philox keys against
oracle/philox.py."""
import pytest
import torch

from oracle import philox
from tests import edit_oracle as EO, inpaint_oracle as IO, util

torch.set_grad_enabled(False)
CFG = dict(heads=2, depth=2)
V, N = 1024, 16


def _setup(seed=1):
    known = torch.randint(0, V, (3, N), generator=torch.Generator().manual_seed(seed))
    return util.transformer_sd(V, 128, N, 2, 2, seed=13, text_dim=128), util.text_embeds("g4.te", 3, 8, 128, 14), known


def _ragged(seed):
    g = torch.Generator().manual_seed(seed)
    e = torch.rand((3, N), generator=g) < torch.tensor([[0.3], [0.7], [1.0]])
    if seed % 2:
        e[0] = False                                            # one image with nothing to edit
    return e


def test_zero_iterations_return_ids0():
    sd, te, known = _setup()
    assert torch.equal(EO.edit_ids(sd, CFG, te, known, torch.ones((3, N), dtype=torch.bool), V, util.torch_noise_fn(3), iterations=0), known)


@pytest.mark.parametrize("seed", [1, 2])
def test_tokens_outside_mask_never_change_and_changes_stay_in_the_selection(seed):
    sd, te, known = _setup(seed)
    editable = _ragged(seed)
    trace = []
    got = EO.edit_ids(sd, CFG, te, known, editable, V, util.torch_noise_fn(40 + seed), iterations=3, fraction=0.4, timesteps=3, trace=trace)
    assert torch.equal(got[~editable], known[~editable])
    assert int(got.max()) < V
    counts = EO.select_counts(editable, 0.4)
    prev = known
    for it in trace:
        sel = it["selected"]
        assert [int(c) for c in sel.sum(dim=1)] == counts
        assert not (sel & ~editable).any()
        assert not ((it["ids"] != prev) & ~sel).any()         # changed tokens are a subset of the iteration's selection
        prev = it["ids"]
    assert not torch.equal(got, known)


def _skip_keys(fn, b):
    """fn after one (b, N) draw: the gumbel / critic draws that follow the keys of an edit iteration."""
    fn(0, (b, N))
    return fn


@pytest.mark.parametrize("critic", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_one_full_fraction_iteration_equals_inpaint(critic, masked):
    sd, te, known = _setup(3)
    editable = _ragged(3) if masked else torch.ones((3, N), dtype=torch.bool)
    kw = dict(critic=dict(kind="token", sd=util.critic_sd(V, 128, N, 1, 2, seed=22, text_dim=128), cfg=dict(heads=2, depth=1)),
              critic_noise_scale=0.7) if critic else {}
    got = EO.edit_ids(sd, CFG, te, known, editable, V, util.torch_noise_fn(9), iterations=1, fraction=1.0, timesteps=5, **kw)
    want = IO.inpaint_ids(sd, CFG, te, known, editable, V, _skip_keys(util.torch_noise_fn(9), 3), timesteps=5, **kw)
    assert torch.equal(got, want)


def test_selection_ties_go_to_the_lowest_position():
    keys = torch.tensor([[0.5, 0.9, 0.5, 0.9, 0.1, 0.5], [0.2, 0.2, 0.2, 0.2, 0.2, 0.2]])
    editable = torch.tensor([[True, False, True, True, True, True], [True] * 6])
    sel = EO.select(keys, editable, [3, 2])
    assert sel[0].nonzero().flatten().tolist() == [0, 2, 3]
    assert sel[1].nonzero().flatten().tolist() == [0, 1]
    assert EO.select_counts(editable, 0.1) == [1, 1] and EO.select_counts(torch.zeros((1, 6), dtype=torch.bool), 0.5) == [0]
    assert EO.select_counts(torch.ones((1, 256), dtype=torch.bool), 0.1) == [25]


def test_philox_keys_match_the_scalar_restatement():
    seed = (7 << 40) | 12345
    keys = EO.philox_keys(seed, 5, 2, 16, row_offset=3)
    for b in range(2):
        for p in (0, 7, 15):
            assert keys[b, p].item() == float(philox.uniform_at(seed, 5, (3 + b) * 16 + p, EO.KEY_C0))
    assert not torch.equal(keys, EO.philox_keys(seed, 6, 2, 16, row_offset=3))

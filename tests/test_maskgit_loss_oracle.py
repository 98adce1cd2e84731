"""CPU: the restatement of MaskGit.forward in tests/loss_oracle.py reproduces the unmodified reference's loss on every case of
tests/golden/loss_small.npz under the same seeds.  This pins the draw order, the label / critic-label rules and the conditioning-drop
handling that MaskGit.forward follows to the reference itself."""
import pytest
import torch

from tests import loss_oracle as LO

CASES = LO.golden_cases()


def test_golden_covers_every_branch():
    assert set(CASES) == {"plain", "drop0", "drop1", "no_mask_token", "ids", "selfcond", "token_critic", "token_critic_temp", "self_critic",
                          "superres"}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_reference_loss(name):
    c = CASES[name]
    torch.manual_seed(c["seed"])
    py = iter(c["py_draws"])
    with torch.no_grad():
        loss = LO.golden_case_loss(c, lambda shape: torch.zeros(shape).uniform_(0, 1), lambda: next(py))
    assert next(py, None) is None, "the oracle made fewer python random() draws than the reference"
    assert abs(float(loss) - c["loss"]) <= 1e-6, (name, float(loss), c["loss"])

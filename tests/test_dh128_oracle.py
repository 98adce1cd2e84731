"""CPU: 128-wide attention heads.  The oracle restatement (oracle/muse_oracle.py, which reads the head width from the weights) reproduces
tests/golden/gen_small_dh128.npz, made by the unmodified reference at dim_head = 128 (tests/golden/make_dh128_golden.py); the parameter
holders of MaskGitTransformer(dim_head=128) have the reference's keys and shapes; head sizes other than 64 and 128 are refused."""
import pytest
import torch

from oracle import muse_oracle as O, shapes, synth
from tests import util

DIM, HEADS, DH, DEPTH = 256, 2, 128, 2
CFG = dict(heads=HEADS, depth=DEPTH)


def dh128_sd(seq_len, seed):
    return util.sd_from_table(shapes.transformer_shapes(1024, DIM, seq_len, DEPTH, heads=HEADS, dim_head=DH, text_dim=128), seed)


def test_forward_matches_reference():
    g = util.golden("gen_small_dh128")
    te = util.text_embeds("g4.te", 3, 8, 128, 14)
    cfg_logits, embed = O.forward_with_cond_scale(dh128_sd(16, 41), CFG, g["ids"], te, cond_scale=3.)
    assert torch.allclose(embed, g["embed"], atol=2e-5, rtol=1e-4)
    assert torch.allclose(cfg_logits, g["logits_cfg"], atol=1e-4, rtol=1e-4)


def test_generate_matches_reference():
    g = util.golden("gen_small_dh128")
    torch.manual_seed(790)
    if not torch.equal(torch.zeros(7).uniform_(0, 1), g["u_probe"]):
        pytest.skip("torch CPU generator differs from the one that made the fixture")
    vsd = util.vae_sd(16, 2, 1024, seed=12)
    te = util.text_embeds("g4.te", 3, 8, 128, 14)
    images, ids = O.generate(dh128_sd(16, 41), CFG, vsd, 10, te, 4, util.torch_noise_fn(790), timesteps=6)
    assert torch.equal(ids.view(3, 4, 4), g["gen_ids"])
    assert torch.allclose(images, g["images"], atol=1e-5)


def test_superres_generate_matches_reference():
    g = util.golden("gen_small_dh128")
    vsd = util.vae_sd(16, 2, 1024, seed=12)
    te = util.text_embeds("g4.te", 3, 8, 128, 14)[:2]
    cond = torch.from_numpy(synth.uniform("g5.cond", (2, 3, 16, 16), 15))
    images, ids = O.generate(dh128_sd(64, 42), CFG, vsd, 10, te, 8, util.torch_noise_fn(791), cond_images=cond, timesteps=8)
    assert torch.equal(ids.view(2, 8, 8), g["sr_ids"])
    assert torch.allclose(images, g["sr_images"], atol=1e-5)


def test_state_dict_keys_match_reference_tables():
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    tr = M.MaskGitTransformer(num_tokens=1024, dim=DIM, seq_len=16, depth=DEPTH, heads=HEADS, dim_head=DH, t5_name="synth-128")
    got = {k: tuple(v.shape) for k, v in tr.state_dict().items()}
    assert got == {k: tuple(v) for k, v in shapes.transformer_shapes(1024, DIM, 16, DEPTH, heads=HEADS, dim_head=DH, text_dim=128).items()}


@pytest.mark.parametrize("dim,dim_head", [(256, 32), (256, 96), (256, 256), (192 + 32, 128)])
def test_unsupported_head_sizes_raise(dim, dim_head):
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    with pytest.raises(ValueError, match="64"):
        M.MaskGitTransformer(num_tokens=1024, dim=dim, seq_len=16, depth=1, heads=2, dim_head=dim_head, t5_name="synth-128")

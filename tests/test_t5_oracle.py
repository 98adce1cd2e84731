"""CPU: the fp64 T5 encoder oracle against HF's T5EncoderModel, the host bucket map, T5Encoder's checkpoint keys and config checks, and the
derivation of the bf16 error bound the GPU tests use."""
import pytest
import torch

from oracle import t5_encoder as O
from tests import t5_common as C


def _hf(c, sd, dtype=torch.float32):
    transformers = pytest.importorskip("transformers")
    m = transformers.T5EncoderModel(C.hf_config(c)).eval()
    m.load_state_dict(sd, strict=True)
    return m.to(dtype)


def _hf_out(m, ids, mask):
    with torch.no_grad():
        out = m(input_ids=ids, attention_mask=mask).last_hidden_state
    return out.masked_fill(~mask.bool()[..., None], 0)


@pytest.mark.parametrize("c", [C.SMALL_RELU, C.SMALL_GATED], ids=["relu", "gated-gelu"])
@pytest.mark.parametrize("T", [1, 7, 77])
def test_oracle_equals_hf_fp64(c, T):
    sd = C.random_sd(c, 10 + T)
    ids, mask = C.random_batch(4, T, c["vocab_size"], T, pad=True)
    got = O.encode(sd, vars(C.config(c)), ids, mask)
    ref = _hf_out(_hf(c, sd, torch.float64), ids, mask)
    assert got.dtype == torch.float64
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("nb,maxd", [(32, 128), (16, 64)])
def test_host_bucket_map_matches_hf(nb, maxd):
    transformers = pytest.importorskip("transformers")
    from muse_maskgit_pytorch_b200.t5 import relative_position_bucket
    rel = torch.arange(-511, 512)
    ref = transformers.models.t5.modeling_t5.T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=nb, max_distance=maxd)
    assert torch.equal(relative_position_bucket(rel, nb, maxd), ref)
    assert torch.equal(O.relative_position_bucket(rel, True, nb, maxd), ref)


@pytest.mark.parametrize("c", [C.SMALL_RELU, C.SMALL_GATED], ids=["relu", "gated-gelu"])
def test_state_dict_keys_match_hf(c):
    from muse_maskgit_pytorch_b200 import T5Encoder
    hf = _hf(c, C.random_sd(c, 3))
    enc = T5Encoder(hf.config)
    assert {k: tuple(v.shape) for k, v in enc.state_dict().items()} == {k: tuple(v.shape) for k, v in hf.state_dict().items()}
    enc.load_state_dict(hf.state_dict(), strict=True)
    assert enc.shared.weight is enc.encoder.embed_tokens.weight
    assert torch.equal(enc.shared.weight, hf.shared.weight)
    enc2 = T5Encoder.from_hf(hf, precision="fp32")
    assert enc2.precision == "fp32" and all(torch.equal(a, b) for a, b in zip(enc2.state_dict().values(), hf.state_dict().values()))


def test_unsupported_configs_raise():
    from muse_maskgit_pytorch_b200 import T5Encoder
    from muse_maskgit_pytorch_b200._lib import MMGError
    for field, value in (("d_kv", 128), ("d_ff", 1000), ("d_model", 100), ("feed_forward_proj", "gated-silu")):
        c = dict(C.SMALL_RELU, **{field: value})
        with pytest.raises(MMGError, match=field):
            T5Encoder(C.config(c))
    with pytest.raises(MMGError, match="precision"):
        T5Encoder(C.config(C.SMALL_RELU), precision="fp16")


def test_bf16_bound_is_pinned_to_hf_bf16_error():
    """BF16_REL_L2_BOUND (the GPU tests' tolerance for the bf16 T5Encoder) is at most 1.5x the relative L2 error HF's own bf16 model makes
    against fp64 at the pinned configuration, so the tolerance is HF's bf16 error and not a free number."""
    c, B, T = C.PIN_CFG, C.PIN_B, C.PIN_T
    sd = C.random_sd(c, 7)
    ids, mask = C.random_batch(B, T, c["vocab_size"], 8)
    ref = O.encode(sd, vars(C.config(c)), ids, mask)
    bf = _hf_out(_hf(c, sd, torch.bfloat16), ids, mask).double()
    live = mask.bool()
    hf_err = C.rel_l2(bf[live], ref[live])
    assert C.BF16_REL_L2_BOUND <= 1.5 * hf_err, (C.BF16_REL_L2_BOUND, hf_err)


def test_fp32_constant_covers_hf_fp32_error():
    """HF_FP32_MAX_ABS (the stand-in for HF's fp32 error when transformers is missing on the GPU machine) is HF's fp32 max-abs error at the
    largest GPU test configuration, within 25 %."""
    c = C.V11_BASE
    sd = C.random_sd(c, 5)
    ids, mask = C.random_batch(64, 32, c["vocab_size"], 6)
    ref = O.encode(sd, vars(C.config(c)), ids, mask)
    err = float((_hf_out(_hf(c, sd), ids, mask).double() - ref)[mask.bool()].abs().max())
    assert 0.75 * C.HF_FP32_MAX_ABS <= err <= 1.25 * C.HF_FP32_MAX_ABS, err

"""GPU: libmmg's T5 encoder.  mmg_t5_attention and mmg_rmsnorm against fp64, the GEGLU_TANH / ReLU GEMM epilogues against fp64, the whole
T5Encoder against the fp64 oracle (oracle/t5_encoder.py) in both precisions, t5_encode_text's "native" switch through generate(), and CUDA
graph capture of T5Encoder.forward."""
import pytest
import torch

from muse_maskgit_pytorch_b200 import ops, _lib
from muse_maskgit_pytorch_b200.t5 import relative_position_bucket
from oracle import t5_encoder as O
from tests import t5_common as C

pytestmark = pytest.mark.gpu
F32_MIN = torch.finfo(torch.float32).min


def _attn_ref(qkv, B, T, heads, bucket, rel_bias, mask):
    """fp64 softmax(q k^T + bias + mask) v, a masked key scoring finfo(fp32).min (an all-masked row averages v over the T keys)."""
    x = qkv.double().view(B, T, 3, heads, 64).permute(2, 0, 3, 1, 4)        # [3, B, H, T, 64]
    q, k, v = x[0], x[1], x[2]
    idx = torch.arange(T, device=qkv.device)
    bias = rel_bias.double()[bucket.long()[idx[None, :] - idx[:, None] + T - 1]].permute(2, 0, 1)   # [H, T(q), T(k)]
    s = q @ k.transpose(-1, -2) + bias[None]
    s = torch.where(mask.bool()[:, None, None, :], s, torch.full_like(s, F32_MIN))
    return (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * T, heads * 64)


def _ragged_mask(B, T, g):
    """row 0 full, row 1 random length, row 2 a single live key (in the middle), row 3 no live key, further rows random holes"""
    m = torch.rand((B, T), generator=g) < 0.7
    m[0] = True
    m[1] = torch.arange(T) < torch.randint(1, T + 1, (1,), generator=g)
    m[2] = False; m[2, T // 2] = True
    m[3] = False
    return m.to(torch.uint8)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("heads", [6, 12])
@pytest.mark.parametrize("T", [1, 7, 64, 77, 128, 129, 256, 512])
def test_t5_attention_vs_fp64(T, heads, dtype):
    g = torch.Generator().manual_seed(T * 100 + heads)
    B, inner = 5, heads * 64
    qkv = (0.4 * torch.randn((B * T, 3 * inner), generator=g)).to("cuda", dtype)
    rel_bias = (2.0 * torch.randn((32, heads), generator=g)).cuda()
    bucket = relative_position_bucket(torch.arange(-(T - 1), T), 32, 128).to(torch.int32).cuda()
    mask = _ragged_mask(B, T, g).cuda()
    out = torch.full((B * T, inner), float("nan"), device="cuda", dtype=dtype)
    s0, f0 = _lib.simt_launch_count(), _lib.simt_fallback_count()
    ops.t5_attention(qkv, out, B, T, heads, bucket, rel_bias, mask)
    torch.cuda.synchronize()
    if dtype == torch.bfloat16:
        assert (_lib.simt_launch_count(), _lib.simt_fallback_count()) == (s0, f0), "the bf16 leg must run on the wgmma kernel"
    ref = _attn_ref(qkv, B, T, heads, bucket, rel_bias, mask)
    err = float((out.double() - ref).abs().max())
    tol = 1.6e-2 if dtype == torch.bfloat16 else 2e-5
    assert err <= tol, (T, heads, dtype, err)
    # the row without a live key is the mean of v over the T keys
    v3 = qkv[3 * T:4 * T, 2 * inner:].double().mean(0)
    assert float((out[3 * T:4 * T].double() - v3).abs().max()) <= tol


@pytest.mark.parametrize("ydt", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("rows,d", [(1, 512), (77, 768), (333, 2048), (64, 4096)])
def test_rmsnorm_row_mask_vs_fp64(rows, d, ydt):
    g = torch.Generator().manual_seed(rows + d)
    x = (3.0 * torch.randn((rows, d), generator=g)).cuda()
    w = (1.0 + 0.2 * torch.randn(d, generator=g)).cuda()
    rm = (torch.rand(rows, generator=g) < 0.7).to(torch.uint8).cuda()
    y = torch.full((rows, d), float("nan"), device="cuda", dtype=ydt)
    ops.rmsnorm(x, w, y, 1e-6, row_mask=rm)
    xd = x.double()
    ref = w.double() * (xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6))
    ref = ref.masked_fill(~rm.bool()[:, None], 0.0)
    assert torch.equal(y[~rm.bool()], torch.zeros_like(y[~rm.bool()]))
    rel = 2 ** -8 if ydt == torch.bfloat16 else 2e-6
    assert float(((y.double() - ref).abs() - rel * ref.abs()).max()) <= 1e-6


def _gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh((2.0 / torch.pi) ** 0.5 * (x + 0.044715 * x ** 3)))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", ["geglu_tanh", "relu"])
@pytest.mark.parametrize("d_ff", [1024, 2048, 2816, 5120])
def test_t5_ff_epilogues_vs_fp64(d_ff, kind, prec):
    g = torch.Generator().manual_seed(d_ff + len(kind))
    K = 256
    for M in (77, 333):
        a = torch.randn((M, K), generator=g)
        w0, w1 = torch.randn((d_ff, K), generator=g) * K ** -0.5, torch.randn((d_ff, K), generator=g) * K ** -0.5
        dt = torch.bfloat16 if prec == "bf16" else torch.float32
        a_d, w0_d, w1_d = a.to(dt).double(), w0.to(dt).double(), w1.to(dt).double()
        if kind == "geglu_tanh":
            w = torch.stack((w0.reshape(-1, 32, K), w1.reshape(-1, 32, K)), 1).reshape(-1, K)
            ref = _gelu_new(a_d @ w0_d.t()) * (a_d @ w1_d.t())
        else:
            w = w0
            ref = torch.relu(a_d @ w0_d.t())
        out = torch.full((M, d_ff), float("nan"), device="cuda", dtype=dt)
        s0, f0 = _lib.simt_launch_count(), _lib.simt_fallback_count()
        if kind == "geglu_tanh":
            ops.linear(a.to("cuda", dt), w.to("cuda", dt).contiguous(), out, ops.EPI_GEGLU_TANH)
        else:
            ops.linear(a.to("cuda", dt), w.to("cuda", dt).contiguous(), out, ops.EPI_STORE, act=2)
        torch.cuda.synchronize()
        assert (_lib.simt_launch_count(), _lib.simt_fallback_count()) == (s0, f0), "both legs run on the wgmma kernel"
        err = (out.double().cpu() - ref).abs()
        if prec == "bf16":
            assert float((err - 2 ** -8 * ref.abs()).max()) <= 2e-3, (M, float(err.max()))
        else:
            assert float((err - 1e-5 * ref.abs()).max()) <= 1e-5, (M, float(err.max()))


# ------------------------------------------------------------------------------------------------ whole encoder
def _encoder(c, seed, precision):
    from muse_maskgit_pytorch_b200 import T5Encoder
    sd = C.random_sd(c, seed)
    enc = T5Encoder(C.config(c), precision=precision, init_weights=False)
    enc.load_state_dict(sd, strict=True)
    return enc.cuda(), sd


def _hf_fp32_error(c, sd, ids, mask, ref):
    try:
        import transformers
    except ImportError:
        return C.HF_FP32_MAX_ABS
    m = transformers.T5EncoderModel(C.hf_config(c)).eval()
    m.load_state_dict(sd, strict=True)
    with torch.no_grad():
        out = m(input_ids=ids, attention_mask=mask).last_hidden_state.double()
    return float((out - ref)[mask.bool()].abs().max())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("c,B,T", [(C.SMALL_RELU, 5, 77), (C.SMALL_GATED, 5, 77), (C.V11_BASE, 64, 32)], ids=["relu", "gated", "v1_1-base"])
def test_encoder_vs_oracle(c, B, T, precision):
    enc, sd = _encoder(c, 31 + T, precision)
    ids, mask = C.random_batch(B, T, c["vocab_size"], 32 + B)
    ref = O.encode(sd, vars(C.config(c)), ids, mask)
    s0, f0 = _lib.simt_launch_count(), _lib.simt_fallback_count()
    out = enc(ids.cuda(), mask.cuda())
    torch.cuda.synchronize()
    assert out.shape == (B, T, c["d_model"]) and out.dtype == torch.float32
    assert _lib.simt_fallback_count() == f0
    if precision == "bf16":
        assert _lib.simt_launch_count() == s0
    live = mask.bool()
    out = out.double().cpu()
    assert torch.equal(out[~live], torch.zeros_like(out[~live])), "padding rows must be exactly 0"
    if precision == "fp32":
        err, hf = float((out - ref)[live].abs().max()), _hf_fp32_error(c, sd, ids, mask, ref)
        print(f"T5Encoder fp32 max-abs {err:.3e} vs HF fp32 {hf:.3e}")
        assert err <= 4 * hf, (err, hf)
    else:
        err = C.rel_l2(out[live], ref[live])
        print(f"T5Encoder bf16 rel-L2 {err:.3e} (bound {C.BF16_REL_L2_BOUND:.1e})")
        assert err <= C.BF16_REL_L2_BOUND, err


# ------------------------------------------------------------------------------------------------ wiring
class _Tok:
    """stand-in tokenizer: fixed ids / mask, whatever the texts"""
    def __init__(self, ids, mask):
        self.ids, self.mask = ids, mask

    def batch_encode_plus(self, texts, **kw):
        import types
        assert len(texts) == self.ids.shape[0]
        return types.SimpleNamespace(input_ids=self.ids, attention_mask=self.mask)


class _NoHF:
    def __getattr__(self, name):
        raise AssertionError(f"the HF model was used ({name})")

    def __call__(self, *a, **k):
        raise AssertionError("the HF model was called")


def test_generate_with_native_text_encoder(monkeypatch):
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    from tests import util
    try:
        import transformers
        monkeypatch.setattr(transformers.T5EncoderModel, "from_pretrained", classmethod(lambda *a, **k: _NoHF()()))
    except ImportError:
        pass
    c = C.SMALL_RELU
    enc, _ = _encoder(c, 5, "bf16")
    ids, mask = C.random_batch(3, 9, c["vocab_size"], 6)
    name = "native-t5-test"
    monkeypatch.setitem(t5.T5_CONFIGS, name, {"native": enc, "tokenizer": _Tok(ids, mask), "model": _NoHF()})
    tr = M.MaskGitTransformer(num_tokens=1024, dim=128, seq_len=16, depth=2, heads=2, t5_name=name, precision="bf16")
    sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
    full = tr.state_dict(); full.update(sd); tr.load_state_dict(full)
    vae = M.VQGanVAE(dim=16, layers=2, codebook_size=1024, precision="bf16")
    vsd = util.vae_sd(16, 2, 1024, seed=12)
    full = vae.state_dict(); full.update(vsd); vae.load_state_dict(full)
    mg = M.MaskGit(image_size=16, transformer=tr.cuda(), vae=vae.cuda()).cuda()
    texts = ["a red apple", "a", "two green pears"]
    mg.sampler_noise_fn = util.torch_noise_fn(777)
    img_native, ids_native = mg.generate(texts=texts, timesteps=4, return_ids=True)
    te = enc(ids.cuda(), mask.cuda())
    tr.encode_text = lambda t: te
    mg.sampler_noise_fn = util.torch_noise_fn(777)
    img_ref, ids_ref = mg.generate(texts=texts, timesteps=4, return_ids=True)
    assert torch.equal(ids_native, ids_ref) and torch.equal(img_native, img_ref)
    assert t5.get_encoded_dim(name) == c["d_model"]


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_encoder_cuda_graph_replay(precision):
    c = C.SMALL_GATED
    enc, _ = _encoder(c, 9, precision)
    B, T = 4, 21
    ids1, mask1 = C.random_batch(B, T, c["vocab_size"], 1)
    ids2, mask2 = C.random_batch(B, T, c["vocab_size"], 2)
    s_ids, s_mask = ids1.cuda(), mask1.cuda()
    enc(s_ids, s_mask)                                   # packs the weights and caches the bucket map for T
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        s_out = enc(s_ids, s_mask)
    s_ids.copy_(ids2.cuda()); s_mask.copy_(mask2.cuda())
    graph.replay()
    eager = enc(ids2.cuda(), mask2.cuda())
    torch.cuda.synchronize()
    assert torch.equal(s_out, eager)
    assert not torch.equal(eager, enc(ids1.cuda(), mask1.cuda()))

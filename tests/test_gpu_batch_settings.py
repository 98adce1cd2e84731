"""GPU: per-image sampling settings (temperature, cond_scale, critic_noise_scale as device tables).

Kernels: each kernel's per-image (or per-row) table gives, row for row, bitwise what the scalar launch with that row's value gives, and a
scale of exactly 1 gives the x_null = NULL launch.  Models: image b of a mixed batch equals image b of a uniform call made with image b's
settings, for generate (no critic, TokenCritic, SelfCritic, superres, native step), inpaint and edit, under injected noise, libmmg's Philox
stream and the ATen stream; one captured graph replays for any settings."""
import math

import pytest
import torch

from oracle import synth
from tests import util
from tests.test_gpu_models import make_branch_maskgit, make_maskgit

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
bf = torch.bfloat16
SCALES = [1.0, 2.0, 3.0, 5.5]
TEMPS = [0.0, 0.5, 1.0, 2.0]
NOISE = [0.3, 1.0, 0.0, 2.5]


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _dev(v):
    return torch.tensor(v, dtype=torch.float32, device="cuda")


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dim,e_dtype", [(128, bf), (512, bf), (1024, torch.float32)])
def test_final_embed_per_image_scale(dim, e_dtype):
    o = ops()
    B, n, nm = 4, 24, 10
    g = torch.Generator(device="cuda").manual_seed(dim)
    xc = torch.randn((B * n, dim), generator=g, device="cuda") + 3
    xn = torch.randn((B * n, dim), generator=g, device="cuda")
    gamma = torch.rand((dim,), generator=g, device="cuda") + 0.5
    mp = torch.stack([torch.sort(torch.randperm(n, generator=g, device="cuda")[:nm]).values for _ in range(B)]).int().contiguous()
    got = torch.empty((B * nm, dim), device="cuda", dtype=e_dtype)
    o.final_embed(xc, xn, gamma, mp, got, B, n, nm, 7.0, cond_scale_dev=_dev(SCALES))
    null_launch = torch.empty_like(got)
    o.final_embed(xc, None, gamma, mp, null_launch, B, n, nm, 7.0)
    rows = (torch.arange(B, device="cuda")[:, None] * n + mp.long()).reshape(-1)
    ln = lambda x: torch.nn.functional.layer_norm(x[rows].double(), (dim,), eps=1e-5) * gamma.double()
    lc, lnull = ln(xc), ln(xn)
    for b, s in enumerate(SCALES):
        sl = slice(b * nm, (b + 1) * nm)
        scalar = torch.empty_like(got)
        o.final_embed(xc, xn, gamma, mp, scalar, B, n, nm, s)
        if s == 1:
            assert torch.equal(got[sl], null_launch[sl])
        else:
            assert torch.equal(got[sl], scalar[sl])
        want = lnull[sl] + (lc[sl] - lnull[sl]) * s
        tol = (2e-5 if e_dtype == torch.float32 else 2 ** -8) * float(want.abs().max())
        assert float((got[sl].double() - want).abs().max()) < tol


def test_critic_score_per_row_scale_and_noise():
    o = ops()
    B, n, dim = 4, 16, 128
    rows = B * n
    g = torch.Generator(device="cuda").manual_seed(3)
    xc, xn = torch.randn((rows, dim), generator=g, device="cuda"), torch.randn((rows, dim), generator=g, device="cuda")
    gamma, w = torch.rand((dim,), generator=g, device="cuda") + 0.5, torch.randn((dim,), generator=g, device="cuda")
    u = torch.rand((rows,), generator=g, device="cuda")
    cs, nm = _dev(SCALES).repeat_interleave(n), _dev(NOISE).repeat_interleave(n)
    for kw in (dict(u=u), dict(seed=99, step=2, row_offset=5)):
        got = torch.empty((rows,), device="cuda")
        o.critic_score(xc, xn, gamma, w, 0.25, 9.0, 9.0, got, cond_scale_dev=cs, noise_mul_dev=nm, **kw)
        for b in range(B):
            sl = slice(b * n, (b + 1) * n)
            want = torch.empty((rows,), device="cuda")
            o.critic_score(xc, None if SCALES[b] == 1 else xn, gamma, w, 0.25, SCALES[b], NOISE[b], want, **kw)
            assert torch.equal(got[sl], want[sl]), b
    # torch reference of the combine on the injected noise
    head = lambda x: (torch.nn.functional.layer_norm(x.double(), (dim,), eps=1e-5) * gamma.double()) @ w.double() + 0.25
    sc, sn = head(xc), head(xn)
    ref = torch.where(cs.double() == 1, sc, sn + (sc - sn) * cs.double()) + (u.double() - 0.5) * nm.double()
    got = torch.empty((rows,), device="cuda")
    o.critic_score(xc, xn, gamma, w, 0.25, 9.0, 9.0, got, u=u, cond_scale_dev=cs, noise_mul_dev=nm)
    assert float((got.double() - ref).abs().max()) < 1e-4


def _sample_case(b, nm, V, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    e = torch.randn((b * nm, K), generator=g, device="cuda").to(bf)
    w = (torch.randn((V, K), generator=g, device="cuda") * K ** -0.5).to(bf)
    n = nm + 3
    mp = torch.stack([torch.sort(torch.randperm(n, generator=g, device="cuda")[:nm]).values for _ in range(b)]).int().contiguous()
    return e, w, n, mp


def _sample(fused, e, w, n, mp, k, temp, **kw):
    o = ops()
    b, nm = mp.shape
    V = w.shape[0]
    ids = torch.full((b, n), V, dtype=torch.long, device="cuda"); sc = torch.full((b, n), -1e5, device="cuda")
    status = None
    if fused:
        R = b * nm
        ws = torch.empty((o.logits_fused_workspace_bytes(R, V, e.shape[1], k),), dtype=torch.uint8, device="cuda")
        status = torch.zeros((2,), dtype=torch.int32, device="cuda")
        o.logits_fused(e, w, mp, ids, sc, nm, k, temp, ws, status, rows_capacity=R, **kw)
    else:
        lg = torch.empty((e.shape[0], V), device="cuda")
        o.linear(e, w, lg)
        o.logits_sample(lg, mp, ids, sc, nm, k, temp, **kw)
    torch.cuda.synchronize()
    return ids, sc, status


@pytest.mark.parametrize("fused", [False, True], ids=["materialised", "fused"])
@pytest.mark.parametrize("bigk", [False, True], ids=["listk", "bigk"])
@pytest.mark.parametrize("noise", ["philox", "injected", "aten"])
def test_logits_sample_per_image_temperature(fused, bigk, noise):
    """Image b's rows under temperature_dev equal the scalar launch at TEMPS[b] bitwise (the fused tail's fallback leg: the next test)."""
    if fused and bigk:
        pytest.skip("the fused path declines k beyond its candidate lists")
    V, K, b, nm = (65536 if bigk else 8192), 128, 4, 20
    e, w, n, mp = _sample_case(b, nm, V, K, seed=11 + bigk)
    k = math.ceil((0.2 if bigk else 0.1) * V)          # 0.2 * 65536 > the candidate list of logits_sample_kernel: the row-walking kernel
    kw = dict(seed=1234, step=3, row_offset=5 * n)
    if noise == "injected":
        kw = dict(u=torch.rand((b, n, V), device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)))
    elif noise == "aten":
        kw = dict(seed=0, seed_dev=torch.tensor([99], dtype=torch.int64, device="cuda"),
                  aten=(16, torch.tensor([8], dtype=torch.int64, device="cuda"), 256 * 40))
    ids, sc, status = _sample(fused, e, w, n, mp, k, 9.0, temperature_dev=_dev(TEMPS), **kw)
    if fused:
        assert int(status[1]) == 0, status
    for i, t in enumerate(TEMPS):
        ids_s, sc_s, _ = _sample(fused, e, w, n, mp, k, t, **kw)
        assert torch.equal(ids[i], ids_s[i]) and torch.equal(sc[i], sc_s[i]), (i, t)
    if noise == "injected":     # fp64 oracle on the rows of image 2 (temperature 1)
        rows = list(range(2 * nm, 3 * nm))
        lg = (e[rows].double() @ w.double().T).cpu()
        u_rows = kw["u"][2, mp[2].long()].cpu().double()
        pred, _, margin = util.oracle_rows(lg, u_rows, TEMPS[2], k)
        ok = margin > 1e-3
        assert bool((ids[2, mp[2].long()].cpu()[ok] == pred[ok]).all())


def test_fused_fallback_rows_read_their_own_image_temperature():
    """The hand-built rows of tests/test_gpu_fused_tail.py, one image each (one-hot embeddings: the logits are exact, the noise injected).
    Images 3..5 hold the rows built to overflow their candidate lists (segment, fifo) or to miss the sampled threshold: they are redone
    through materialised logits and the row_index list, whose entry i is not image i.  Their logits are not constant, and the segment and
    fifo rows sample a different token at their own temperature than at image 0's or the scalar's (checked on the oracle below), so a
    fallback that read the wrong temperature would fail.  Every row equals the scalar launch at its image's temperature and the fp64 oracle."""
    from oracle import fused_tail as FT
    from tests.test_gpu_fused_tail import _constructed_rows
    o = ops()
    V, K = 65536, 512
    k = math.ceil(0.1 * V)
    plan = FT.lf_plan(1, V, torch.cuda.get_device_properties(0).multi_processor_count)
    names, x, u = _constructed_rows(V, k, plan, torch.Generator().manual_seed(17))
    order = ["plain", "tie", "excl10", "segment", "fifo", "threshold"]        # list rows first, then the fallback rows
    sel = [names.index(m) for m in order]
    x, u = x[sel], u[sel]
    temps = [1.0, 1.0, 1.0, 0.3, 1.7, 0.6]             # the list rows keep the temperature they were built for
    R = len(order)
    assert FT.lf_plan(R, V, torch.cuda.get_device_properties(0).multi_processor_count) == plan
    preds = [util.oracle_rows(x[r:r + 1].double(), u[r:r + 1], t, k) for r, t in enumerate(temps)]
    for r in (3, 4):                                   # the test can tell a wrong temperature apart on these rows
        wrong, _, _ = util.oracle_rows(x[r:r + 1].double(), u[r:r + 1], 1.0, k)
        assert int(wrong) != int(preds[r][0]), order[r]
    assert min(float(m) for _, _, m in preds) > 1e-4
    w = torch.zeros((V, K), dtype=bf)
    w[:, :R] = x.T.to(bf)
    w = w.cuda()
    e = torch.zeros((R, K), dtype=bf, device="cuda")
    e[torch.arange(R), torch.arange(R)] = 1
    uc = u.cuda().view(R, 1, V)
    mp = torch.zeros((R, 1), dtype=torch.int32, device="cuda")
    ws = torch.empty((o.logits_fused_workspace_bytes(R, V, K, k),), dtype=torch.uint8, device="cuda")

    def run(temp, temperature_dev=None):
        status = torch.zeros((2,), dtype=torch.int32, device="cuda")
        ids = torch.full((R, 1), V, dtype=torch.long, device="cuda"); sc = torch.full((R, 1), -1e5, device="cuda")
        o.logits_fused(e, w, mp, ids, sc, 1, k, temp, ws, status, rows_capacity=R, u=uc, temperature_dev=temperature_dev)
        torch.cuda.synchronize()
        return ids[:, 0], sc[:, 0], status.tolist()

    ids, sc, status = run(1.0, _dev(temps))
    assert status == [3, 0], status                    # segment, fifo, threshold took the fallback leg
    for r, t in enumerate(temps):
        ids_s, sc_s, _ = run(t)
        assert int(ids[r]) == int(ids_s[r]) and float(sc[r]) == float(sc_s[r]), (order[r], t)
        pred, osc, _ = preds[r]
        assert int(ids[r]) == int(pred), (order[r], int(ids[r]), int(pred))
        assert abs(float(sc[r]) - float(osc)) < 1e-5, order[r]


# ------------------------------------------------------------------------------------------------ models
def _te():
    return util.text_embeds("g4.te", 3, 8, 128, 14).cuda().repeat(2, 1, 1)[:4]


def _images(size):
    return torch.from_numpy(synth.uniform("settings.img", (4, 3, size, size), 41)).cuda()


def _ragged(f=4):
    g = torch.Generator().manual_seed(2)
    m = torch.stack([torch.rand((f, f), generator=g) < fr for fr in (0.5, 0.8, 0.3, 1.1)])
    m[2, 0, 0] = True
    return m.cuda()


def _variant(name):
    """(maskgit, call(**settings) -> (images, ids), critic present, noise: a function that resets the noise before each call)."""
    te = _te()
    kw, critic = {}, False
    if name in ("token_critic", "self_critic"):
        mg, kw, seed = make_branch_maskgit("gen_critic_small" if name == "token_critic" else "gen_selfcritic_small", "fp32")
        kw.pop("critic_noise_scale", None)
        critic = True
    elif name == "superres":
        mg = make_maskgit("bf16", superres=True)
    else:
        mg = make_maskgit("fp32" if name in ("generate_fp32", "edit_fp32") else "bf16")
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    texts = ["a"] * 4
    if name == "superres":
        cond = _images(16)
        call = lambda **s: mg.generate(texts, cond_images=cond, timesteps=5, return_ids=True, **s)
    elif name == "inpaint":
        img, m = _images(16), _ragged()
        call = lambda **s: mg.inpaint(texts, img, m, timesteps=5, return_ids=True, **s)
    elif name in ("edit", "edit_fp32"):
        img, m = _images(16), _ragged()
        call = lambda **s: mg.edit(texts, img, mask=m, iterations=2, fraction=0.5, timesteps=3, return_ids=True, **s)
    else:
        call = lambda **s: mg.generate(texts, timesteps=6, return_ids=True, **kw, **s)
    if name == "native":
        mg.use_native_step = True
    if name in ("generate_fp32", "edit_fp32", "token_critic", "self_critic"):
        reset = lambda: setattr(mg, "sampler_noise_fn", util.torch_noise_fn(901))
    elif name == "aten":
        mg.sampler_rng = "aten"
        reset = lambda: torch.manual_seed(902)
    else:
        mg.sampler_seed = 903
        reset = lambda: None
    return mg, call, critic, reset


VARIANTS = ["generate_fp32", "generate_bf16", "aten", "token_critic", "self_critic", "superres", "inpaint", "edit", "edit_fp32", "native"]


@pytest.mark.parametrize("name", VARIANTS)
def test_mixed_batch_equals_uniform_calls_image_by_image(name):
    mg, call, critic, reset = _variant(name)
    mixed = dict(cond_scale=SCALES, temperature=torch.tensor(TEMPS))
    if critic:
        mixed["critic_noise_scale"] = NOISE
    reset()
    img, ids = call(**mixed)
    for b in range(4):
        uni = dict(cond_scale=SCALES[b], temperature=TEMPS[b])
        if critic:
            uni["critic_noise_scale"] = NOISE[b]
        reset()
        img_u, ids_u = call(**uni)
        assert torch.equal(ids[b], ids_u[b]), (name, b, int((ids[b] != ids_u[b]).sum()))
        assert torch.equal(img[b], img_u[b]), (name, b)


@pytest.mark.parametrize("bad", [dict(cond_scale=[3, 3]), dict(temperature=[1, float("nan"), 1, 1]), dict(critic_noise_scale=float("inf")),
                                 dict(temperature=[1, -0.5, 1, 1])], ids=["length", "nan", "inf", "negative"])
def test_bad_settings_raise_before_any_launch_on_the_device(bad):
    """On a CUDA model whose graphs and workspaces are warm: the failing call launches nothing (mmg_launch_count unchanged) and leaves
    the graph cache as it was."""
    from muse_maskgit_pytorch_b200 import _lib
    mg, call, _, _ = _variant("generate_bf16")
    images = _images(16)
    call(cond_scale=3)
    torch.cuda.synchronize()
    keys = list(mg._graphs)
    before = _lib.launch_count()
    for fn in (lambda: call(**bad), lambda: mg.inpaint(["a"] * 4, images, _ragged(), timesteps=5, **bad),
               lambda: mg.edit(["a"] * 4, images, iterations=1, timesteps=3, **bad)):
        with pytest.raises(ValueError):
            fn()
    assert _lib.launch_count() == before and list(mg._graphs) == keys


def test_scalar_call_equals_repeated_per_image_values():
    mg, call, _, _ = _variant("generate_bf16")
    for s in (dict(cond_scale=3, temperature=0.7), dict(cond_scale=1, temperature=1.3)):
        img, ids = call(**s)
        img2, ids2 = call(**{k: [v] * 4 for k, v in s.items()})
        assert torch.equal(ids, ids2) and torch.equal(img, img2)


def test_one_graph_replays_for_any_settings():
    mg, call, _, _ = _variant("generate_bf16")
    img0, ids0 = call(cond_scale=3, temperature=1)
    keys = list(mg._graphs)
    graph = mg._graphs[keys[-1]].graph
    for s in (dict(cond_scale=5, temperature=0.7), dict(cond_scale=SCALES, temperature=TEMPS),
              dict(cond_scale=torch.tensor([2., 4., 6., 8.], device="cuda"), temperature=(0.1, 0.2, 0.3, 0.4))):
        img, ids = call(**s)
        assert list(mg._graphs) == keys and mg._graphs[keys[-1]].graph is graph, s
        mg.use_cuda_graph = False
        img_e, ids_e = call(**s)
        mg.use_cuda_graph = True
        assert torch.equal(ids, ids_e) and torch.equal(img, img_e), s
    mg._graphs.clear()
    for s in (2, 3, 4, 5, 6, 7.5):
        call(cond_scale=s)
    assert len(mg._graphs) == 1
    call(cond_scale=1)
    assert len(mg._graphs) == 2


@pytest.mark.parametrize("settings", [dict(cond_scale=3, temperature=0.8), dict(cond_scale=SCALES, temperature=TEMPS)], ids=["scalar", "per_image"])
def test_whole_call_captured_by_the_caller(settings):
    """generate() with use_cuda_graph = False captured into the caller's own CUDA graph (the settings tables are then built with fill
    kernels, which a capture can record): the replay equals the eager call."""
    mg, call, _, _ = _variant("generate_bf16")
    mg.use_cuda_graph, mg.check_fused_tail = False, False
    img_e, ids_e = call(**settings)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        img_g, ids_g = call(**settings)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(ids_g, ids_e) and torch.equal(img_g, img_e)


def test_generate_sharded_per_image_settings_on_device():
    """row_offset sharding with per-image settings: a shard generated alone reproduces its rows of the whole batch."""
    mg, call, _, _ = _variant("generate_bf16")
    te = _te()
    _, ids = call(cond_scale=SCALES, temperature=TEMPS)
    mg.row_offset = 1
    mg.transformer.encode_text = lambda texts: te[1:1 + len(texts)]
    _, ids_s = mg.generate(["a"] * 3, timesteps=6, return_ids=True, cond_scale=SCALES[1:], temperature=TEMPS[1:])
    assert torch.equal(ids_s, ids[1:])

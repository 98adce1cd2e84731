"""The GEMM oracle checked on the CPU: the fp64 references against torch's F.linear / F.conv2d / F.conv_transpose2d, the restated dispatch
against a hand-written table at 132 and 114 SMs, the clean restatement of the tiled product inside the bound, and every planted defect
outside it by more than 100 times on the probe cases."""
import pytest
import torch
import torch.nn.functional as F

from tests import gemm_oracle as G

torch.set_grad_enabled(False)


# ------------------------------------------------------------------------------------------------ references
def test_linear_reference_agrees_with_torch():
    a, w = G.probe_dense("ref.lin", 70, 192, 128, bf16=False)
    bias = G.rnd("ref.lin.b", (192,))
    resid = G.rnd("ref.lin.r", (70, 192))
    ref, S, _ = G.linear_ref(a, w, G.RESIDUAL, {"bias": bias, "resid": resid})
    want = F.linear(a.double(), w.double(), bias.double()) + resid.double()
    assert float((ref - want).abs().max()) < 1e-12
    assert bool((S >= ref.abs() - 1e-12).all())
    ref, _, _ = G.linear_ref(a, w, G.STORE, {"bias": bias, "act": 1})
    assert float((ref - F.leaky_relu(F.linear(a.double(), w.double(), bias.double()), 0.1)).abs().max()) < 1e-12


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_conv_reference_agrees_with_torch(kind):
    k, pad = ((1, 0), (3, 1), (4, 1), (5, 2))[kind]
    stride = 2 if kind == 2 else 1
    x = G.probe_image(f"ref.conv{kind}", 2, 8, 6, 5, bf16=False)
    wt = G.rnd(f"ref.conv{kind}.w", (7, 5, k, k))
    ref, _, _ = G.conv_ref(x, G.pack_conv_weight(wt), kind, G.STORE, {})
    want = F.conv2d(x.permute(0, 3, 1, 2).double(), wt.double(), stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(ref.shape)
    assert float((ref - want).abs().max()) < 1e-12


@pytest.mark.parametrize("rgb", [False, True], ids=["convt", "convt_rgb"])
def test_conv_transpose_reference_agrees_with_torch(rgb):
    x = G.probe_image("ref.ct", 2, 4, 6, 5, bf16=False)
    wt = G.rnd("ref.ct.w", (5, 8, 4, 4))
    bias = G.rnd("ref.ct.b", (8,))
    p = {"bias": bias}
    y = F.leaky_relu(F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), wt.double(), bias.double(), stride=2, padding=1), 0.1)
    if rgb:
        p.update(rgb_w=G.rnd("ref.ct.rw", (3, 8)), rgb_b=G.rnd("ref.ct.rb", (3,)))
        y = F.conv2d(y, p["rgb_w"].double()[:, :, None, None], p["rgb_b"].double())
    else:
        y = y.permute(0, 2, 3, 1)
    ref, _, _ = G.convt_ref(x, G.pack_convt_weight(wt), p, rgb)
    assert float((ref - y).abs().max()) < 1e-12


# ------------------------------------------------------------------------------------------------ dispatch
TC, SIMT = G.TC, G.SIMT
F32 = {"out": "f32"}


def test_dispatch_table():
    L = G.linear_kernels
    for sms in (132, 114):
        assert L(300, 192, 128, G.STORE, F32, sms=sms) == [TC(64, G.M_REGS)]                       # N % 128 == 64
        assert L(300, 256, 128, G.STORE, F32, sms=sms) == [TC(64, G.M_REGS)]                       # plain fp32, but 64 wide
        assert L(300, 256, 128, G.STORE, {"out": "f32", "bias": True}, sms=sms) == [TC(64, G.M_REGS)]
        assert L(12800, 256, 64, G.STORE, F32, sms=sms) == [TC(128, G.M_TSTORE)]                    # 100 m-tiles x 2 >= 96
        assert L(300, 1024, 64, G.STORE, {"out": "f32", "bias": True}, sms=sms) == [TC(128, G.M_REGS)]
        assert L(300, 192, 128, G.RESIDUAL, {"out": "f32", "in_place": True}, sms=sms) == [TC(64, G.M_REDUCE)]
        assert L(300, 192, 128, G.RESIDUAL, {"out": "f32", "in_place": True, "ldo": 194}, sms=sms) == [SIMT("bf16", False, False)]
        assert L(300, 192, 128, G.RESIDUAL, {"out": "f32", "in_place": True, "out_aligned": False}, sms=sms) == [TC(64, G.M_REGS)]
        assert L(300, 192, 128, G.GEGLU_TANH, {"out": "bf16"}, sms=sms) == [TC(128, G.M_ACT)]
        assert L(300, 192, 128, G.STORE, {"out": "bf16", "act": 2}, dtype="f32", sms=sms) == [SIMT("f32", False, True)]
        assert L(300, 192, 100, G.STORE, F32, sms=sms) == [SIMT("bf16", False, False)]
        assert L(300, 192, 128, G.STORE, F32, lda=132, sms=sms) == [SIMT("bf16", False, False)]
        assert L(300, 192, 128, G.STORE, F32, lda=136, ldw=200, sms=sms) == [TC(64, G.M_REGS)]
        assert L(300, 192, 128, G.STORE, F32, dtype="f32", split=True, sms=sms) == [G.SPLIT3, TC(64, G.M_REGS)]
        q = {"out": "bf16", "tokens": 64, "nk": 2, "nv": 2}
        assert L(256, 384, 128, G.QKV, q, sms=sms) == [TC(64, G.M_REGS)]                            # bn 64: no tile epilogue
        assert L(2048, 768, 128, G.QKV, q, sms=sms) == [TC(128, G.M_QKV)]                           # 16 x 6 tiles >= 96
        assert L(2048, 768, 128, G.QKV, dict(q, tokens=16), sms=sms) == [TC(128, G.M_REGS)]
        assert G.conv_kernels(1, 3, 8, 8, 64, 64, G.STORE, F32, sms=sms) == [TC(64, G.M_REGS)]
        assert G.conv_kernels(3, 3, 8, 8, 64, 64, G.STORE, F32, sms=sms) == [SIMT("bf16", True, False)]
        assert G.conv_kernels(1, 3, 3, 3, 64, 64, G.STORE, F32, sms=sms) == [SIMT("bf16", True, False)]
        assert G.conv_kernels(1, 3, 8, 8, 32, 64, G.STORE, F32, dtype="f32", split=True, sms=sms) == [G.SPLIT3, TC(64, G.M_REGS)]
        assert G.convt_kernels(2, 8, 8, 64, 128, True, sms=sms) == [TC(128, G.M_REGS)] * 4
        assert G.convt_kernels(2, 8, 8, 64, 256, True, sms=sms) == [TC(256, G.M_REGS)] * 4
        assert G.convt_kernels(2, 3, 3, 64, 64, False, sms=sms) == [SIMT("bf16", True, False)] * 4
        with pytest.raises(ValueError):
            G.convt_kernels(2, 3, 3, 64, 64, True, sms=sms)
    # where the SM count decides the tile width: 33 m-tiles x 4 256-column tiles = 132 < 2 * 114
    assert G.linear_kernels(33 * 128, 1024, 64, G.STORE, F32, sms=132) == [TC(128, G.M_TSTORE)]
    assert G.linear_kernels(66 * 128, 1024, 64, G.STORE, F32, sms=132) == [TC(256, G.M_TSTORE)]
    assert G.linear_kernels(58 * 128, 1024, 64, G.STORE, F32, sms=114) == [TC(256, G.M_TSTORE)]
    assert G.linear_kernels(58 * 128, 1024, 64, G.STORE, F32, sms=132) == [TC(128, G.M_TSTORE)]
    assert G.linear_kernels(58 * 128, 1024, 64, G.GEGLU, {"out": "bf16"}, sms=114) == [TC(256, G.M_GEGLU)]
    assert G.linear_kernels(58 * 128, 1024, 64, G.GEGLU, {"out": "bf16"}, sms=132) == [TC(128, G.M_REGS)]
    # e4m3 (mmg_linear_fp8) always takes its tile epilogue: the small-M cross-attention q product runs <128, QKV> where bf16 runs <64, REGS>
    assert G.fp8_plan(G.QKV, 256, 128, 128, 132) == (128, G.M_QKV, 0)
    assert G.linear_kernels(256, 128, 128, G.QKV, {"out": "bf16", "tokens": 64, "nk": 0, "nv": 0}, sms=132) == [TC(64, G.M_REGS)]
    assert G.fp8_plan(G.QKV, 32768, 1536, 512, 132) == (256, G.M_QKV, 1)
    assert G.fp8_plan(G.QKV128, 384, 768, 256, 132) == (128, G.M_QKV128, 1)
    assert G.fp8_plan(G.GEGLU, 129, 2816, 256, 132) == (256, G.M_GEGLU, 1)
    assert G.fp8_plan(G.GEGLU, 1000, 4352, 512, 132) == (256, G.M_GEGLU, 0)                  # 17 column tiles


def test_tile_geometry():
    assert G.tile_geometry(8, 8) == (8, 8, 2, 1, 1)
    assert G.tile_geometry(4, 16) == (16, 4, 2, 1, 1)
    assert G.tile_geometry(8, 256) == (128, 1, 1, 2, 8)
    assert G.tile_geometry(6, 128) == (128, 1, 1, 1, 6)
    assert G.tile_geometry(32, 32) == (32, 4, 1, 1, 8)
    assert G.tile_geometry(3, 3) is None and G.tile_geometry(6, 8) is None and G.tile_geometry(8, 48) is None


# ------------------------------------------------------------------------------------------------ probe cases of the restatement
def _dense(kind, p_extra=None, M=300, N=256, K=192):
    a, w = G.probe_dense(f"probe.{kind}", M, N, K)
    p = {"bias": G.bf(G.rnd(f"probe.{kind}.b", (N,)))}
    if kind == G.RESIDUAL:
        p["resid"] = G.rnd(f"probe.{kind}.r", (M, N))
    if kind == G.GEGLU:
        p = {}
    if kind == G.LNFOLD:
        h = G.rnd("probe.ln.h", (M, 256)) + 0.5
        p = {"bias": G.rnd("probe.ln.c", (N,)), "resid": G.rnd("probe.ln.r", (M, N)), "ln_width": 256,
             "stats": torch.stack([h.reshape(M, 4, 64).sum(-1), (h * h).reshape(M, 4, 64).sum(-1)], -1)}
    if kind == G.QKV:
        p = {"heads": 2, "tokens": 50, "key_off": 1, "q_rows": 50, "kv_rows": 56, "q_scale": 1 + 0.1 * G.rnd("probe.qs", (64,)),
             "k_scale": 1 + 0.1 * G.rnd("probe.ks", (64,)), "null_k": G.rnd("probe.nk", (2, 64)), "null_v": G.rnd("probe.nv", (2, 64))}
        N = 384
        a, w = G.probe_dense("probe.qkv", M, N, K)
    p.update(p_extra or {})
    return a, w, p


def _flat(out):
    return torch.cat([v.reshape(-1) for v in out.values()]) if isinstance(out, dict) else out


def _ratio_dense(kind, defect, data, out_bf16=False, old=False, plan=(64, 1)):
    a, w, p = data
    ref, S, A = G.linear_ref(a, w, kind, p)
    got = G.emulate_linear(a, w, kind, p, plan, defect, out_bf16)
    ref, S, A, got = _flat(ref), _flat(S), _flat(A), _flat(got)
    tol = G.old_tolerance(ref, out_bf16) if old else G.tolerance(G.TC(64, 0), a.shape[1], ref, S, A, out_bf16)
    return G.worst_ratio(got, ref, tol)


def _conv_case(tag, kind, B, H, W, C=64, N=128):
    x = G.probe_image(tag, B, H, W, C)
    k = (1, 3, 4, 5)[kind]
    wp = G.bf(G.pack_conv_weight(G.rnd(tag + ".w", (N, C, k, k), 0.2)))
    return x, wp, {"bias": G.rnd(tag + ".b", (N,))}


def _ratio_conv(kind, defect, data, out_bf16=False, old=False):
    x, wp, p = data
    Ho, Wo = G.conv_out_hw(kind, x.shape[1], x.shape[2])
    ref, S, A = G.conv_ref(x, wp, kind, G.STORE, p)
    got = G.emulate_conv(x, wp, kind, G.STORE, p, (64, 1), G.tile_geometry(Ho, Wo), defect, out_bf16)
    tol = G.old_tolerance(ref, out_bf16) if old else G.tolerance(G.TC(64, 0), wp.shape[1], ref, S, A, out_bf16)
    return G.worst_ratio(got, ref, tol)


def _convt_case(tag, B=3, H=8, W=8, C=64, N=64):
    x = G.probe_image(tag, B, H, W, C)
    wp = G.bf(G.pack_convt_weight(G.rnd(tag + ".w", (C, N, 4, 4), 0.2)))
    return x, wp, {"bias": G.rnd(tag + ".b", (N,))}


def _ratio_convt(defect, data, out_bf16=False, old=False):
    x, wp, p = data
    ref, S, A = G.convt_ref(x, wp, p)
    got = G.emulate_convt(x, wp, p, (64, 1), G.tile_geometry(x.shape[1], x.shape[2]), defect, out_bf16)
    tol = G.old_tolerance(ref, out_bf16) if old else G.tolerance(G.TC(64, 0), wp.shape[2], ref, S, A, out_bf16)
    return G.worst_ratio(got, ref, tol)


# defect -> the probe case it is planted in
def _probe(defect, out_bf16=False, old=False, data_of=None):
    dense = {"drop_last_kblock": G.STORE, "kblock_twice": G.RESIDUAL, "ragged_row_off_by_one": G.STORE, "tile_order_swapped": G.STORE,
             "geglu_x_gate_swapped": G.GEGLU, "lnfold_one_slot_short": G.LNFOLD, "qkv_next_head": G.QKV, "null_row_missing": G.QKV}
    if defect in dense:
        kind = dense[defect]
        return _ratio_dense(kind, defect, (data_of or _dense)(kind), out_bf16, old)
    if defect == "convt_parity_swapped":
        return _ratio_convt(defect, _convt_case("probe.ct"), out_bf16, old)
    kind, B, H, W = {"tap_dx_dy_swapped": (1, 3, 8, 8), "parity_py_px_swapped": (2, 3, 16, 16), "wrong_image_in_tile": (1, 5, 8, 8)}[defect]
    return _ratio_conv(kind, defect, _conv_case("probe." + defect, kind, B, H, W), out_bf16, old)


CLEAN = [("dense", G.STORE), ("dense", G.RESIDUAL), ("dense", G.GEGLU), ("dense", G.LNFOLD), ("dense", G.QKV), ("conv", 1), ("conv", 2),
         ("conv", 0), ("convt", None)]


@pytest.mark.parametrize("out_bf16", [False, True], ids=["f32out", "bf16out"])
@pytest.mark.parametrize("what,kind", CLEAN, ids=[f"{w}{k}" for w, k in CLEAN])
def test_clean_restatement_is_inside_the_bound(what, kind, out_bf16):
    """fp32 outputs: at most half the bound.  bf16 outputs: the fp32 value before the output rounding at most half the bound without its
    rounding term, and the rounded output inside the whole bound (the half-ulp rounding reaches its own term by construction)."""
    if what == "dense":
        r = _ratio_dense(kind, None, _dense(kind), False)
        rb = _ratio_dense(kind, None, _dense(kind), True) if out_bf16 else 0.0
    elif what == "conv":
        B, H, W = {0: (3, 4, 16), 1: (5, 8, 8), 2: (3, 16, 16)}[kind]
        r = _ratio_conv(kind, None, _conv_case(f"clean{kind}", kind, B, H, W), False)
        rb = _ratio_conv(kind, None, _conv_case(f"clean{kind}", kind, B, H, W), True) if out_bf16 else 0.0
    else:
        r = _ratio_convt(None, _convt_case("clean.ct"), False)
        rb = _ratio_convt(None, _convt_case("clean.ct"), True) if out_bf16 else 0.0
    print(f"{what} {kind}: fp32 worst err / tol {r:.4f}" + (f", bf16 out {rb:.3f}" if out_bf16 else ""))
    assert r <= 0.5 and rb <= 1.0, (r, rb)


@pytest.mark.parametrize("defect", G.DEFECTS)
def test_every_planted_defect_is_rejected(defect):
    r, rb = _probe(defect), _probe(defect, out_bf16=True)
    print(f"{defect}: worst err / tol {r:.3g} (fp32 out), {rb:.3g} (bf16 out)")
    assert r > 100 and rb > 100, (r, rb)


def _old_data(kind):
    """the kind of data tests/test_gpu_kernels.py uses: bf16-representable N(0, 1) operands, no probe structure"""
    a, w, p = _dense(kind)
    M, K = a.shape
    return G.bf(G.rnd(f"old.{kind}.a", (M, K))), G.bf(G.rnd(f"old.{kind}.w", (w.shape[0], K))), p


def test_what_the_old_rules_accepted():
    """a report: which planted defects 2e-2 + 1e-2 |ref| (bf16 out) and 2e-4 + 1e-3 |ref| (fp32 out) accept on random N(0, 1) operands
    of the dense probe shapes, and on the probe data of the conv cases"""
    lines = []
    for d in G.DEFECTS:
        acc = {o: _probe(d, out_bf16=o, old=True, data_of=_old_data) <= 1.0 for o in (False, True)}
        lines.append(f"{d}: fp32 rule {'ACCEPTED' if acc[False] else 'rejected'}, bf16 rule {'ACCEPTED' if acc[True] else 'rejected'}")
    print("\n".join(lines))

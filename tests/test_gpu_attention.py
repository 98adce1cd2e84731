"""GPU tests of mmg_attention, variant by variant, against the fp64 reference and the tolerances of tests/attention_oracle.py.

Five kernels sit behind the one entry point: attention_tc_kernel<64> (bf16, 1..640 real keys), attention_tc_kernel<128> (641..4095),
attention_tc_split_kernel (fp32 operands as three bf16 terms), and the CUDA-core attention_simt_kernel<__nv_bfloat16> / <float> that take
what the wgmma kernels cannot (unaligned pointers, ldo % 8 != 0, Tk < 2 or > 4096, fp32 with fp32_tc(False)).  Every case names the kernel
its arguments are chosen to reach and asserts, from a torch.profiler capture, that exactly that kernel ran; cases on the wgmma kernels also
assert that the CUDA-core launch counter did not move, the fallback cases that it rose by one.  The captures are taken in a process of
their own (see PROFILE): this file runs early in a whole-suite process, and a few hundred profiler sessions there, before the model and
graph tests, made the short captures of tests/test_gpu_row_kernels.py come back empty later in the same process.  The operands carry probe data (dominant keys
at the block and tail edges, a per-key signature in V), so an indexing slip moves the output by orders of magnitude more than the
tolerance.  The last test prints, per variant, how many cases reached it and the worst |err| / tol."""
import os
import subprocess
import sys

import pytest
import torch

from tests import attention_oracle as A
from tests.test_gpu_row_kernels import kernels_of, assert_ran

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

BF, F32 = torch.bfloat16, torch.float32
FILL = -77.0                       # guard value of the output buffer: columns past heads * 64 and rows past B * Tq keep it
STATS = {}                         # (variant, softmax mode, masked) -> [cases, worst err / tol]
# Set in the child process that test_every_case_reached_its_kernel starts: there every case runs under torch.profiler and asserts the
# kernel it reached.  Without it the cases check everything else (numbers, guards, the CUDA-core launch counter) and take no capture.
PROFILE = os.environ.get("MMG_ATTENTION_PROFILE") == "1"


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def lib():
    from muse_maskgit_pytorch_b200 import _lib
    return _lib


@pytest.fixture(scope="module", autouse=True)
def _warm_up():
    """one throw-away capture: the first CUPTI session of a process pays its set-up inside the capture"""
    if PROFILE and torch.cuda.is_available():
        kernels_of(lambda: torch.ones(8, device="cuda").sum())


def observed(fn, *want):
    """fn() and, in the profiling process, the assertion that exactly the libmmg kernels `want` ran"""
    if not PROFILE:
        return fn()
    out, names = kernels_of(fn)
    assert_ran(names, *want)
    return out


class fp32_on_cuda_cores:
    """fp32_tc(False) for the duration of a block"""

    def __enter__(self):
        self.was = ops().fp32_tc()
        ops().fp32_tc(False)

    def __exit__(self, *exc):
        ops().fp32_tc(self.was)


def garbage(shape, dtype):
    """large finite values of alternating sign"""
    g = torch.full(shape, 1e30, dtype=torch.float32)
    g[..., 1::2] = -1e30
    return g.to(dtype)


def launch(q, k, v, mask, dtype, *, scale=8.0, bound=0.0, pad=None, pad_garbage=False, ldo_extra=0, guard_rows=0, q_offset=0):
    """Uploads fp32 CPU operands as `dtype`, runs ops.attention into a FILL-ed buffer of B * Tq + guard_rows rows of heads * 64 + ldo_extra
    columns and returns (the buffer, the rise of the CUDA-core launch counter).  K / V get `pad` rows past Tk (default: up to a multiple of
    8), zero or garbage; q starts q_offset elements into its allocation."""
    B, H, Tq, _ = q.shape
    Bk, Tk = k.shape[0], k.shape[2]
    alloc = Tk + ((-Tk) % 8 if pad is None else pad)

    def kv(t):
        buf = torch.zeros((Bk * H, alloc, 64), dtype=dtype)
        if pad_garbage:
            buf[:, Tk:] = garbage((Bk * H, alloc - Tk, 64), dtype)
        buf[:, :Tk] = t.reshape(Bk * H, Tk, 64).to(dtype)
        return buf.cuda()
    n = B * H * Tq * 64
    qflat = torch.zeros(n + 16, dtype=dtype, device="cuda")
    qd = qflat[q_offset:q_offset + n].view(B * H, Tq, 64)
    qd.copy_(q.reshape(B * H, Tq, 64).to(dtype))
    out = torch.full((B * Tq + guard_rows, H * 64 + ldo_extra), FILL, dtype=dtype, device="cuda")
    md = None if mask is None else mask.to(torch.uint8).contiguous().cuda()
    before = lib().simt_launch_count()
    ops().attention(qd, kv(k), kv(v), out, B, H, Tk, key_mask=md, kv_shared=Bk == 1 and B > 1, scale=scale, logit_bound=bound)
    torch.cuda.synchronize()
    return out, lib().simt_launch_count() - before


def run_case(tag, B, H, Tq, Tk, dtype, want, *, mask_kind=None, kv_shared=False, scale=8.0, bound=0.0, **kw):
    """One call on probe operands: which kernel ran, the CUDA-core counter, fp64 tolerance, guard columns and rows, and (bf16 wgmma) the
    fully masked entry equal to the null value bit for bit.  Returns the output [B, H, Tq, 64] on the CPU."""
    q, k, v = A.operands(tag, B, H, Tq, Tk, dtype == BF, kv_shared=kv_shared)
    mask = A.mask_of(mask_kind, tag, B, Tk)
    buf, simt = observed(lambda: launch(q, k, v, mask, dtype, scale=scale, bound=bound, **kw), want, *((A.SPLIT3,) if want == A.SPLIT else ()))
    assert simt == (1 if want in (A.SIMT_BF16, A.SIMT_F32) else 0), f"{want}: CUDA-core launch counter moved by {simt}"
    buf = buf.cpu()
    got = buf[:B * Tq, :H * 64].reshape(B, Tq, H, 64).transpose(1, 2)
    ref, w = A.reference(q, k, v, mask, scale)
    assert bool(torch.isfinite(got.float()).all()), f"{want}: non-finite output at {(~torch.isfinite(got.float())).nonzero()[:4].tolist()}"
    r = A.worst_ratio(got, ref, A.tolerance(want, ref, w, scale, Tk))
    mode = "single-pass" if want in (A.TC64, A.TC128) and A.single_pass(scale, bound) else "two-pass"
    st = STATS.setdefault((want, mode, "masked" if mask is not None else "unmasked"), [0, 0.0])
    st[0] += 1; st[1] = max(st[1], r)
    if r > 1.0:
        err = (got.double() - ref).abs() / A.tolerance(want, ref, w, scale, Tk)
        b, h, i, d = (int(x) for x in (err == err.max()).nonzero()[0])
        raise AssertionError(f"{want} {tag}: worst err / tol {r:.2f} at (batch {b}, head {h}, query {i}, column {d}): got {float(got[b, h, i, d]):.6e} "
                             f"want {float(ref[b, h, i, d]):.6e}; {int((err > 1).sum())} elements out of tolerance")
    assert bool((buf[:, H * 64:] == FILL).all()) and bool((buf[B * Tq:] == FILL).all()), f"{want}: guard columns or rows were written"
    if want in (A.TC64, A.TC128) and mask is not None and not bool(mask[0].any()):
        null_v = v[0, :, :1].expand(-1, Tq, -1).to(BF)
        assert torch.equal(got[0].contiguous().view(torch.int16), null_v.contiguous().view(torch.int16)), \
            f"{want}: a fully masked entry must be the null value bit for bit (max diff {float((got[0].float() - null_v.float()).abs().max()):.3e})"
    return got


# ------------------------------------------------------------------------------------------------ block edges, bf16 wgmma
REAL_KEYS = [1, 31, 32, 33, 63, 64, 65, 96, 97, 129, 639, 640, 641, 672, 704, 736, 1000, 1024, 4095]


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("bound", [0.0, 1.02], ids=["twopass", "singlepass"])
@pytest.mark.parametrize("real", REAL_KEYS)
def test_wgmma_block_edges(real, bound, masked):
    """1..640 real keys on 64-key blocks, 641..4095 on 128-key blocks, with tails of 32, 64, 96 and 128 keys; heads = 3 with a per-entry
    mask (the mask row is bh / heads)"""
    want = A.TC64 if real <= 640 else A.TC128
    assert A.block_plan(real)[0] == (64 if want == A.TC64 else 128)
    run_case(f"edge{real}", 3, 3, 130 if real < 4095 else 70, real + 1, BF, want, mask_kind="sweep" if masked else None, bound=bound)


@pytest.mark.parametrize("kind", [m for m in A.MASKS if m != "sweep"])
@pytest.mark.parametrize("Tk,want", [(290, A.TC64), (737, A.TC128)])
def test_wgmma_mask_families(Tk, want, kind):
    run_case(f"mask{Tk}", 3, 2, 70, Tk, BF, want, mask_kind=kind, bound=1.02)


# ------------------------------------------------------------------------------------------------ query edge
@pytest.mark.parametrize("Tq", [1, 127, 128, 129, 200])
@pytest.mark.parametrize("dtype,Tk,want", [(BF, 98, A.TC64), (BF, 737, A.TC128), (F32, 98, A.SPLIT)], ids=["tc64", "tc128", "split"])
def test_query_tile_edges(dtype, Tk, want, Tq):
    """a ragged last query tile writes its own rows only: the output buffer is 64 columns wider and 5 rows longer than needed"""
    run_case(f"q{Tq}", 3, 3, Tq, Tk, dtype, want, mask_kind="sweep", ldo_extra=64, guard_rows=5)


# ------------------------------------------------------------------------------------------------ arguments
def _variant_case(name):
    """(dtype, expected kernel, extra launch arguments, needs fp32_tc(False)) of a named route to a kernel"""
    return {"tc-twopass": (BF, A.TC64, {}, False), "tc-singlepass": (BF, A.TC64, {"bound": 1.02}, False),
            "tc128": (BF, A.TC128, {"bound": 1.02}, False), "split": (F32, A.SPLIT, {}, False),
            "simt-f32": (F32, A.SIMT_F32, {}, True), "simt-bf16": (BF, A.SIMT_BF16, {"ldo_extra": 4}, False)}[name]


def _run_variant(name, tag, B, H, Tq, Tk, **kw):
    dtype, want, extra, cuda_cores = _variant_case(name)
    if want == A.TC128:
        Tk = max(Tk, 737)
    if cuda_cores:
        with fp32_on_cuda_cores():
            return run_case(tag, B, H, Tq, Tk, dtype, want, **extra, **kw)
    return run_case(tag, B, H, Tq, Tk, dtype, want, **extra, **kw)


@pytest.mark.parametrize("scale", [1.0, 8.0, 32.0])
@pytest.mark.parametrize("name", ["tc-twopass", "tc-singlepass", "split", "simt-f32", "simt-bf16"])
def test_scale(name, scale):
    _run_variant(name, f"scale{scale:g}", 2, 3, 70, 161, mask_kind="random", scale=scale)


@pytest.mark.parametrize("Tk,want", [(98, A.TC64), (737, A.TC128)])
def test_logit_bound_guard(Tk, want):
    """a bound too loose for single pass (20 at scale 8: the weights would underflow and the row sum be 0) must give the two-pass result;
    4.3 is just inside the guard and still runs single pass"""
    assert not A.single_pass(8.0, 20.0) and A.single_pass(8.0, 4.3)
    two = run_case(f"bound{Tk}", 3, 3, 130, Tk, BF, want, mask_kind="sweep", bound=0.0)
    loose = run_case(f"bound{Tk}", 3, 3, 130, Tk, BF, want, mask_kind="sweep", bound=20.0)
    assert torch.equal(two.contiguous().view(torch.int16), loose.contiguous().view(torch.int16))
    run_case(f"bound{Tk}", 3, 3, 130, Tk, BF, want, mask_kind="sweep", bound=4.3)


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("name", ["tc-twopass", "tc128", "split", "simt-f32", "simt-bf16"])
def test_kv_shared_by_the_batch(name, masked):
    """kv_batch_stride_zero: one K / V per head, read by every batch entry"""
    _run_variant(name, "shared", 3, 3, 70, 98, kv_shared=True, mask_kind="sweep" if masked else None)


# ------------------------------------------------------------------------------------------------ padding rows
@pytest.mark.parametrize("pad", [0, 7, 40])
@pytest.mark.parametrize("name", ["tc-twopass", "tc-singlepass", "tc128", "split", "simt-f32", "simt-bf16"])
def test_padding_rows_do_not_reach_the_output(name, pad):
    """K / V rows [Tk, Tk_alloc) are multiplied by zero weights on the wgmma kernels and never read by the others: large finite values
    there give the bytes zeros give"""
    zero = _run_variant(name, "pad", 2, 3, 70, 98, mask_kind="random", pad=pad)
    junk = _run_variant(name, "pad", 2, 3, 70, 98, mask_kind="random", pad=pad, pad_garbage=True)
    assert torch.equal(zero.float(), junk.float())


# ------------------------------------------------------------------------------------------------ fallbacks
def test_bf16_fallback_unaligned_q():
    run_case("fb.q", 2, 3, 70, 98, BF, A.SIMT_BF16, mask_kind="random", q_offset=4)             # 8 bytes past a 16-byte boundary


def test_bf16_fallback_ldo():
    run_case("fb.ldo", 2, 3, 130, 290, BF, A.SIMT_BF16, mask_kind="sweep", ldo_extra=4)


@pytest.mark.parametrize("dtype,want", [(BF, A.SIMT_BF16), (F32, A.SIMT_F32)], ids=["bf16", "fp32"])
def test_null_key_only(dtype, want):
    """Tk = 1: the output is the null value"""
    got = run_case("fb.tk1", 2, 3, 70, 1, dtype, want)
    _, _, v = A.operands("fb.tk1", 2, 3, 70, 1, dtype == BF)
    assert torch.equal(got.float(), v.expand(-1, -1, 70, -1))


@pytest.mark.parametrize("dtype,want", [(BF, A.SIMT_BF16), (F32, A.SIMT_F32)], ids=["bf16", "fp32"])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
def test_more_keys_than_the_wgmma_kernels_take(dtype, want, masked):
    run_case("fb.4097", 2, 2, 40, 4097, dtype, want, mask_kind="sweep" if masked else None)


@pytest.mark.parametrize("Tk,kind", [(2, None), (33, "sweep"), (65, None), (290, "sweep"), (290, "only_last")])
def test_fp32_on_cuda_cores(Tk, kind):
    with fp32_on_cuda_cores():
        run_case(f"simt{Tk}", 3, 3, 130, Tk, F32, A.SIMT_F32, mask_kind=kind)
    assert ops().fp32_tc()


# ------------------------------------------------------------------------------------------------ split kernel
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("Tk", [2, 33, 64, 65, 257, 290, 1025, 4096])
def test_split_block_edges(Tk, masked):
    """the fp32 tensor-core kernel walks all Tk keys (null key included) in 64-key blocks"""
    run_case(f"split{Tk}", 3, 2, 130 if Tk < 4096 else 70, Tk, F32, A.SPLIT, mask_kind="sweep" if masked else None)


@pytest.mark.parametrize("Tk", [290, 4096])
def test_split_against_cuda_cores(Tk):
    """the two fp32 kernels on the same inputs.  The signed error shows the tensor core's truncating accumulation: the split kernel's
    outputs are low in magnitude by an amount that grows with the key count, the CUDA-core kernel's are unbiased."""
    B, H, Tq = 2, 3, 130
    q, k, v = A.operands("split.vs", B, H, Tq, Tk, False)
    mask = A.mask_of("random", "split.vs", B, Tk)
    ref, w = A.reference(q, k, v, mask, 8.0)
    out, _ = launch(q, k, v, mask, F32)
    with fp32_on_cuda_cores():
        out_cc, simt = launch(q, k, v, mask, F32)
    assert simt == 1
    view = lambda o: o.cpu().reshape(B, Tq, H, 64).transpose(1, 2).double()
    e_tc, e_cc = float((view(out) - ref).abs().max()), float((view(out_cc) - ref).abs().max())
    bias = lambda o: float((((view(o) - ref) * ref.sign()) / w).mean())
    print(f"Tk {Tk}: max |err| vs fp64: tensor-core split {e_tc:.3e}, CUDA-core fp32 {e_cc:.3e}; "
          f"mean signed err / w: split {bias(out):.3e}, CUDA-core {bias(out_cc):.3e}")
    if Tk <= 1025:                                   # the key counts of the models: the split kernel is at the CUDA-core kernel's level
        assert e_tc <= max(4 * e_cc, 2e-6), (e_tc, e_cc)
    assert A.worst_ratio(view(out), view(out_cc), 2 * A.tolerance(A.SPLIT, ref, w, 8.0, Tk)) <= 1.0


# ------------------------------------------------------------------------------------------------ argument checks
def _args(q, k, v, out, B, H, Tq, Tk, Tk_alloc, dtype, ldo, split3=0):
    a = lib().AttentionArgs()
    a.q, a.k, a.v, a.out = (None if t is None else t.data_ptr() for t in (q, k, v, out))
    a.B = B; a.heads = H; a.Tq = Tq; a.Tk = Tk; a.Tk_alloc = Tk_alloc; a.dtype = dtype; a.ldo = ldo; a.scale = 8.0; a.split3 = split3
    return a


def test_argument_errors_launch_nothing():
    L = lib()
    B, H, Tq = 1, 2, 16
    z = lambda *shape: torch.zeros(shape, dtype=BF, device="cuda")
    q, k, out = z(B * H, Tq, 64), z(B * H, 40, 64), z(B * Tq, H * 64)
    q3, k3, out3 = z(B * H * Tq, 384), z(B * H * 4104, 384), torch.zeros((B * Tq, H * 64 + 2), device="cuda")       # split operands, fp32 out
    bad = {"NULL pointer": _args(q, None, k, out, B, H, Tq, 33, 40, L.BF16, H * 64),
           "Tk_alloc < Tk": _args(q, k, k, out, B, H, Tq, 41, 40, L.BF16, H * 64),
           "split3 with 4097 keys": _args(q3, k3, k3, out3, B, H, Tq, 4097, 4104, L.BF16, H * 64, split3=1),
           "split3 with ldo % 4 != 0": _args(q3, k3, k3, out3, B, H, Tq, 33, 40, L.BF16, H * 64 + 2, split3=1)}
    before = L.launch_count()
    for a in bad.values():
        with pytest.raises(L.MMGError):
            L.call("mmg_attention", a)
    torch.cuda.synchronize()
    assert L.launch_count() == before


# ------------------------------------------------------------------------------------------------ ordering and repeatability
@pytest.mark.parametrize("n,want", [(96, A.TC64), (700, A.TC128)])
def test_attention_right_after_the_qkv_product(n, want):
    """The wgmma attention kernel is a programmatic dependent launch: issued right behind the QKV product on one stream it must read what
    that product wrote.  Three rounds with the input changed between them give the bytes of the same calls separated by a synchronise."""
    o = ops()
    b, heads, dim = 2, 3, 128
    inner, alloc = heads * 64, (n + 1 + 7) // 8 * 8
    rnd = lambda name, shape, std=1.0: A._rnd("qkv." + name, shape) * std
    w = rnd("w", (3 * inner, dim), dim ** -0.5).to(BF).cuda()
    xs = [rnd(f"x{i}", (b * n, dim)).to(BF).cuda() for i in range(2)]
    qs, ks = (1 + 0.1 * rnd("qs", (64,))).cuda(), (1 + 0.1 * rnd("ks", (64,))).cuda()
    nk, nv = rnd("nk", (heads, 64)).to(BF).cuda(), rnd("nv", (heads, 64)).to(BF).cuda()
    q = torch.zeros((b * heads, n, 64), device="cuda", dtype=BF)
    k = torch.zeros((b * heads, alloc, 64), device="cuda", dtype=BF)
    v = torch.zeros_like(k)
    e = o.qkv_epilogue(BF, heads, n, q=q, k=k, v=v, q_scale=qs, k_scale=ks, key_off=1, null_k=nk, null_v=nv)

    def rounds(separate):
        outs = []
        for x in (xs[0], xs[1], xs[0]):
            o.linear(x, w, None, epilogue=o.EPI_QKV, epi=e)
            if separate:
                torch.cuda.synchronize()
            out = torch.empty((b * n, inner), device="cuda", dtype=BF)
            o.attention(q, k, v, out, b, heads, n + 1)
            outs.append(out)
        torch.cuda.synchronize()
        return outs
    before = lib().simt_launch_count()
    if PROFILE:                                    # the product's kernel is in the capture too
        apart, names = kernels_of(lambda: rounds(True))
        assert any(want in nm for nm in names), names
    else:
        apart = rounds(True)
    together = rounds(False)
    assert lib().simt_launch_count() == before
    for i, (a, t) in enumerate(zip(apart, together)):
        assert torch.equal(a, t), f"round {i}: {int((a != t).sum())} elements differ when attention follows the product without a synchronise"
    assert not torch.equal(apart[0], apart[1]) and torch.equal(apart[0], apart[2])
    # q, k, v now hold round 2 (= round 0): the result is attention of what the product wrote
    qc = q.view(b, heads, n, 64).float().cpu()
    kc, vc = (t.view(b, heads, alloc, 64)[:, :, :n + 1].float().cpu() for t in (k, v))
    ref, wt = A.reference(qc, kc, vc, None, 8.0)
    got = apart[2].cpu().view(b, n, heads, 64).transpose(1, 2)
    assert A.worst_ratio(got, ref, A.tolerance(want, ref, wt)) <= 1.0


@pytest.mark.parametrize("Tk,want", [(290, A.TC64), (737, A.TC128)])
def test_eager_runs_and_graph_replay_are_bit_identical(Tk, want):
    B, H, Tq = 2, 3, 130
    q, k, v = A.operands("graph", B, H, Tq, Tk, True)
    mask = A.mask_of("random", "graph", B, Tk).to(torch.uint8).cuda()
    alloc = (Tk + 7) // 8 * 8
    qd = q.reshape(B * H, Tq, 64).to(BF).cuda()
    kd = torch.zeros((B * H, alloc, 64), dtype=BF, device="cuda"); kd[:, :Tk] = k.reshape(B * H, Tk, 64).to(BF).cuda()
    vd = torch.zeros_like(kd); vd[:, :Tk] = v.reshape(B * H, Tk, 64).to(BF).cuda()
    out = torch.empty((B * Tq, H * 64), dtype=BF, device="cuda")
    run = lambda: ops().attention(qd, kd, vd, out, B, H, Tk, key_mask=mask, logit_bound=1.02)
    eager = []
    for _ in range(2):
        out.fill_(FILL); run(); torch.cuda.synchronize()
        eager.append(out.clone())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    observed(run, want)
    out.fill_(FILL)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager[0], eager[1]) and torch.equal(eager[0], out)
    ref, w = A.reference(q, k, v, mask.bool().cpu(), 8.0)
    assert A.worst_ratio(out.cpu().view(B, Tq, H, 64).transpose(1, 2), ref, A.tolerance(want, ref, w)) <= 1.0


# ------------------------------------------------------------------------------------------------ which kernel ran
def test_every_case_reached_its_kernel():
    """this file again, in a fresh process, with every case under torch.profiler"""
    if PROFILE:
        pytest.skip("this is the profiling process")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-rP", "-m", "gpu", "--no-header", "-p", "no:cacheprovider"],
                       cwd=root, env=dict(os.environ, MMG_ATTENTION_PROFILE="1"), capture_output=True, text=True, timeout=900)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ report
def test_every_variant_was_reached(request):
    """per variant, softmax mode and mask: the number of cases above that reached it and the worst |err| / tol (the figures recorded in
    tests/attention_oracle.py)"""
    if request.config.getoption("keyword") or not STATS:
        pytest.skip("a report over the whole file")
    print(torch.cuda.get_device_name())
    for (variant, mode, masked), (cases, worst) in sorted(STATS.items()):
        print(f"{variant:42s} {mode:11s} {masked:8s} cases {cases:3d}  worst err / tol {worst:.3f}")
    for variant in (A.TC64, A.TC128):
        for mode in ("two-pass", "single-pass"):
            for masked in ("masked", "unmasked"):
                assert (variant, mode, masked) in STATS, (variant, mode, masked)
    for variant in (A.SPLIT, A.SIMT_BF16, A.SIMT_F32):
        for masked in ("masked", "unmasked"):
            assert (variant, "two-pass", masked) in STATS, (variant, masked)

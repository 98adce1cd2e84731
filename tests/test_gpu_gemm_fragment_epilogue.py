"""The wgmma GEMM's tile epilogues (in-place residual / LNFOLD as a TMA reduction, plain fp32 TMA store, QKV heads, GEGLU + row
statistics), which go from the accumulator fragments into 16-row output boxes: ragged last row blocks that boxes straddle, both QKV tile
widths with the null key / value row and a key offset, GEGLU statistics bit for bit, and repeatability (two eager launches and a
CUDA-graph replay give the same bytes).  Every launch is checked to stay on the wgmma kernel.  A partial last column tile cannot reach
the tile epilogues: the wgmma path needs N % 64 == 0 and takes them only at a tile width that divides N."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_kernels import close, dev, ops, rnd

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
bf = torch.bfloat16


def mm64(a, w):
    return a.double() @ w.double().t()


@contextlib.contextmanager
def on_wgmma():
    """The products launched inside run on tc_gemm_kernel: none falls back to the CUDA-core kernel."""
    from muse_maskgit_pytorch_b200 import _lib
    counts = lambda: (_lib.simt_fallback_count(), _lib.simt_launch_count())
    c0 = counts()
    yield
    torch.cuda.synchronize()
    assert counts() == c0, "a product left the wgmma kernel"


@pytest.mark.parametrize("M,N,K", [(300, 25600, 64), (2008, 4096, 512)], ids=["bn256", "bn128"])
def test_tstore_ragged_m(M, N, K):
    """Plain fp32 output (tc_gemm_kernel<256 | 128, TSTORE>) into a padded buffer: the 16-row box past M is clipped, nothing past the
    output's rows or columns is written."""
    a, w = rnd("fa", (M, K), bf), rnd("fw", (N, K), bf, std=K ** -0.5)
    buf = torch.full((M + 5, N + 8), 7.0, device="cuda")
    out = buf[:M, :N]
    with on_wgmma():
        ops().linear(dev(a, bf), dev(w, bf), out)
    ok, msg = close(out, mm64(a, w), 2e-4)
    assert ok, msg
    assert bool((buf[M:] == 7.0).all()) and bool((buf[:, N:] == 7.0).all()), "written past the output"


@pytest.mark.parametrize("M,N,K,bias", [(2008, 4096, 128, True), (16850, 512, 64, True), (16850, 512, 64, False)],
                         ids=["bn128_bias", "bn256_bias", "bn256"])
def test_residual_in_place_ragged_m(M, N, K, bias):
    """x += a W^T (+ bias) as a TMA reduction (tc_gemm_kernel<128 | 256, REDUCE>) in a padded buffer, with rows past M in the last box."""
    a, w, x = rnd("ra", (M, K), bf), rnd("rw", (N, K), bf, std=K ** -0.5), rnd("rx", (M, N))
    b = rnd("rb", (N,)) if bias else None
    buf = torch.full((M + 3, N + 8), 7.0, device="cuda")
    buf[:M, :N] = dev(x)
    xd = buf[:M, :N]
    with on_wgmma():
        ops().linear(dev(a, bf), dev(w, bf), xd, epilogue=ops().EPI_RESIDUAL, resid=xd, bias=dev(b) if bias else None)
    ref = x.double() + mm64(a, w) + (b.double() if bias else 0)
    ok, msg = close(xd, ref, 3e-4)
    assert ok, msg
    assert bool((buf[M:] == 7.0).all()) and bool((buf[:, N:] == 7.0).all()), "written past the output"


@pytest.mark.parametrize("M", [300, 16850], ids=["bn64", "bn256"])
def test_lnfold_ragged_m(M):
    """Folded LayerNorm + residual in place (tc_gemm_kernel<64 | 256, REDUCE>) on a ragged last row block: x += rstd (h W^T - mean cvec)
    with (mean, rstd) from the per-chunk statistics of each row."""
    Fu, Fp, dim, slots = 341, 384, 512, 12
    h, w = rnd("lh", (M, Fp), bf), rnd("lw", (dim, Fp), bf, std=Fu ** -0.5)
    cvec, x = rnd("lc", (dim,)), rnd("lx", (M, dim))
    g = torch.Generator().manual_seed(5)
    stats = torch.stack((torch.randn((M, slots), generator=g) * 2, torch.rand((M, slots), generator=g) * 40 + 20), -1)
    xd = dev(x)
    with on_wgmma():
        ops().linear(dev(h, bf), dev(w, bf), xd, epilogue=ops().EPI_LNFOLD_RESIDUAL, bias=dev(cvec), resid=xd, row_stats=dev(stats), ln_width=Fu)
    s = stats.double().sum(1)
    mean = s[:, 0] / Fu
    rstd = 1.0 / torch.sqrt((s[:, 1] / Fu - mean * mean).clamp_min(0) + 1e-5)
    ref = x.double() + rstd[:, None] * (mm64(h, w) - mean[:, None] * cvec.double()[None])
    ok, msg = close(xd, ref, 1e-3, 1e-3)
    assert ok, msg


@pytest.mark.parametrize("b,key_off", [(16, 2), (32, 1)], ids=["bn128", "bn256"])
def test_qkv_null_rows_key_offset(b, key_off):
    """tc_gemm_kernel<128 | 256, QKV>: every 16-token box lands on its head's rows after key_off, the null key / value goes to key
    row 0 of every (sequence, head), and rows between them and past the keys stay untouched."""
    n, heads, dim = 256, 8, 64
    x = rnd("qx", (b * n, dim), bf)
    w = rnd("qw", (3 * heads * 64, dim), bf, std=dim ** -0.5)
    qs, ks = 1 + 0.1 * rnd("qqs", (64,)), 1 + 0.1 * rnd("qks", (64,))
    nk, nv = rnd("qnk", (heads, 64), bf), rnd("qnv", (heads, 64), bf)
    kv_rows = n + key_off + 5
    q = torch.zeros((b * heads, n, 64), device="cuda", dtype=bf)
    k = torch.zeros((b * heads, kv_rows, 64), device="cuda", dtype=bf)
    v = torch.zeros_like(k)
    qsd, ksd, nkd, nvd = dev(qs), dev(ks), dev(nk, bf), dev(nv, bf)         # the epilogue block holds raw pointers: keep them alive
    e = ops().qkv_epilogue(bf, heads, n, q=q, k=k, v=v, q_scale=qsd, k_scale=ksd, key_off=key_off, null_k=nkd, null_v=nvd)
    with on_wgmma():
        ops().linear(dev(x, bf), dev(w, bf), None, epilogue=ops().EPI_QKV, epi=e)
    y = mm64(x, w).view(b, n, 3, heads, 64).permute(2, 0, 3, 1, 4)
    ok, msg = close(q.view(b, heads, n, 64), F.normalize(y[0], dim=-1) * qs.double(), 2e-2, 1e-2)
    assert ok, "q: " + msg
    kk, vv = k.view(b, heads, kv_rows, 64), v.view(b, heads, kv_rows, 64)
    ok, msg = close(kk[:, :, key_off:key_off + n], F.normalize(y[1], dim=-1) * ks.double(), 2e-2, 1e-2)
    assert ok, "k: " + msg
    ok, msg = close(vv[:, :, key_off:key_off + n], y[2], 2e-2, 1e-2)
    assert ok, "v: " + msg
    assert torch.equal(kk[:, :, 0].float().cpu(), nk.expand(b, -1, -1)) and torch.equal(vv[:, :, 0].float().cpu(), nv.expand(b, -1, -1))
    assert float(kk[:, :, 1:key_off].float().abs().sum()) == 0. and float(vv[:, :, 1:key_off].float().abs().sum()) == 0.
    assert float(kk[:, :, key_off + n:].abs().max()) == 0. and float(vv[:, :, key_off + n:].abs().max()) == 0.


def test_geglu_row_stats_bitwise():
    """tc_gemm_kernel<256, GEGLU> on a ragged last row block: the output matches fp64 torch, and each chunk's (sum, sumsq) equals, bit for
    bit, the sequential fp32 sum over the chunk's 32 bf16 outputs in ascending column order (x * x is exact in fp32 for a bf16 x, so
    sq + x * x rounds once, like the kernel's fma)."""
    M, K, F2 = 3032, 512, 1408
    a = rnd("ga", (M, K), bf)
    w1 = rnd("gw", (2 * F2, K), bf, std=K ** -0.5)
    h = torch.empty((M, F2), device="cuda", dtype=bf)
    stats = torch.full((M, F2 // 32, 2), float("nan"), device="cuda")
    with on_wgmma():
        ops().linear(dev(a, bf), dev(w1, bf), h, epilogue=ops().EPI_GEGLU, row_stats=stats)
    y = mm64(a, w1).view(M, F2 // 32, 2, 32)
    href = (y[:, :, 1] * F.gelu(y[:, :, 0])).reshape(M, F2)
    ok, msg = close(h, href, 2e-2, 1e-2)
    assert ok, msg
    hq = h.float().cpu().view(M, F2 // 32, 32)
    sx, sq = torch.zeros(M, F2 // 32), torch.zeros(M, F2 // 32)
    for i in range(32):
        t = hq[:, :, i]
        sx = sx + t
        sq = sq + t * t
    assert torch.equal(stats[..., 0].cpu(), sx) and torch.equal(stats[..., 1].cpu(), sq)


def test_tile_epilogues_repeat_and_graph_replay():
    """The four tile epilogues at the C3 decode shapes give the same bytes on two eager launches and on a CUDA-graph replay."""
    R, dim, F2, heads, n = 4096, 512, 1408, 8, 256
    g = torch.Generator(device="cuda").manual_seed(11)
    rn = lambda *s, std=1.0: (torch.randn(s, device="cuda", generator=g) * std)
    xn = rn(R, dim).to(bf)
    wqkv, wo, w1, w2 = rn(3 * dim, dim, std=dim ** -0.5).to(bf), rn(dim, dim, std=dim ** -0.5).to(bf), rn(2 * F2, dim, std=dim ** -0.5).to(bf), rn(dim, F2, std=F2 ** -0.5).to(bf)
    ws = rn(4096, dim, std=dim ** -0.5).to(bf)
    qs, ks, cvec = rn(64) + 1, rn(64) + 1, rn(dim)
    nk, nv = rn(heads, 64).to(bf), rn(heads, 64).to(bf)
    x0 = rn(R, dim)
    q = torch.empty((R // n * heads, n, 64), device="cuda", dtype=bf)
    k = torch.zeros((R // n * heads, n + 8, 64), device="cuda", dtype=bf)
    v = torch.zeros_like(k)
    h = torch.empty((R, F2), device="cuda", dtype=bf)
    stats = torch.empty((R, F2 // 32, 2), device="cuda")
    x = torch.empty_like(x0)
    s = torch.empty((R, 4096), device="cuda")
    e = ops().qkv_epilogue(bf, heads, n, q=q, k=k, v=v, q_scale=qs, k_scale=ks, key_off=1, null_k=nk, null_v=nv)

    def run():
        x.copy_(x0)
        ops().linear(xn, wqkv, None, epilogue=ops().EPI_QKV, epi=e)
        ops().linear(xn, wo, x, epilogue=ops().EPI_RESIDUAL, resid=x)
        ops().linear(xn, w1, h, epilogue=ops().EPI_GEGLU, row_stats=stats)
        ops().linear(h, w2, x, epilogue=ops().EPI_LNFOLD_RESIDUAL, bias=cvec, resid=x, row_stats=stats, ln_width=1365)
        ops().linear(xn, ws, s)

    outs = []
    for _ in range(2):
        for t in (q, k, v, h, stats, x, s):
            t.fill_(0)
        with on_wgmma():
            run()
        outs.append([t.clone() for t in (q, k, v, h, stats, x, s)])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    for t in (q, k, v, h, stats, x, s):
        t.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    outs.append([t.clone() for t in (q, k, v, h, stats, x, s)])
    for other in outs[1:]:
        for name, a_, b_ in zip("q k v h stats x s".split(), outs[0], other):
            assert torch.equal(a_.view(torch.uint8), b_.view(torch.uint8)), name

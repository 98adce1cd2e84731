"""GPU: the VAE decoder's GLU convolutions and conv-transposes on 128 x 256 tiles with tile epilogues from the accumulator fragments,
tc_gemm_kernel<256, 9 (GLU) | 10 (CONVT), __nv_bfloat16>.

Each case runs one mmg_conv2d (3x3, GLU) or mmg_conv_transpose2d (CONVT) call at a batch where pick_bn gives 256, and checks
- every output against fp64 on the exact bf16 operands, within tests/gemm_oracle.py's accumulation bound and GLU / CONVT epilogue terms;
- every output bitwise against the same images run in batches small enough that pick_bn gives 128, which runs the register epilogue
  tc_gemm_kernel<128, 0> (an output pixel depends only on its own image, and the epilogue arithmetic is the same per element).
The cases are the C3 decoder shapes (bench.py: 64 images, 16 x 16 latents, dim 256), and two small-map shapes whose M is not a multiple of
128 (a batch that is not a multiple of TB = 2 images per tile).  Between them both tile orders run for both kinds: N-fastest needs
N K 2 <= 8 MiB in 2 to 16 column tiles.  Which kernel each call ran is asserted from torch.profiler captures in a process of their own
(test_every_case_reached_its_kernel), as tests/test_gpu_dim_head128.py does."""
import os
import subprocess
import sys

import pytest
import torch

from tests import gemm_oracle as G

pytestmark = pytest.mark.gpu

PROFILE = os.environ.get("MMG_VAE_TILES_PROFILE") == "1"
REACHED = set()
BF = torch.bfloat16
GLU_T, CONVT_T, REGS128 = "tc_gemm_kernel<256, 9, __nv_bfloat16>", "tc_gemm_kernel<256, 10, __nv_bfloat16>", "tc_gemm_kernel<128, 0, __nv_bfloat16>"


def ops():
    from muse_maskgit_pytorch_b200 import ops as o
    return o


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module", autouse=True)
def _warm_up():
    """one throw-away capture: the first CUPTI session of a process pays its set-up inside the capture"""
    if PROFILE and torch.cuda.is_available():
        kernels_of(lambda: torch.ones(8, device="cuda").sum())


def kernels_of(fn):
    """(fn(), the libmmg kernels it launched) in the profiling process; (fn(), None) elsewhere"""
    if not PROFILE:
        return fn(), None
    from torch.profiler import profile, ProfilerActivity
    from muse_maskgit_pytorch_b200 import _lib
    names = []
    for _ in range(4):
        torch.cuda.synchronize()
        launched = _lib.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        launched = _lib.launch_count() - launched
        ev = [e for e in prof.key_averages() if e.self_device_time_total > 0 and "mmg::" in e.key]
        names = sorted({e.key for e in ev})
        if names and sum(e.count for e in ev) >= launched:
            break
    REACHED.update(names)
    return out, names


def assert_only(names, variant):
    """the call launched exactly one libmmg kernel, and it is `variant`"""
    if names is not None:
        assert len(names) == 1 and variant in names[0], (variant, names)


def operands(seed, shape_x, shape_w, K, n_bias):
    """bf16 x ~ N(0, 1), w ~ N(0, 1 / K) (bf16-representable), fp32 bias ~ N(0, 1 / 4), on the GPU"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape_x, generator=g, device="cuda").to(BF)
    w = (torch.randn(shape_w, generator=g, device="cuda") / K ** 0.5).to(BF)
    b = torch.randn((n_bias,), generator=g, device="cuda") * 0.5
    return x, w, b


def check_fp64(got, cols, w, kind, bias, variant):
    """got (bf16 [rows, out columns]) against the fp64 epilogue of cols @ w^T, within the oracle's bound"""
    acc, s = G.product(cols, w)
    ref, S, A = G.epilogue(kind, acc, s, {"bias": bias})
    ratio = G.worst_ratio(got, ref, G.tolerance(variant, cols.shape[1], ref, S, A, True))
    assert ratio <= 1.0, (variant, ratio)
    return ratio


def planned(m_tiles, N, variant):
    """the case's tile width restated: BN = 256 for the tile epilogue, 128 for the register one"""
    assert G.pick_bn(m_tiles, N, G.STORE, sms()) == (128 if variant == REGS128 else 256), (m_tiles, N, variant)


# ------------------------------------------------------------------------------------------------ GLU 3x3 convolutions
def glu_run(x, w, b, B, H, W, Cin, Cout):
    out = torch.full((B * H * W, Cout // 2), float("nan"), device="cuda", dtype=BF)
    _, names = kernels_of(lambda: ops().conv2d(x.view(-1, Cin), w, out, B, H, W, Cin, Cout, 1, epilogue=ops().EPI_GLU, bias=b))
    return out, names


# (B, H, W, Cin, Cout, images per register-epilogue batch): the C3 res-block GLU (K = 18432, M-fastest); 8 x 8 maps, TB = 2, an odd batch
# (M = 263 * 64, N-fastest)
GLU_CASES = {"c3": (64, 16, 16, 2048, 4096, 8), "odd_batch_8x8": (263, 8, 8, 256, 512, 131)}


@pytest.mark.parametrize("case", list(GLU_CASES))
def test_glu_tile_epilogue(case):
    B, H, W, Cin, Cout, chunk = GLU_CASES[case]
    TW, TH, TB, tx, ty = G.tile_geometry(H, W)
    planned(tx * ty * ((B + TB - 1) // TB), Cout, GLU_T)
    planned(tx * ty * ((chunk + TB - 1) // TB), Cout, REGS128)
    x, w, b = operands(list(GLU_CASES).index(case), (B, H, W, Cin), (Cout, 9 * Cin), 9 * Cin, Cout)
    out, names = glu_run(x, w, b, B, H, W, Cin, Cout)
    assert_only(names, GLU_T)
    # the register epilogue on the same images, `chunk` at a time (the last batch may be smaller)
    for b0 in range(0, B, chunk):
        n = min(chunk, B - b0)
        part, pn = glu_run(x[b0:b0 + n].contiguous(), w, b, n, H, W, Cin, Cout)
        if n == chunk:
            assert_only(pn, REGS128)
        rows = slice(b0 * H * W, (b0 + n) * H * W)
        assert torch.equal(out[rows].view(torch.int16), part.view(torch.int16)), f"images {b0}..{b0 + n - 1} differ from <128, 0>"
    if not PROFILE:
        ratio = check_fp64(out.double(), G.im2col(x.double(), 1), w, G.GLU, b, GLU_T)
        print(f"GLU {case}: worst |err| / tol {ratio:.3f}")


# ------------------------------------------------------------------------------------------------ conv-transposes (CONVT)
def convt_run(x, w, b, B, H, W, Cin, Cout):
    out = torch.full((B, 2 * H, 2 * W, Cout), float("nan"), device="cuda", dtype=BF)
    _, names = kernels_of(lambda: ops().conv_transpose2d(x, w, out, B, H, W, Cin, Cout, bias=b))
    return out, names


# (B, H, W, Cin, Cout, images per register-epilogue batch): the C3 decoder's three up-sampling conv-transposes (M-fastest, N-fastest at
# 1024 -> 512, M-fastest); 4 x 16 maps, TB = 2, an odd batch (M = 527 * 64)
CONVT_CASES = {"c3_2048to1024_16": (64, 16, 16, 2048, 1024, 16), "c3_1024to512_32": (64, 32, 32, 1024, 512, 16),
               "c3_512to256_64": (64, 64, 64, 512, 256, 8), "odd_batch_4x16": (527, 4, 16, 64, 256, 263)}


@pytest.mark.parametrize("case", list(CONVT_CASES))
def test_convt_tile_epilogue(case):
    B, H, W, Cin, Cout, chunk = CONVT_CASES[case]
    TW, TH, TB, tx, ty = G.tile_geometry(H, W)
    planned(tx * ty * ((B + TB - 1) // TB), Cout, CONVT_T)
    planned(tx * ty * ((chunk + TB - 1) // TB), Cout, REGS128)
    x, w, b = operands(100 + list(CONVT_CASES).index(case), (B, H, W, Cin), (4, Cout, 4 * Cin), 4 * Cin, Cout)
    out, names = convt_run(x, w, b, B, H, W, Cin, Cout)
    assert_only(names, CONVT_T)
    for b0 in range(0, B, chunk):
        n = min(chunk, B - b0)
        part, pn = convt_run(x[b0:b0 + n].contiguous(), w, b, n, H, W, Cin, Cout)
        if n == chunk:
            assert_only(pn, REGS128)
        assert torch.equal(out[b0:b0 + n].view(torch.int16), part.view(torch.int16)), f"images {b0}..{b0 + n - 1} differ from <128, 0>"
    if not PROFILE:
        worst = 0.0
        for py in range(2):
            for px in range(2):
                got = out[:, py::2, px::2].reshape(-1, Cout).double()
                worst = max(worst, check_fp64(got, G.convt_cols(x.double(), py, px), w[2 * py + px], G.CONVT, b, CONVT_T))
        print(f"CONVT {case}: worst |err| / tol {worst:.3f}")


# ------------------------------------------------------------------------------------------------ which kernel ran
def test_every_case_reached_its_kernel():
    """the cases of this file again, in a fresh process, each under torch.profiler"""
    if PROFILE:
        pytest.skip("this is the profiling process")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-rP", "-m", "gpu", "--no-header", "-p", "no:cacheprovider"],
                       cwd=root, env=dict(os.environ, MMG_VAE_TILES_PROFILE="1"), capture_output=True, text=True, timeout=900)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-2000:]


def test_every_new_variant_was_reached():
    """report of the profiling process: both new instantiations, and the register epilogue they are compared with, were reached"""
    if not PROFILE:
        pytest.skip("reported by the profiling process (test_every_case_reached_its_kernel)")
    missing = [v for v in (GLU_T, CONVT_T, REGS128) if not any(v in n for n in REACHED)]
    print("reached:", sorted(n.split("(")[0] for n in REACHED))
    assert not missing, missing

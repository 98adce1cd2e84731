"""CPU: the e4m3 quantiser oracle (tests/fp8_oracle.py) against torch.float8_e4m3fn, and the packer's per-row weight quantisation
(muse_maskgit.quantize_rows_e4m3) against the oracle, including the GEGLU row interleave of FF1's weight and scales."""
import numpy as np
import torch

from tests import fp8_oracle as Q


def _torch_bits(x):
    return torch.from_numpy(np.asarray(x, dtype=np.float32)).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def test_rounding_matches_torch_on_clamped_values():
    g = np.random.default_rng(0)
    x = np.concatenate([
        g.standard_normal(20000) * 100,
        g.standard_normal(20000) * 2.0 ** -7,                        # subnormal range
        np.array([0.0, -0.0, 448.0, -448.0, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -11, 2.0 ** -6, 1.0625, 1.1875, 240.0, 232.0, 1e-30]),
        (np.arange(-64, 64) + 0.5) * 2.0 ** -9,                      # ties at the subnormal spacing
        (np.arange(8, 16) + 0.5) * 0.125,                            # ties in [1, 2)
    ]).astype(np.float32)
    x = np.clip(x, -448.0, 448.0)
    assert np.array_equal(Q.e4m3_bits(x), _torch_bits(x))
    back = torch.from_numpy(Q.e4m3_bits(x)).view(torch.float8_e4m3fn).float().numpy()
    assert np.array_equal(back, Q.e4m3_round(x).astype(np.float32))


def test_satfinite_and_zero_rows():
    x = np.array([449.0, 464.0, 1e6, -500.0, -1e30], dtype=np.float32)
    assert list(Q.e4m3_bits(x)) == [0x7E, 0x7E, 0x7E, 0xFE, 0xFE]      # +-448, never NaN
    y = np.zeros((3, 64), dtype=np.float32)
    y[1, 5] = -3.0
    y[2] = np.linspace(-1, 2, 64)
    q, s = Q.quantize_rows(y)
    assert s[0] == 0 and not q[0].any()
    assert s[1] == np.float32(3.0) / np.float32(448.0) and q[1, 5] == 0xFE and not np.delete(q[1], 5).any()
    assert q[2, -1] == 0x7E and (q[2] & 0x7F).max() == 0x7E           # the row's largest |y| (2.0, last column) lands on 448


def test_packer_weight_quantiser_matches_oracle_and_geglu_permutation():
    from muse_maskgit_pytorch_b200 import muse_maskgit as MM
    g = torch.Generator().manual_seed(1)
    F, Fp, K = 90, 128, 256                                           # F not a multiple of 64: padding rows in the interleave
    w1 = torch.randn((2 * F, K), generator=g) * 0.05
    w1[3] = 0.                                                        # a zero row: scale 0, all-zero bytes
    q, s = MM.quantize_rows_e4m3(w1)
    qo, so = Q.quantize_rows(w1.numpy())
    assert np.array_equal(q.view(torch.uint8).numpy(), qo) and np.array_equal(s.numpy(), so)
    assert float(s[3]) == 0. and not q[3].view(torch.uint8).any()
    # quantising the interleaved matrix (what the packer does) == interleaving the quantised rows and their scales
    qp, sp = MM.quantize_rows_e4m3(MM._geglu_interleave(w1, Fp))
    assert torch.equal(qp.view(torch.uint8), MM._geglu_interleave(q.view(torch.uint8), Fp))
    assert torch.equal(sp, MM._geglu_interleave(s, Fp))
    # and the scales sit on the rows of their weights: unit u of the gelu arm at 64 (u // 32) + u % 32, its gate 32 rows on
    for u in (0, 31, 32, 89):
        r = 64 * (u // 32) + u % 32
        assert float(sp[r]) == float(s[u]) and float(sp[r + 32]) == float(s[F + u])
    deq = qp.float() * sp[:, None]
    assert torch.allclose(deq, MM._geglu_interleave(w1, Fp), rtol=0.07, atol=1e-6)

"""CPU oracle of the e4m3 quantiser of precision="fp8" (mmg_layernorm_fp8, the packer's per-row weight scales), in numpy.

e4m3 (OCP E4M3FN): 1 sign, 4 exponent (bias 7), 3 mantissa bits; largest finite 448, subnormals down to 2^-9, no infinities.
A row y quantises as  amax = max |y|,  inv = 448 / amax (fp32 IEEE division, 0 when amax == 0),
q = round-to-nearest-even, saturating to +-448 (cvt.rn.satfinite.e4m3) of the fp32 product y * inv,  scale = amax / 448 (fp32)."""
import numpy as np


def e4m3_round(x):
    """float32 array -> float64 array of the e4m3 values cvt.rn.satfinite gives (finite inputs)."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    a = np.abs(x)
    _, e = np.frexp(a)                                  # a = m 2^e, m in [0.5, 1): the binade of a starts at 2^(e - 1)
    step = np.ldexp(1.0, np.maximum(e - 1, -6) - 3)     # 3 mantissa bits; the subnormal spacing 2^-9 below 2^-6
    q = np.minimum(np.rint(a / step) * step, 448.0)    # np.rint: ties to even; a / step is exact (power-of-two scaling)
    return np.where(np.signbit(x), -q, q)


def e4m3_bits(x):
    """float32 array -> uint8 array of the e4m3 encodings of e4m3_round(x) (a -0 result keeps its sign bit)."""
    x = np.asarray(x, dtype=np.float32)
    q = e4m3_round(x)
    a = np.abs(q)
    _, e = np.frexp(np.where(a > 0, a, 1.0))
    ex = e - 1                                          # floor(log2 a)
    normal = (a >= 2.0 ** -6)
    exp_field = np.where(normal, ex + 7, 0)
    mant = np.where(normal, a / np.ldexp(1.0, ex - 3) - 8, a / 2.0 ** -9)
    bits = (exp_field.astype(np.int64) << 3) | np.rint(mant).astype(np.int64)
    bits = np.where(a > 0, bits, 0) | (np.signbit(x).astype(np.int64) << 7)
    return bits.astype(np.uint8)


def quantize_rows(y):
    """fp32 [rows, width] -> (uint8 e4m3 bits [rows, width], fp32 row scales [rows]) with the rounding pinned above."""
    y = np.asarray(y, dtype=np.float32)
    amax = np.abs(y).max(axis=1).astype(np.float32)
    with np.errstate(divide="ignore"):
        inv = np.where(amax > 0, np.float32(448.0) / np.where(amax > 0, amax, np.float32(1)), np.float32(0)).astype(np.float32)
    return e4m3_bits((y * inv[:, None]).astype(np.float32)), (amax / np.float32(448.0)).astype(np.float32)

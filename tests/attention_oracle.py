"""CPU oracle of mmg_attention (head dim 64, learned null key at row 0): fp64 reference, operand and mask builders with probe data, the
tolerance of each kernel variant, and a restatement of the bf16 wgmma kernel's rounding points that can carry one injected defect.
Imports no CUDA code; tests/test_attention_oracle.py runs it on the CPU and tests/test_gpu_attention.py holds the kernels to it.

Operation.  q [B, H, Tq, 64]; k, v [B or 1, H, Tk, 64] (one K / V per head shared by the batch when the leading dimension is 1); mask
[B, Tk - 1] bool, one entry per REAL key (key 0, the null key, is always live).  out = softmax(scale * q k^T, masked keys at -FLT_MAX) v.

Tolerances.  u = 2^-24; a round-to-nearest to bf16 (8 significant bits) has relative error <= 2^-8, half an ulp at the bottom of a
binade.  With p_j the softmax weights of one query row, an output element is sum_j p_j v_j and every rounding of a weight or of the
exponent's argument moves it in proportion to  w = sum_j p_j |v_j|  (>= |ref|), which `reference` returns beside the output.
  bf16 wgmma (attention_tc_kernel<64 | 128>)   |err| <= 2^-8 |ref| + C_BF16 * 2^-8 * w,  C_BF16 = 2.
      Each real key's weight is rounded to bf16 before the P V product: at most 2^-8 w in the numerator.  Masked and ragged chunks
      normalise by the sum of the rounded weights (<= 2^-8 |ref| <= 2^-8 w more), full unmasked chunks by the unrounded sum (nothing
      more).  The output is rounded to bf16 once (<= 2^-8 |ref|).  That is the bound, reached only if every rounding falls the same way
      at the bottom of its binade; the fp32 terms (64-term dot product, scale * log2e * s - max in one fma, ex2.approx at 2^-22) stay
      below 3e-4 w up to scale 32.  The roundings are unbiased: rows with many live keys sit far below the bound, rows where two or
      three keys carry the weight (the dominant-key probes) come to about half of it.
  fp32 (attention_tc_split_kernel, attention_simt_kernel<float>)   |err| <= C_F32 * 2^-17 * max(scale, 8) / 8 * w + 8 u |ref|,  C_F32 = 2.
      A weight is exp of an fp32 argument of magnitude up to 2 * scale * log2e (23 at scale 8): its rounding (23 u = 2^-19.5), the fp32
      logit (scale * a few u) and ex2.approx / expf (2^-22) give each weight a relative error near 2^-19, which enters the numerator and
      the row sum: about 2^-18 w.  The argument grows with scale, and so does the bound.  C_F32 = 2 leaves a factor 4.
  attention_tc_split_kernel adds 6 * ceil(Tk / 16) * u * w.  Its O accumulators live in the tensor core across all key blocks, and the
      tensor core's fp32 accumulation truncates where an fp32 add rounds to nearest: each of the 6 * Tk / 16 accumulating MMAs of a row
      loses up to 2 u of the accumulator, always towards zero, so the loss grows linearly with the key count instead of as its square
      root.  Measured (tests/test_gpu_attention.py::test_split_against_cuda_cores): the mean signed error, as a share of w, is -4.0e-7
      at 290 keys and -4.3e-6 at 4096 for the split kernel and 1e-9 / 1e-8 for the CUDA-core kernel; the worst element at 4096 keys is
      low by 3.4e-5 relative.  Up to the 1025 keys the models use the first bound alone holds.  The term allows u per MMA.
  bf16 CUDA-core fallback (attention_simt_kernel<__nv_bfloat16>)   the fp32 bound + 2^-8 |ref|: fp32 arithmetic on the bf16 operands and
      one rounding of the output to bf16.  The half-ulp bound is attained by some element of any large output, so the worst ratio of
      this variant is close to 1 by construction.

Observed worst |err| / tol per variant over tests/test_gpu_attention.py: OBSERVED below, on one NVIDIA H100 80GB HBM3 (driver 580.159.03,
700 W power limit).  The constants are the derived ones, not fits; the emulation below gives the wgmma figures to three digits on the CPU.

What the old rule let through.  tests/test_gpu_kernels.py::test_attention accepts |err| <= 2e-2 + 2e-2 |ref| on random unit-norm q, k and
v ~ N(0, 1).  `old_rule_accepts` replays the injected defects of `emulate_bf16` against that rule on that data (bf16; masked 200 x 290 and
256 x 33 with one entry fully masked, unmasked 256 x 257 and 1024 x 1025).  Taken over every output element the old rule rejects six of
the seven on every shape where they apply, and accepts normalise_without_null on both unmasked shapes (the null key carries 1 / Tk of the
weight there).  What that test cannot see is which kernel ran: its data never reaches either CUDA-core kernel, a 128-key block with a
ragged tail or a mask, or any argument besides the defaults.  Every one of the seven defects is rejected by the rule above on the probe
cases, with |err| / tol above 100."""
import torch
import torch.nn.functional as F

from oracle import synth

U = 2.0 ** -24
NEG_MAX = -torch.finfo(torch.float32).max
C_BF16 = 2.0
C_F32 = 2.0
LOG2E = 1.4426950408889634

TC64, TC128 = "attention_tc_kernel<64>", "attention_tc_kernel<128>"
SPLIT, SPLIT3 = "attention_tc_split_kernel", "split3_kernel"
SIMT_BF16, SIMT_F32 = "attention_simt_kernel<__nv_bfloat16>", "attention_simt_kernel<float>"

# worst |err| / tol per variant in one run of tests/test_gpu_attention.py (card and driver in the module docstring); a record, not a limit
OBSERVED = {TC64: 0.504, TC128: 0.491, SPLIT: 0.297, SIMT_F32: 0.243, SIMT_BF16: 0.989}

DEFECTS = ("drop_last_key", "mask_shift_by_one", "mask_row_of_wrong_batch", "no_null_key", "tail_block_skipped", "normalise_without_null",
           "v_of_next_head")


# ------------------------------------------------------------------------------------------------ dispatch, restated
def block_plan(real_keys):
    """(KB, blocks, KB_tail) of the wgmma kernel over `real_keys` = Tk - 1 keys: 64-key blocks up to 640 keys, 128-key blocks above; the
    last block holds the remainder rounded up to 32 keys."""
    kb = 64 if real_keys <= 640 else 128
    full, rem = divmod(real_keys, kb)
    return (kb, full, kb) if rem == 0 else (kb, full + 1, (rem + 31) // 32 * 32)


def single_pass(scale, logit_bound):
    """the guard of the single-pass softmax: exp2((s - bound) * scale * log2e) must stay inside the fp32 range for |s| <= bound"""
    return logit_bound > 0 and scale > 0 and 2.0 * logit_bound * scale * LOG2E < 100.0


def probe_keys(Tk):
    """key rows (0 = null) a dominant-key probe is placed on: the null key, the first and last real key, the first key of the tail block
    and the key before it, the first key of the second block and the last key of the first"""
    if Tk < 2:
        return [0]
    kb, nb, _ = block_plan(Tk - 1)
    want = [0, 1, Tk - 1, 1 + (nb - 1) * kb, (nb - 1) * kb, 1 + kb, kb, 33, 32]
    out = []
    for j in want:
        if 0 <= j < Tk and j not in out:
            out.append(j)
    return out


# ------------------------------------------------------------------------------------------------ operands
def _rnd(tag, shape, seed=11):
    return torch.from_numpy(synth.normal(tag, shape, seed))


def operands(tag, B, H, Tq, Tk, bf16, kv_shared=False, probe=True):
    """fp32 q [B, H, Tq, 64], k, v [B or 1, H, Tk, 64]: unit-norm q and k, v ~ N(0, 1); bf16-representable when `bf16`.
    With `probe`: V row j carries +16 in column j % 64 (a dropped, shifted or duplicated key moves the output far beyond tolerance), and
    query rows i and Tq - 1 - i equal key probe_keys(Tk)[i], so that key carries most of the row's weight."""
    Bk = 1 if kv_shared else B
    q = F.normalize(_rnd(tag + ".q", (B, H, Tq, 64)), dim=-1)
    k = F.normalize(_rnd(tag + ".k", (Bk, H, Tk, 64)), dim=-1)
    v = _rnd(tag + ".v", (Bk, H, Tk, 64))
    if probe:
        j = torch.arange(Tk)
        v[:, :, j, j % 64] += 16.0
    if bf16:
        q, k, v = (t.to(torch.bfloat16).float() for t in (q, k, v))
    if probe:
        for i, key in enumerate(probe_keys(Tk)):
            for row in {i, Tq - 1 - i}:
                if 0 <= row < Tq:
                    q[:, :, row] = k[:, :, key]
    return q, k, v


MASKS = ("random", "first_entry_dead", "only_last", "only_first", "chunk_dead", "per_entry", "sweep")


def mask_of(kind, tag, B, Tk):
    """[B, Tk - 1] bool (True = attend) or None."""
    Tr = Tk - 1
    if kind is None or kind == "none" or Tr == 0:
        return None
    u = torch.from_numpy(synth.uniform(tag + ".m", (B, Tr), 11))
    m = u > 0.4
    if kind == "random":
        m[-1, 0] = m[-1, -1] = True                 # the first and the last real key are live somewhere
    elif kind == "first_entry_dead":
        m[0] = False
    elif kind == "only_last":
        m[:] = False; m[:, -1] = True
    elif kind == "only_first":
        m[:] = False; m[:, 0] = True
    elif kind == "chunk_dead":                      # a whole 32-key chunk dead inside a live block (the second chunk where there is one)
        m[:] = True
        lo = 32 if Tr >= 64 else 0
        m[:, lo:lo + 32] = False
    elif kind == "per_entry":                       # a different density for every batch entry
        m = u > torch.linspace(0.1, 0.9, B)[:, None]
    elif kind == "sweep":                           # entry 0 fully masked, entry 1 random, entry 2 a dead chunk in a random mask, ...
        m[0] = False
        if B > 2:
            lo = 32 if Tr >= 64 else 0
            m[2, lo:lo + 32] = False
            m[2, -1] = True
    else:
        raise ValueError(kind)
    return m


# ------------------------------------------------------------------------------------------------ reference and tolerance
def reference(q, k, v, mask, scale):
    """fp64 attention on the exact operand values.  Returns (out [B, H, Tq, 64], w = sum_j p_j |v_j| of the same shape)."""
    qd, kd, vd = q.double(), k.double(), v.double()
    sim = (qd @ kd.transpose(-1, -2)) * float(scale)                       # [B, H, Tq, Tk], k broadcast over the batch when shared
    if mask is not None:
        live = F.pad(mask, (1, 0), value=True)[:, None, None, :]
        sim = sim.masked_fill(~live, NEG_MAX)
    p = sim.softmax(-1)
    return p @ vd, p @ vd.abs()


def tolerance(variant, ref, w, scale=8.0, keys=0):
    """elementwise bound on |got - ref| for a kernel variant; `keys` = Tk (the split kernel's bound grows with it)"""
    fp32 = C_F32 * 2.0 ** -17 * max(float(scale), 8.0) / 8.0 * w + 8 * U * ref.abs()
    if variant in (TC64, TC128):
        return 2.0 ** -8 * ref.abs() + C_BF16 * 2.0 ** -8 * w
    if variant == SIMT_BF16:
        return fp32 + 2.0 ** -8 * ref.abs()
    if variant == SPLIT:
        return fp32 + 6 * ((keys + 15) // 16) * U * w
    if variant == SIMT_F32:
        return fp32
    raise ValueError(variant)


def old_tolerance(ref):
    return 2e-2 + 2e-2 * ref.abs()


def worst_ratio(got, ref, tol):
    """max |got - ref| / tol; inf where got is not finite"""
    got = got.double()
    r = (got - ref).abs() / tol
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
    return float(r.max())


def merge_heads(x):
    """[B, H, Tq, 64] -> [B * Tq, H * 64], the layout mmg_attention writes"""
    B, H, Tq, _ = x.shape
    return x.transpose(1, 2).reshape(B * Tq, H * 64)


# ------------------------------------------------------------------------------------------------ the wgmma kernel's arithmetic
def emulate_bf16(q, k, v, mask, scale, *, logit_bound=0.0, defect=None):
    """The rounding points of attention_tc_kernel on bf16-representable operands, in torch on the CPU: fp32 logits, weights
    exp2(s * scale*log2e - max * scale*log2e) in fp32 (max = the row maximum over live keys, or logit_bound in single pass), real-key weights
    rounded to bf16 for the P V product, fp32 accumulation, the null key's weight and value added unrounded, normalisation by the unrounded
    sum on full unmasked 32-key chunks and by the rounded sum elsewhere, output rounded to bf16.  Returns fp32 [B, H, Tq, 64] holding bf16
    values.  `defect` (one of DEFECTS) plants one indexing or normalisation error of the kind the kernel could have."""
    assert defect is None or defect in DEFECTS, defect
    B, H, Tq, _ = q.shape
    Tk, Tr = k.shape[2], k.shape[2] - 1
    k, v = k.expand(B, -1, -1, -1), v.expand(B, -1, -1, -1)
    if defect == "v_of_next_head":
        v = v.reshape(B * H, Tk, 64).roll(-1, 0).reshape(B, H, Tk, 64)
    live = torch.ones((B, H, Tk), dtype=torch.bool)
    if mask is not None:
        m = mask
        if defect == "mask_shift_by_one":                                   # byte j + 1 of the flat mask read for key j
            flat = torch.cat((mask.reshape(-1), torch.ones(1, dtype=torch.bool)))
            m = flat[1:].reshape(B, Tr)
        m = m[:, None, :].expand(B, H, Tr)
        if defect == "mask_row_of_wrong_batch":                             # row (b * heads + h) % B instead of b
            rows = (torch.arange(B * H) % B).reshape(B, H)
            m = mask[rows]
        live = torch.cat((torch.ones((B, H, 1), dtype=torch.bool), m), -1)
    if defect == "drop_last_key" and Tr > 0:
        live = live.clone(); live[..., -1] = False
    if defect == "tail_block_skipped" and Tr > 0:
        kb, nb, _ = block_plan(Tr)
        live = live.clone(); live[..., 1 + (nb - 1) * kb:] = False
    live = live[:, :, None, :]                                              # [B, H, 1, Tk]
    sl = torch.tensor(float(scale) * LOG2E, dtype=torch.float32)
    s = q.float() @ k.float().transpose(-1, -2)                             # fp32 accumulation of exact bf16 products
    if single_pass(scale, logit_bound):
        mx = torch.full((B, H, Tq, 1), float(logit_bound), dtype=torch.float32)
    else:
        mx = s.masked_fill(~live, -float("inf")).amax(-1, keepdim=True)
    p = torch.exp2(s * sl - mx * sl)
    p = torch.where(live, p, torch.zeros_like(p))
    p_null, p_real = p[..., :1], p[..., 1:]
    p_bf = p_real.to(torch.bfloat16).float()
    # chunks of 32 real keys: unmasked chunks that end inside the key range sum the unrounded weights
    fast = torch.zeros(Tr, dtype=torch.bool)
    if mask is None:
        fast[:Tr // 32 * 32] = True
    den = torch.where(fast, p_real, p_bf).sum(-1, keepdim=True)
    if defect == "no_null_key":
        p_null = torch.zeros_like(p_null)
    if defect != "normalise_without_null":
        den = den + p_null
    num = p_bf @ v[:, :, 1:].float() + p_null * v[:, :, :1].float()
    return (num / den).to(torch.bfloat16).float()


def old_rule_accepts():
    """{case: {defect: accepted by 2e-2 + 2e-2 |ref| on the random data test_attention used}} for the two bf16 shapes named in the module
    docstring; a report, recomputed by tests/test_attention_oracle.py"""
    out = {}
    for name, B, Tq, Tk, kind in (("masked 200x290", 2, 200, 290, "first_entry_dead"), ("masked 256x33", 2, 256, 33, "first_entry_dead"),
                                  ("unmasked 256x257", 2, 256, 257, None), ("unmasked 1024x1025", 1, 1024, 1025, None)):
        q, k, v = operands("old." + name, B, 2, Tq, Tk, True, probe=False)
        mask = mask_of(kind, "old." + name, B, Tk)
        ref, _ = reference(q, k, v, mask, 8.0)
        out[name] = {d: worst_ratio(emulate_bf16(q, k, v, mask, 8.0, defect=d), ref, old_tolerance(ref)) <= 1.0
                     for d in DEFECTS if mask is not None or not d.startswith("mask_")}
    return out

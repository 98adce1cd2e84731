"""TEST INFRASTRUCTURE (imported only by tests/): the selection logic of libmmg's fused logits + sampling tail restated in numpy, to show on
the CPU that it returns exactly what the reference's  argmax(top_k(logits) / T + gumbel(u))  returns (muse_maskgit_pytorch.py:403-418, 576-582).

The fused path (csrc/mmg_logits_fused.cu) never forms a row's V logits.  It keeps (a) every logit >= a per-row threshold t chosen from a
4096-column sample so that about k + 4 sigma logits pass (the CANDIDATES: a superset of the exact top-k whenever at least k pass) and (b) the
row's softmax statistics.  The finisher then
  pass 1: perturbs every candidate that has not been excluded, p_v = x_v / T + g_v (g_v a pure function of (row, v)), takes the argmax
          (ties -> lowest vocabulary index);
  pass 2: counts the candidates that beat the winner's LOGIT (x > x_w, or x == x_w with a lower index) = its exact rank in the whole row,
          because every logit above x_w is >= t and therefore in the list;
  rank < k -> done; else the winner lies between t and the true k-th value: exclude it and repeat pass 1.
torch.topk's choice among logits equal to the k-th value is unspecified; libmmg keeps the lowest vocabulary indices (DESIGN.md 4).

The second half restates the host planner of mmg_logits_fused (lf_plan / lf_carve / lf_supported): which split count S and per-segment
list capacity a call with R rows gets on a device with `units` SMs, and the workspace bytes.  tests/test_abi.py pins it to the library's
own workspace query; the GPU tests use it to pick row counts that reach a given plan on the card at hand, and `fused_leg` to predict,
from exact logits, which leg (candidate lists or materialised fallback) a row takes."""
import math
import numpy as np

LF_BM = LF_BN = 128            # logits GEMM tile
LF_SEGS = 2                    # list segments per (row, split): the two 64-column halves of every tile
LF_FIFO = 32                   # per-thread shared-memory FIFO entries: more than LF_FIFO - 3 candidates in one 64-column chunk overflow it
LF_MAX_SPLITS = 64
LF_FB_CAP = 128                # rows per call that may take the in-call materialised fallback
SMP_SAMPLE, SMP_CAP = 4096, 9216


def lf_plan(R, V, units):
    """(S, npt, cap, stride, ns, num_m_tiles) of a call with R rows: the smallest power-of-two split count whose static-schedule makespan
    is within 4 % of the best, npt = 128-column tiles per split, cap = list entries per (row, split, half), the sample stride / size."""
    num_pm = (R + LF_BM - 1) // LF_BM
    NT = V // LF_BN
    splits = []
    s = 1
    while s <= LF_MAX_SPLITS and s <= NT:
        if NT % s or (s > 1 and NT // s < 2):
            break
        splits.append(s)
        s *= 2
    span = lambda s: ((num_pm * s + units - 1) // units) * (NT // s)
    best = min(span(s) for s in splits)
    S = next(s for s in splits if span(s) * 100 <= best * 104)
    npt = NT // S
    per = SMP_CAP / (LF_SEGS * S)
    cap = min(int(per + 6.0 * math.sqrt(per) + 8.0), 64 * npt)
    stride = V // SMP_SAMPLE if V > SMP_SAMPLE else 1
    return dict(S=S, npt=npt, cap=(cap + 3) // 4 * 4, stride=stride, ns=V // stride, num_m_tiles=num_pm)


def rows_for_plan(V, S, units, ragged=77, lo=1, hi=40000):
    """The smallest row count in [lo, hi] that is `ragged` rows past a multiple of 128 (a partial last M-tile) and gets S splits; None if
    no such count exists on `units` SMs."""
    for R in range(lo + (ragged - lo) % LF_BM, hi + 1, LF_BM):
        if lf_plan(R, V, units)["S"] == S:
            return R
    return None


def lf_supported(V, K, k):
    if V < 1024 or V % 256 or K % 64 or K < 64 or k < 1 or k > V:
        return False
    if V > SMP_SAMPLE and V % SMP_SAMPLE:
        return False
    stride = V // SMP_SAMPLE if V > SMP_SAMPLE else 1
    ns = V // stride
    if ns == V:
        return k + 64 <= SMP_CAP
    pf = k / V
    mu = pf * ns
    rs = mu + 4.0 * math.sqrt(mu * (1 - pf)) + 2.0
    return rs * stride + 4.0 * stride * math.sqrt(mu * (1 - pf)) <= SMP_CAP


def workspace_bytes(R_max, V, K, k, units):
    """mmg_logits_fused_workspace_bytes: parts and lists are sized for the largest of every row count up to R_max (S shrinks as R grows)."""
    if R_max <= 0 or not lf_supported(V, K, k):
        return 0
    up = lambda x: (x + 255) // 256 * 256
    parts = lists = 0
    R = LF_BM
    while True:
        Rc = min(R, R_max)
        pl = lf_plan(Rc, V, units)
        parts = max(parts, Rc * pl["S"] * LF_SEGS * 16)
        lists = max(lists, Rc * pl["S"] * LF_SEGS * pl["cap"] * 8)
        if R >= R_max:
            break
        R += LF_BM
    ns = lf_plan(1, V, units)["ns"]
    return (up(R_max * ns * 4) + up(R_max * 4) + up(parts) + up(lists) + 256 + up(LF_FB_CAP * 4) + up(LF_FB_CAP * K * 2)
            + up(LF_FB_CAP * V * 4))


def sampled_threshold(x, V, k):
    """The candidate threshold of one row of fp32 logits x: the exact k-th largest value when V <= 4096, else the fp16-rounded sample
    value whose rank among the every-`stride`-th columns is rs = mu + 4 sigma + 2 (fp32 arithmetic, as the threshold kernel)."""
    x = np.asarray(x, dtype=np.float32)
    if V <= SMP_SAMPLE:
        return np.sort(x)[::-1][k - 1]
    stride = V // SMP_SAMPLE
    smp = np.sort(x[::stride].astype(np.float16).astype(np.float32))[::-1]
    pf = np.float32(k) / np.float32(V)
    mu = pf * np.float32(SMP_SAMPLE)
    rs = int(mu + np.float32(4.0) * np.sqrt(mu * (np.float32(1.0) - pf)) + np.float32(2.0))
    return smp[rs - 1]


def fused_leg(x, V, k, plan):
    """Which leg mmg_logits_fused sends a row of exact fp32 logits down, before the finisher's exclusion loop: 'lists', or the fallback
    reason 'threshold' (fewer than k candidates), 'fifo' (more than LF_FIFO - 3 candidates in one 64-column chunk) or 'segment' (more
    candidates in one (split, half) segment than its list capacity)."""
    x = np.asarray(x, dtype=np.float32)
    t = sampled_threshold(x, V, k)
    cand = (x >= t).reshape(plan["S"], plan["npt"], LF_SEGS, 64).sum(-1)          # [split, tile, half] candidates per chunk
    if (cand > LF_FIFO - 3).any():
        return "fifo"
    if (cand.sum(1) > plan["cap"]).any():
        return "segment"
    if int(cand.sum()) < k:
        return "threshold"
    return "lists"


def reference_choice(logits, gumbel, k, temperature):
    """argmax over the top-k set (k largest logits, ties at the k-th value -> lowest indices) of logits / T + gumbel; ties -> lowest index."""
    order = np.lexsort((np.arange(logits.size), -logits.astype(np.float64)))          # by logit descending, then index ascending
    keep = order[:k]
    p = logits[keep].astype(np.float32) / np.float32(max(temperature, 1e-10)) + gumbel[keep].astype(np.float32)
    best = np.lexsort((keep, -p.astype(np.float64)))[0]
    return int(keep[best])


def fused_choice(logits, gumbel, k, temperature, threshold, max_excl=24):
    """The finisher's procedure on the candidate list {v : logits[v] >= threshold}.  Returns (token, passes) or (None, passes) when the list
    is too short (the kernel then sends the row through the materialised path)."""
    idx = np.nonzero(logits >= threshold)[0]
    if idx.size < k:
        return None, 0
    x = logits[idx].astype(np.float32)
    p = x / np.float32(max(temperature, 1e-10)) + gumbel[idx].astype(np.float32)
    excluded = np.zeros(idx.size, dtype=bool)
    for n_pass in range(1, max_excl + 2):
        live = np.nonzero(~excluded)[0]
        w = live[np.lexsort((idx[live], -p[live].astype(np.float64)))[0]]               # pass 1
        rank = int(np.sum((x > x[w]) | ((x == x[w]) & (idx < idx[w]))))                 # pass 2
        if rank < k:
            return int(idx[w]), n_pass
        excluded[w] = True
    return None, max_excl + 1

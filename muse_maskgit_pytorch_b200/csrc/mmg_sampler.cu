// Sampler kernels for MaskGit.generate(): re-mask and the fused top-k / gumbel-argmax / confidence tail.
//
// mmg_logits_sample reads every logits row from HBM exactly once (the algorithmic minimum once logits are
// materialised: 4 B / logit).  Per row (one 512-thread CTA):
//   A. a 4096-element strided sample (128 lines of 128 B) gives a provisional threshold t_lo whose expected
//      exceedance count is ~k + 4.5 sigma;
//   B. one streaming pass (128-bit loads, L1 no-allocate): online softmax statistics (max, sum exp) and the
//      candidates {x >= t_lo} appended to a shared-memory list with one atomic per warp-iteration;
//   C. on the list only (~1.2 k entries): gumbel noise (2 logs per candidate instead of per logit), block argmax of
//      the perturbed value, accepted iff the candidate's exact rank (#greater + #equal-with-lower-index) is < k,
//      else excluded and repeated.  This equals argmax over torch.topk's kept set without ever forming the set.
//   If the list would miss the top-k (count < k) or overflow, an exact bitwise radix descent over the L2-resident
//   row finds the k-th largest key and the list is rebuilt (rare; exercised by the tests with adversarial rows).
#include "mmg_sampler.cuh"

namespace mmg {

// MODE: the noise stream (RowNoise in mmg_sampler.cuh)
template <int MODE>
__global__ void __launch_bounds__(SMP_THREADS)
logits_sample_kernel(const mmg_logits_sample_args a, float tdiv) {
  extern __shared__ uint8_t smraw[];
  float* lval = reinterpret_cast<float*>(smraw);                 // [SMP_CAP] candidate logits
  int* lidx = reinterpret_cast<int*>(lval + SMP_CAP);            // [SMP_CAP] candidate vocabulary indices
  float4* scr = reinterpret_cast<float4*>(lidx + SMP_CAP);       // [4][SMP_THREADS] per-thread staging of the 16 values in flight
  __shared__ int s_count, s_n, s_k;
  __shared__ SampleScratch sc;
  __shared__ float s_max, s_sum;

  pdl_wait(); pdl_trigger();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int V = a.V;
  int64_t r = blockIdx.x;
  const float* row = a.logits + r * (int64_t)V;
  if (a.row_index) {                                  // fallback leg of mmg_logits_fused: logits row j belongs to sampled row row_index[j]
    if ((int)blockIdx.x >= *a.row_count_dev) return;
    r = a.row_index[blockIdx.x];
  }
  const int b = (int)(r / a.num_masked);
  const int pos = a.masked_pos[r];

  // ---------------- phase A: sample (registers) -> provisional threshold ----------------
  const int ns = V < SMP_SAMPLE ? V : SMP_SAMPLE;
  constexpr int SPT = SMP_SAMPLE / SMP_THREADS;                  // sample keys per thread
  uint32_t sk[SPT];
  {
    const int nlines = ns / 32, vlines = V / 32;                 // 128-byte lines spread evenly over the row
#pragma unroll
    for (int j = 0; j < SPT; ++j) {
      const int i = tid + j * SMP_THREADS;
      uint32_t key = 0;                                          // key 0 sorts below every real value
      if (i < ns) {
        const int src = (ns == V) ? i : (int)(((int64_t)(i >> 5) * vlines) / nlines) * 32 + (i & 31);
        key = fkey(row[src]);
      }
      sk[j] = key;
    }
  }
  // the row's own k (per-image table): parked in shared memory across phase B, where a register holding it made MODE 0 spill.  A count
  // above the list capacity belongs to the row-walking kernel's route (mmg.h); clamped, it cannot make the exact rebuild write past the list.
  if (tid == 0) { s_count = 0; s_k = min(image_k(a, b), SMP_CAP); }
  const float tlo = sample_threshold(sk, ns, V, image_k(a, b), sc, warp, lane);
  const bool degenerate = (tlo == -FLT_MAX);                         // no usable threshold: every element is a candidate (-> exact rebuild)

  // ---------------- phase B: one streaming pass over the row ----------------
  constexpr float LOG2E = 1.4426950408889634f;
  constexpr float NEG_BIG = -1e30f;                                // "minus infinity" that stays finite after * log2e
  float m_t = NEG_BIG, s_t = 0.f;                                  // running max and sum of 2^((x - m) * log2e)
  if ((V & 3) == 0 && ((reinterpret_cast<uintptr_t>(row) & 15) == 0)) {
    const float4* r4 = reinterpret_cast<const float4*>(row);
    const int n4 = V >> 2;
    constexpr int UNR = 4;                                          // 4 independent 128-bit loads per thread and group
    constexpr int GRP = SMP_THREADS * UNR;                          // float4s per group (16 elements per thread)
    // one group of 16 elements per thread: load (the whole group in range: no padding moves) ...
    auto load_group = [&](float4 (&g)[UNR], int i0) {
      if (i0 + GRP <= n4) {
#pragma unroll
        for (int u = 0; u < UNR; ++u) g[u] = ld_stream4(r4 + i0 + u * SMP_THREADS + tid);
      } else {
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          const int i = i0 + u * SMP_THREADS + tid;
          g[u] = make_float4(NEG_BIG, NEG_BIG, NEG_BIG, NEG_BIG);
          if (i < n4) g[u] = ld_stream4(r4 + i);
        }
      }
    };
    // ... and consume: online softmax statistics + append the elements >= tlo to the candidate list
    auto consume_group = [&](const float4 (&g)[UNR], int i0) {
      const float xs[UNR * 4] = {g[0].x, g[0].y, g[0].z, g[0].w, g[1].x, g[1].y, g[1].z, g[1].w,
                                 g[2].x, g[2].y, g[2].z, g[2].w, g[3].x, g[3].y, g[3].z, g[3].w};
      const bool full = i0 + GRP <= n4;                              // block-uniform: every thread's 16 elements are in range
      const bool has = full || (i0 + tid) < n4;                      // a thread with no element must not touch the statistics:
      float lm = xs[0];                                              // fma(-1e30, log2e, -fl(-1e30 * log2e)) is a huge rounding residue
#pragma unroll
      for (int j = 1; j < UNR * 4; ++j) lm = fmaxf(lm, xs[j]);
      if (has && lm > m_t) { s_t *= ex2_approx((m_t - lm) * LOG2E); m_t = lm; }
      const float mb = m_t * LOG2E;
      unsigned mask = 0;                                             // bit j: element j of this thread is a top-k candidate
      if (has) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int j = 0; j < UNR * 4; j += 2) {                       // padding lanes hold -1e30: 2^-huge = 0, never >= tlo
          s0 += ex2_approx(fmaf(xs[j], LOG2E, -mb)); s1 += ex2_approx(fmaf(xs[j + 1], LOG2E, -mb));
          mask |= (xs[j] >= tlo ? 1u : 0u) << j; mask |= (xs[j + 1] >= tlo ? 1u : 0u) << (j + 1);
        }
        s_t += s0 + s1;
        if (degenerate) {                                            // no usable threshold: everything in range is a candidate
          mask = 0;
#pragma unroll
          for (int u = 0; u < UNR; ++u) if (i0 + u * SMP_THREADS + tid < n4) mask |= 0xFu << (4 * u);
        }
      }
      // warp-aggregated append (one shared-memory atomic per warp per 16 elements per thread); the values pass through a
      // per-thread shared-memory staging row so the set bits can be walked without dynamic register indexing
      const int c = __popc(mask);
      if (mask) {
#pragma unroll
        for (int u = 0; u < UNR; ++u) scr[u * SMP_THREADS + tid] = g[u];
      }
      int incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      const int tot = __shfl_sync(0xffffffffu, incl, 31);
      if (tot) {
        int start = 0;
        if (lane == 0) start = atomicAdd(&s_count, tot);
        start = __shfl_sync(0xffffffffu, start, 0) + incl - c;
        while (mask) {
          const int j = __ffs(mask) - 1; mask &= mask - 1;
          if (start < SMP_CAP) {
            lidx[start] = (i0 + (j >> 2) * SMP_THREADS + tid) * 4 + (j & 3);
            lval[start] = reinterpret_cast<const float*>(scr + (j >> 2) * SMP_THREADS + tid)[j & 3];
          }
          ++start;
        }
      }
    };
    // two register groups in ping-pong: the loads of one are in flight while the other is consumed (no register copies)
    float4 ga[UNR], gb[UNR];
    load_group(ga, 0);
    for (int i0 = 0; i0 < n4; i0 += 2 * GRP) {
      const bool second = i0 + GRP < n4;                            // block-uniform
      if (second) load_group(gb, i0 + GRP);
      consume_group(ga, i0);
      if (i0 + 2 * GRP < n4) load_group(ga, i0 + 2 * GRP);
      if (second) consume_group(gb, i0 + GRP);
    }
  } else {
    for (int i0 = 0; i0 < V; i0 += SMP_THREADS) {
      const int i = i0 + tid;
      float x = NEG_BIG; int c = 0;
      if (i < V) {
        x = ld_stream(row + i);
        if (x > m_t) { s_t *= ex2_approx((m_t - x) * LOG2E); m_t = x; }
        s_t += ex2_approx((x - m_t) * LOG2E);
        c = (x >= tlo) | degenerate;
      }
      int incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      const int tot = __shfl_sync(0xffffffffu, incl, 31);
      if (tot) {
        int start = 0;
        if (lane == 0) start = atomicAdd(&s_count, tot);
        start = __shfl_sync(0xffffffffu, start, 0) + incl - c;
        if (c && start < SMP_CAP) { lidx[start] = i; lval[start] = x; }
      }
    }
  }
  // block softmax statistics
  {
    float m = warp_max(m_t);
    __syncthreads();
    if (lane == 0) sc.redf[warp] = m;
    __syncthreads();
    float M = sc.redf[lane % (SMP_THREADS / 32)];
    M = warp_max(M);
    float sm = s_t * ex2_approx((m_t - M) * LOG2E);
    sm = warp_sum(sm);
    __syncthreads();
    if (lane == 0) sc.redf[warp] = sm;
    __syncthreads();
    if (tid == 0) { float t = 0.f; for (int w = 0; w < SMP_THREADS / 32; ++w) t += sc.redf[w]; s_sum = t; s_max = M; s_n = s_count; }
    __syncthreads();
  }
  int n = s_n;
  const int k = s_k;

  // ---------------- rare: exact rebuild when the sample threshold missed ----------------
  if (n < k || n > SMP_CAP) {
    uint32_t prefix = 0;                       // k-th largest key of the row by bitwise descent (row is L2 resident now)
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = prefix | (1u << bit);
      int c = 0;
      for (int i = tid; i < V; i += SMP_THREADS) c += (fkey(row[i]) >= cand);
      int tot, dummy;
      block_sum2(c, 0, sc.red, warp, lane, tot, dummy);
      if (tot >= k) prefix = cand;
    }
    // list = all keys > prefix (fewer than k of them), then ties (== prefix) in index order until k entries
    __syncthreads();
    if (tid == 0) s_count = 0;
    __syncthreads();
    for (int i0 = 0; i0 < V; i0 += SMP_THREADS) {
      const int i = i0 + tid;
      const float x = i < V ? row[i] : 0.f;
      const bool in = i < V && fkey(x) > prefix;
      const unsigned bal = __ballot_sync(0xffffffffu, in);
      int start = 0;
      if (lane == 0 && bal) start = atomicAdd(&s_count, __popc(bal));
      start = __shfl_sync(0xffffffffu, start, 0) + __popc(bal & ((1u << lane) - 1));
      if (in) { lval[start] = x; lidx[start] = i; }
    }
    __syncthreads();
    if (warp == 0) {             // ties, serial in index order (one warp), lowest indices first
      int cnt = s_count;
      for (int i0 = 0; i0 < V && cnt < k; i0 += 32) {
        const int i = i0 + lane;
        const float x = i < V ? row[i] : 0.f;
        const bool tie = i < V && fkey(x) == prefix;
        const unsigned bal = __ballot_sync(0xffffffffu, tie);
        const int slot = cnt + __popc(bal & ((1u << lane) - 1));
        if (tie && slot < k) { lval[slot] = x; lidx[slot] = i; }
        cnt += __popc(bal);
      }
      if (lane == 0) s_n = cnt < k ? cnt : k;
    }
    __syncthreads();
    n = s_n;
  }

  // ---------------- phase C: perturbed argmax restricted to the exact top-k ----------------
  int win_v; float win_x;
  sample_from_list(row_noise<MODE>(a, b, pos, V, tdiv), lval, lidx, n, k, sc, tid, warp, lane, win_v, win_x);
  if (tid == 0) {
    if (win_v < 0) { win_v = 0; win_x = row[0]; }                 // degenerate rows (all -inf / NaN)
    write_sample(a, b, pos, win_v, expf(win_x - s_max) / s_sum);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Any top-k threshold (k > SMP_CAP: topk_filter_thres below ~0.86 at V = 65536; muse_maskgit_pytorch.py:413-418 takes any value):
// the kept set no longer fits a shared-memory list, so the row (256 KB, L2 resident after the first touch) is walked instead:
//   1. exact k-th largest key by a bitwise descent over the whole row (32 counting passes);
//   2. one more pass: online softmax statistics + the perturbed value of every kept element ( > k-th, plus the first k - #greater
//      elements EQUAL to it in index order, as torch.topk keeps exactly k ) -> per-thread best -> block argmax.
// ~35 passes over the row: a correctness path for unusual thresholds, not a fast one.
// ---------------------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(SMP_THREADS)
logits_sample_bigk_kernel(const mmg_logits_sample_args a, float tdiv) {
  __shared__ SampleScratch sc;
  __shared__ int s_cut;
  __shared__ float s_m, s_s;
  __shared__ RowNoise<MODE> s_noise;
  pdl_wait(); pdl_trigger();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int V = a.V;
  int64_t r = blockIdx.x;
  const float* row = a.logits + r * (int64_t)V;
  if (a.row_index) { if ((int)blockIdx.x >= *a.row_count_dev) return; r = a.row_index[blockIdx.x]; }
  const int b = (int)(r / a.num_masked);
  const int pos = a.masked_pos[r];
  const int k = image_k(a, b);                       // this row's own k: the call reached this kernel by its largest one
  // the row's noise, set up by one thread and read after the descent loop's barriers.  Held in registers across that loop, the
  // temperature made MODE 2 spill 8 bytes.
  if (tid == 0) s_noise = row_noise<MODE>(a, b, pos, V, tdiv);
  // 1. k-th largest key
  uint32_t prefix = 0;
  for (int bit = 31; bit >= 0; --bit) {
    const uint32_t cand = prefix | (1u << bit);
    int c = 0;
    for (int i = tid; i < V; i += SMP_THREADS) c += (fkey(row[i]) >= cand);
    int tot, dummy;
    block_sum2(c, 0, sc.red, warp, lane, tot, dummy);
    if (tot >= k) prefix = cand;
  }
  int cg = 0, ce = 0;
  for (int i = tid; i < V; i += SMP_THREADS) { const uint32_t key = fkey(row[i]); cg += (key > prefix); ce += (key == prefix); }
  int n_gt, n_eq;
  block_sum2(cg, ce, sc.red, warp, lane, n_gt, n_eq);
  const int need = k - n_gt;                         // ties kept, lowest indices first (1 <= need <= n_eq)
  // index of the last kept tie; all ties are kept in the common case (n_eq == need)
  if (tid == 0) s_cut = V;
  __syncthreads();
  if (n_eq > need && warp == 0) {
    int cnt = 0, cut = V;
    for (int i0 = 0; i0 < V && cnt < need; i0 += 32) {
      const int i = i0 + lane;
      const bool tie = i < V && fkey(row[i]) == prefix;
      const unsigned bal = __ballot_sync(0xffffffffu, tie);
      const int c = __popc(bal);
      if (cnt + c >= need) {                         // the need-th tie is in this group: its lane is the (need - cnt)-th set bit
        unsigned m = bal;
        for (int t = 0; t < need - cnt - 1; ++t) m &= m - 1;
        cut = i0 + __ffs(m) - 1;
      }
      cnt += c;
    }
    if (lane == 0) s_cut = cut;
  }
  __syncthreads();
  const int cut = s_cut;
  // 2. statistics + perturbed argmax over the kept set
  const RowNoise<MODE> noise = s_noise;
  constexpr float LOG2E = 1.4426950408889634f;
  float m_t = -1e30f, s_t = 0.f;
  float bv = -FLT_MAX, bx = 0.f; int bi = 0x7fffffff;
  for (int v = tid; v < V; v += SMP_THREADS) {
    const float x = row[v];
    if (x > m_t) { s_t *= ex2_approx((m_t - x) * LOG2E); m_t = x; }
    s_t += ex2_approx((x - m_t) * LOG2E);
    const uint32_t key = fkey(x);
    if (key > prefix || (key == prefix && v <= cut)) {
      const float p = noise.perturbed(x, v);
      if (bi == 0x7fffffff || better(p, v, bv, bi)) { bv = p; bi = v; bx = x; }
    }
  }
  // block reductions: softmax statistics, then the argmax (ties -> lowest vocabulary index)
  {
    float M = warp_max(m_t);
    if (lane == 0) sc.redf[warp] = M;
    __syncthreads();
    M = sc.redf[lane % (SMP_THREADS / 32)];
    M = warp_max(M);
    float sm = warp_sum(s_t * ex2_approx((m_t - M) * LOG2E));
    __syncthreads();
    if (lane == 0) sc.redf[warp] = sm;
    __syncthreads();
    if (tid == 0) { float t = 0.f; for (int w = 0; w < SMP_THREADS / 32; ++w) t += sc.redf[w]; s_s = t; s_m = M; }
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o), ox = __shfl_xor_sync(0xffffffffu, bx, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi != 0x7fffffff && (bi == 0x7fffffff || better(ov, oi, bv, bi))) { bv = ov; bi = oi; bx = ox; }
  }
  __syncthreads();
  if (lane == 0) { sc.redf[warp] = bv; sc.redi[warp] = bi; sc.redj[warp] = __float_as_int(bx); }
  __syncthreads();
  if (tid == 0) {
    bv = sc.redf[0]; bi = sc.redi[0]; bx = __int_as_float(sc.redj[0]);
    for (int w = 1; w < SMP_THREADS / 32; ++w) {
      const float ov = sc.redf[w]; const int oi = sc.redi[w];
      if (oi != 0x7fffffff && (bi == 0x7fffffff || better(ov, oi, bv, bi))) { bv = ov; bi = oi; bx = __int_as_float(sc.redj[w]); }
    }
    if (bi == 0x7fffffff) { bi = 0; bx = row[0]; }                 // degenerate rows (all -inf / NaN)
    write_sample(a, b, pos, bi, expf(bx - s_m) / s_s);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// rank selection of one batch row held in shared memory: flag[i] = 1 for the num_masked largest sc[i] (ties: lowest
// position).  FROZEN: positions with fz[i] != 0 are neither ranked nor selected.  Thread tid writes flag[tid + 256 k].
// ---------------------------------------------------------------------------------------------------------------
template <bool FROZEN>
__device__ __forceinline__ void rank_select(const float* sc, const uint8_t* fz, int* flag, int n, int num_masked, int tid) {
  for (int i = tid; i < n; i += 256) {
    const float s = sc[i]; int rank = 0;
    if (FROZEN) {
      for (int j = 0; j < n; ++j) { const float t = sc[j]; rank += !fz[j] && ((t > s) || (t == s && j < i)); }
      flag[i] = !fz[i] && rank < num_masked;
    } else {
      for (int j = 0; j < n; ++j) { const float t = sc[j]; rank += (t > s) || (t == s && j < i); }
      flag[i] = rank < num_masked;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// re-mask: per batch row pick the num_masked largest scores (ties: lowest position), scatter mask_id, reset scores.
// FROZEN (inpainting): positions with frozen[b, i] != 0 are neither ranked nor selected; row b selects
// min(num_masked_dev[b], rows) positions and pads masked_pos[b, c_b .. rows) with its first frozen position.
// ---------------------------------------------------------------------------------------------------------------
template <bool FROZEN>
__device__ __forceinline__ void remask_row(int64_t* __restrict__ ids, float* __restrict__ scores, int32_t* __restrict__ masked_pos,
                                           const uint8_t* __restrict__ frozen, int n, int num_masked, int rows, int64_t mask_id,
                                           float* sc, int* flag, uint8_t* fz, int* woff) {
  const int b = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < n; i += 256) sc[i] = scores[(int64_t)b * n + i];
  if (FROZEN) for (int i = tid; i < n; i += 256) fz[i] = frozen[(int64_t)b * n + i] != 0;
  __syncthreads();
  rank_select<FROZEN>(sc, fz, flag, n, num_masked, tid);
  __syncthreads();
  // ordered compaction: each thread owns a contiguous chunk
  const int per = (n + 255) / 256, lo = tid * per, hi = min(n, lo + per);
  int c = 0;
  for (int i = lo; i < hi; ++i) c += flag[i];
  int incl = c;
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) woff[warp + 1] = incl;
  if (tid == 0) woff[0] = 0;
  __syncthreads();
  if (tid == 0) for (int w = 1; w <= 8; ++w) woff[w] += woff[w - 1];
  __syncthreads();
  int o = woff[warp] + incl - c;
  for (int i = lo; i < hi; ++i) {
    if (flag[i]) { masked_pos[(int64_t)b * rows + o++] = i; ids[(int64_t)b * n + i] = mask_id; }
    scores[(int64_t)b * n + i] = -1e5f;
  }
  if (FROZEN) {
    // pad rows: the sampler computes them but (only_masked) writes no id at a frozen position, and every pad row of this image computes
    // the same value, so the repeated score writes are deterministic.  An image without frozen positions has count == rows (mmg.h).
    const int selected = woff[8];
    if (selected < rows) {
      int first = n;
      for (int i = 0; i < n; ++i) if (fz[i]) { first = i; break; }
      // no frozen position (generate() with per-image step counts: an image that needs fewer rows than the step's largest count): the pad
      // rows repeat the image's first selected row, whose id and score they recompute bit for bit, so no other position's score changes
      if (first == n) for (int i = 0; i < n; ++i) if (flag[i]) { first = i; break; }
      for (int r = selected + tid; r < rows; r += 256) masked_pos[(int64_t)b * rows + r] = first < n ? first : 0;
    }
  }
}

__global__ void __launch_bounds__(256)
remask_kernel(int64_t* __restrict__ ids, float* __restrict__ scores, int32_t* __restrict__ masked_pos, int n, int num_masked, int64_t mask_id) {
  extern __shared__ float sc[];                       // [n] scores, then [n] flags (as int)
  __shared__ int woff[9];
  pdl_wait(); pdl_trigger();
  remask_row<false>(ids, scores, masked_pos, nullptr, n, num_masked, num_masked, mask_id, sc, reinterpret_cast<int*>(sc + n), nullptr, woff);
}

__global__ void __launch_bounds__(256)
remask_frozen_kernel(const mmg_remask_frozen_args a) {
  extern __shared__ float sc[];                       // [n] scores, [n] flags (as int), [n] frozen bytes
  __shared__ int woff[9];
  pdl_wait(); pdl_trigger();
  const int count = a.num_masked[blockIdx.x];
  const int limit = count < a.rows ? (count > 0 ? count : 0) : a.rows;
  remask_row<true>(a.ids, a.scores, a.masked_pos, a.frozen, a.n, limit, a.rows, a.mask_id, sc, reinterpret_cast<int*>(sc + a.n),
                   reinterpret_cast<uint8_t*>(sc + 2 * a.n), woff);
}

// ---------------------------------------------------------------------------------------------------------------
// mask-free editing (MaskGit.edit): row b draws one uniform key per position (injected, or Philox with counter
// (0xFFFFFFFE, iteration, global position) next to the gumbel (c0 = vocabulary index) and critic (c0 = 0xFFFFFFFF) streams),
// selects the num_select[b] largest keys among its editable positions (keep == 0; ties: lowest position), writes
// frozen_out = !selected, mask_id at the selected ids and 0 into every score of the row.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
edit_select_kernel(const mmg_edit_select_args a) {
  extern __shared__ float sc[];                       // [n] keys, [n] flags (as int), [n] keep bytes
  pdl_wait(); pdl_trigger();
  const int b = blockIdx.x, tid = threadIdx.x, n = a.n;
  int* flag = reinterpret_cast<int*>(sc + n);
  uint8_t* fz = reinterpret_cast<uint8_t*>(sc + 2 * n);
  const int64_t base = (int64_t)b * n;
  // per-image seeds: image b's own key and the image-local position as the row counter
  const uint64_t seed = a.image_seed ? a.image_seed[b] : call_seed(a.seed, a.seed_dev);
  const int64_t row0 = a.image_seed ? 0 : a.row_offset + base;
  for (int i = tid; i < n; i += 256) {
    sc[i] = a.u ? a.u[base + i] : philox_uniform(PHILOX_C0_EDIT, (uint32_t)a.iteration, row0 + i, seed);
    fz[i] = a.keep[base + i] != 0;
  }
  __syncthreads();
  const int count = a.num_select[b];
  rank_select<true>(sc, fz, flag, n, count > 0 ? count : 0, tid);
  for (int i = tid; i < n; i += 256) {                // flag[i] was written by this thread
    const bool sel = flag[i] != 0;
    a.frozen_out[base + i] = !sel;
    if (sel) a.ids[base + i] = a.mask_id;
    a.scores[base + i] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// image extrapolation (MaskGit.extrapolate): one thread per window token.  Load copies the canvas block into ids with
// mask_id on the strip and zeroes the scores; store writes the strip of ids back into the canvas.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
extrapolate_window_kernel(const mmg_extrapolate_window_args a) {
  pdl_wait(); pdl_trigger();
  const int nn = a.f * a.f;
  const int64_t total = (int64_t)a.B * nn;
  for (int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x; t < total; t += (int64_t)gridDim.x * 256) {
    const int64_t b = t / nn;
    const int p = (int)(t - b * nn), i = p / a.f, j = p - i * a.f;
    const int k = a.direction < 2 ? j : i;                                   // position across the strip's axis
    const bool strip = (a.direction & 1) ? k < a.stride : k >= a.f - a.stride;
    const int64_t c = (b * a.canvas_h + a.row0 + i) * a.canvas_w + a.col0 + j;
    if (a.store) {
      if (strip) a.canvas[c] = a.ids[t];
    } else {
      a.ids[t] = strip ? a.mask_id : a.canvas[c];
      a.scores[t] = 0.f;
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------
// token-critic scores (muse_maskgit_pytorch.py:590-600): per sequence position, the dim_out = 1 head applied to the
// final-LayerNorm embedding of the critic's forward(s), CFG-combined, plus annealed uniform noise.  One warp per row.
//   s = dot(LN(x_cond)*gamma, w) [+ bias];  if x_null: s = s_null + (s - s_null) * cond_scale;  s += (u - 0.5) * noise_mul
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float critic_head(const float* __restrict__ xr, const float* __restrict__ gamma, const float* __restrict__ w, int dim, int lane) {
  float sum = 0.f;
  for (int c = lane; c < dim; c += 32) sum += xr[c];
  const float mean = warp_sum(sum) / (float)dim;
  float sq = 0.f, dot = 0.f;
  for (int c = lane; c < dim; c += 32) { const float d = xr[c] - mean; sq += d * d; dot += d * __ldg(gamma + c) * __ldg(w + c); }
  sq = warp_sum(sq); dot = warp_sum(dot);
  return dot * rsqrtf(sq / (float)dim + 1e-5f);
}

__global__ void __launch_bounds__(256)
critic_score_kernel(mmg_critic_score_args a) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= a.rows) return;
  float s = critic_head(a.x_cond + row * a.dim, a.gamma, a.w, a.dim, lane) + a.bias;
  const float cs = a.cond_scale_dev ? a.cond_scale_dev[row] : a.cond_scale;
  if (a.x_null && !(a.cond_scale_dev && cs == 1.f)) {       // a per-row scale of exactly 1 scores x_cond alone, as x_null == NULL
    const float sn = critic_head(a.x_null + row * a.dim, a.gamma, a.w, a.dim, lane) + a.bias;
    s = sn + (s - sn) * cs;
  }
  if (lane == 0) {
    float u;
    if (a.u) u = a.u[row];
    else {
      // per-row keys: the row's image seed and image-local position
      const uint64_t seed = a.row_key ? a.row_key[2 * row] : call_seed(a.seed, a.seed_dev);
      const int64_t grow = a.row_key ? (int64_t)a.row_key[2 * row + 1] : a.row_offset + row;
      if (a.rng_mode == 1) {      // ATen stream of `uniform(scores.shape)`: flat index = global position
        const uint64_t k = (uint64_t)grow / a.aten_stride;
        u = aten_uniform((uint32_t)((uint64_t)grow - k * a.aten_stride), k, aten_offset4(a.aten_offset, a.aten_offset_dev), seed);
      } else
        u = philox_uniform(PHILOX_C0_CRITIC, (uint32_t)a.step, grow, seed);
    }
    a.scores[row] = s + (u - 0.5f) * (a.noise_mul_dev ? a.noise_mul_dev[row] : a.noise_mul);
  }
}

}  // namespace mmg

using namespace mmg;

extern "C" int mmg_logits_sample(const mmg_logits_sample_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->logits && a->masked_pos && a->ids && a->scores, "mmg_logits_sample: NULL pointer");
  MMG_CHECK_ARG(a->V >= 32 && a->V % 32 == 0, "mmg_logits_sample: V=%d must be a positive multiple of 32", a->V);
  MMG_CHECK_ARG(a->k >= 1 && a->k <= a->V, "mmg_logits_sample: k=%d out of range (1 .. V=%d)", a->k, a->V);
  MMG_CHECK_ARG(!a->row_index || (a->row_count_dev && a->row_index_cap > 0), "mmg_logits_sample: row_index needs row_count_dev and row_index_cap");
  const int64_t R = a->row_index ? a->row_index_cap : (int64_t)a->B * a->num_masked;
  if (R == 0) return MMG_OK;
  static const size_t smem = (size_t)SMP_CAP * 8 + (size_t)SMP_THREADS * 64;
  if (int rc = check_noise_args(*a, "mmg_logits_sample")) return rc;
  static void (*const list_kernels[3])(mmg_logits_sample_args, float) = {logits_sample_kernel<0>, logits_sample_kernel<1>, logits_sample_kernel<2>};
  static void (*const bigk_kernels[3])(mmg_logits_sample_args, float) = {logits_sample_bigk_kernel<0>, logits_sample_bigk_kernel<1>,
                                                                         logits_sample_bigk_kernel<2>};
  static const cudaError_t attr = [] {
    for (auto kern : list_kernels)
      if (cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;
    return cudaSuccess;
  }();
  if (attr != cudaSuccess) return fail(MMG_ECUDA, "cudaFuncSetAttribute(logits_sample): %s", cudaGetErrorString(attr));
  float t = a->temperature; if (t < 1e-10f) t = 1e-10f;      // max(temperature, 1e-10): muse_maskgit_pytorch.py:411
  const int mode = noise_mode(*a);
  if (a->k > SMP_CAP)                                          // kept set larger than the candidate list (of the largest per-image k): the row-walking kernel
    MMG_CUDA(launch_pdl(bigk_kernels[mode], dim3((unsigned)R), dim3(SMP_THREADS), 0, st, *a, t));
  else
    MMG_CUDA(launch_pdl(list_kernels[mode], dim3((unsigned)R), dim3(SMP_THREADS), smem, st, *a, t));
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_remask(const mmg_remask_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->ids && a->scores && a->masked_pos, "mmg_remask: NULL pointer");
  MMG_CHECK_ARG(a->n > 0 && a->num_masked >= 1 && a->num_masked <= a->n && a->n <= 16384, "mmg_remask: n=%d num_masked=%d", a->n, a->num_masked);
  if (a->B == 0) return MMG_OK;
  MMG_CUDA(launch_pdl(remask_kernel, dim3(a->B), dim3(256), (size_t)a->n * 8, st, a->ids, a->scores, a->masked_pos, a->n, a->num_masked, a->mask_id));
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_remask_frozen(const mmg_remask_frozen_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->ids && a->scores && a->masked_pos && a->frozen && a->num_masked, "mmg_remask_frozen: NULL pointer");
  MMG_CHECK_ARG(a->B >= 0 && a->n > 0 && a->rows >= 1 && a->rows <= a->n && a->n <= 16384, "mmg_remask_frozen: B=%d n=%d rows=%d", a->B, a->n, a->rows);
  if (a->B == 0) return MMG_OK;
  const size_t smem = (size_t)a->n * 9;                 // scores, flags, frozen bytes
  static const cudaError_t attr = cudaFuncSetAttribute(remask_frozen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 9);
  if (attr != cudaSuccess) return fail(MMG_ECUDA, "cudaFuncSetAttribute(remask_frozen): %s", cudaGetErrorString(attr));
  MMG_CUDA(launch_pdl(remask_frozen_kernel, dim3(a->B), dim3(256), smem, st, *a));
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_edit_select(const mmg_edit_select_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->ids && a->scores && a->frozen_out && a->keep && a->num_select, "mmg_edit_select: NULL pointer");
  MMG_CHECK_ARG(a->B >= 0 && a->n > 0 && a->n <= 16384 && a->iteration >= 0, "mmg_edit_select: B=%d n=%d iteration=%d", a->B, a->n, a->iteration);
  MMG_CHECK_ARG(!a->image_seed || !a->u, "mmg_edit_select: image_seed needs u == NULL");
  if (a->B == 0) return MMG_OK;
  const size_t smem = (size_t)a->n * 9;                 // keys, flags, keep bytes
  static const cudaError_t attr = cudaFuncSetAttribute(edit_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 9);
  if (attr != cudaSuccess) return fail(MMG_ECUDA, "cudaFuncSetAttribute(edit_select): %s", cudaGetErrorString(attr));
  MMG_CUDA(launch_pdl(edit_select_kernel, dim3(a->B), dim3(256), smem, st, *a));
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_extrapolate_window(const mmg_extrapolate_window_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->canvas && a->ids && a->scores, "mmg_extrapolate_window: NULL pointer");
  MMG_CHECK_ARG(a->B >= 0 && a->f > 0 && a->f <= 128 && a->stride >= 1 && a->stride <= a->f && a->direction >= 0 && a->direction <= 3 &&
                (a->store == 0 || a->store == 1), "mmg_extrapolate_window: B=%d f=%d stride=%d direction=%d store=%d", a->B, a->f, a->stride,
                a->direction, a->store);
  MMG_CHECK_ARG(a->row0 >= 0 && a->col0 >= 0 && (int64_t)a->row0 + a->f <= a->canvas_h && (int64_t)a->col0 + a->f <= a->canvas_w,
                "mmg_extrapolate_window: window at (%d, %d) of size %d outside the %d x %d canvas", a->row0, a->col0, a->f, a->canvas_h,
                a->canvas_w);
  if (a->B == 0) return MMG_OK;
  const int64_t blocks = ((int64_t)a->B * a->f * a->f + 255) / 256;
  MMG_CUDA(launch_pdl(extrapolate_window_kernel, dim3((unsigned)(blocks < 65535 ? blocks : 65535)), dim3(256), 0, st, *a));
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_critic_score(const mmg_critic_score_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x_cond && a->gamma && a->w && a->scores, "mmg_critic_score: NULL pointer");
  MMG_CHECK_ARG(a->dim > 0 && a->rows >= 0, "mmg_critic_score: dim=%d", a->dim);
  MMG_CHECK_ARG(a->rng_mode == 0 || (a->rng_mode == 1 && a->aten_stride >= 256 && a->aten_offset % 4 == 0), "mmg_critic_score: rng_mode=%d aten_stride=%u", a->rng_mode, a->aten_stride);
  MMG_CHECK_ARG(!a->row_key || (a->rng_mode == 0 && !a->u), "mmg_critic_score: row_key needs rng_mode 0 and u == NULL");
  if (a->rows == 0) return MMG_OK;
  MMG_CUDA(launch_pdl(critic_score_kernel, dim3((unsigned)((a->rows + 7) / 8)), dim3(256), 0, st, *a));
  MMG_LAUNCHED();
  return MMG_OK;
}

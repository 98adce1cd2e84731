// Device-side pieces of the sampling tail shared by the materialised-logits kernel (mmg_sampler.cu) and the fused
// logits + sampling path (mmg_logits_fused.cu): order-preserving keys, Philox, the sample-quantile threshold (phase A) and the
// perturbed argmax restricted to the exact top-k on a candidate list (phase C).
#pragma once
#include "mmg_common.cuh"
#include <float.h>

namespace mmg {

constexpr int SMP_THREADS = 512;
constexpr int SMP_SAMPLE = 4096;
constexpr int SMP_CAP = 9216;

__device__ __forceinline__ uint32_t fkey(float x) {           // order-preserving float -> uint32
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ld_stream(const float* p) {
  float v; asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p)); return v;
}
__device__ __forceinline__ float4 ld_stream4(const float4* p) {
  float4 v; asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p)); return v;
}

// Philox4x32-10, counter = (v, step, row_lo, row_hi), key = seed; returns the first output word.
__device__ __forceinline__ uint32_t philox_first(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;     // one IMAD.WIDE each
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}

// The same function for many counters that differ only in c0 (one row of logits: c1 = step, c2 / c3 = global row, key = seed): the key schedule
// and everything of rounds 1 and 2 that does not depend on c0 is computed once per row (2 of the 20 multiplies, the 20 key additions).
struct PhiloxRow {
  uint32_t rk0[10], rk1[10];      // round keys
  uint32_t a, b, cx;              // round 1: n0 = a, n1 = b (constants), n2 = hi(M0 c0) ^ cx, n3 = lo(M0 c0)
  uint32_t hi2, lo2;              // round 2: M0 * a
};
__device__ __forceinline__ PhiloxRow philox_row(uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
  PhiloxRow r;
#pragma unroll
  for (int i = 0; i < 10; ++i) { r.rk0[i] = k0; r.rk1[i] = k1; k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
  const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
  r.a = (uint32_t)(p1 >> 32) ^ c1 ^ r.rk0[0]; r.b = (uint32_t)p1; r.cx = c3 ^ r.rk1[0];
  const uint64_t p0 = (uint64_t)0xD2511F53u * r.a;
  r.hi2 = (uint32_t)(p0 >> 32); r.lo2 = (uint32_t)p0;
  return r;
}
__device__ __forceinline__ uint32_t philox_first_row(uint32_t c0, const PhiloxRow& r) {
  // round 1
  const uint64_t q0 = (uint64_t)0xD2511F53u * c0;
  uint32_t n2 = (uint32_t)(q0 >> 32) ^ r.cx, n3 = (uint32_t)q0;
  // round 2: counter (a, b, n2, n3)
  const uint64_t q1 = (uint64_t)0xCD9E8D57u * n2;
  uint32_t d0 = (uint32_t)(q1 >> 32) ^ r.b ^ r.rk0[1], d1 = (uint32_t)q1, d2 = r.hi2 ^ n3 ^ r.rk1[1], d3 = r.lo2;
#pragma unroll
  for (int i = 2; i < 10; ++i) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * d0, p1 = (uint64_t)0xCD9E8D57u * d2;
    const uint32_t e0 = (uint32_t)(p1 >> 32) ^ d1 ^ r.rk0[i], e1 = (uint32_t)p1, e2 = (uint32_t)(p0 >> 32) ^ d3 ^ r.rk1[i], e3 = (uint32_t)p0;
    d0 = e0; d1 = e1; d2 = e2; d3 = e3;
  }
  return d0;
}

// Philox4x32-10, all four output words
__device__ __forceinline__ uint4 philox4(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// The value ATen's CUDA `uniform_(0, 1)` writes at flat index t + stride * k of an fp32 tensor (generator seed / offset):
// word (k & 3) of Philox(counter = offset/4 + (k >> 2), subsequence = t), mapped like curand_uniform4 (w * 2^-32 + 2^-33, in
// (0, 1]) and then 1 -> 0.  (DistributionTemplates.h: distribution_elementwise_grid_stride_kernel + uniform_kernel.)
__device__ __forceinline__ float aten_uniform(uint32_t t, uint64_t k, uint64_t off4, uint64_t seed) {
  const uint64_t ctr = off4 + (k >> 2);
  const uint4 w4 = philox4((uint32_t)ctr, (uint32_t)(ctr >> 32), t, 0u, (uint32_t)seed, (uint32_t)(seed >> 32));
  const uint32_t ii = (uint32_t)k & 3u;
  const uint32_t w = ii == 0 ? w4.x : ii == 1 ? w4.y : ii == 2 ? w4.z : w4.w;
  const float u = fmaf(__uint2float_rn(w), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
  return u == 1.0f ? 0.0f : u;
}

__device__ __forceinline__ bool better(float v, int vi, float w, int wi) { return v > w || (v == w && vi < wi); }
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float key_to_float(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// block-wide sum of two packed counters (each < 2^15), one __syncthreads pair; result broadcast to every thread
__device__ __forceinline__ void block_sum2(int a, int b, int* red, int warp, int lane, int& oa, int& ob) {
  a = __reduce_add_sync(0xffffffffu, a); b = __reduce_add_sync(0xffffffffu, b);
  __syncthreads();
  if (lane == 0) { red[warp] = a; red[32 + warp] = b; }
  __syncthreads();
  oa = 0; ob = 0;
#pragma unroll
  for (int w = 0; w < SMP_THREADS / 32; ++w) { oa += red[w]; ob += red[32 + w]; }
}


// scratch shared by the phases below (one per CTA)
struct SampleScratch {
  int red[64];
  float redf[32]; int redi[32]; int redj[32];
};

// ---------------- phase A: sample keys (registers) -> provisional threshold ----------------
// sk: this thread's SMP_SAMPLE / SMP_THREADS order-preserving keys of an `ns`-element sample of a V-wide row (key 0 = no element).
// ns == V: the "sample" is the whole row -> exact k-th largest by a block-wide radix descent (two key bits per round).
// ns <  V: every warp finds the rank-(rs/16) key of ITS 256 samples with shuffles only, the block threshold is the mean of the 16
//          warp estimates (same variance as one 4096-sample quantile; exactness is restored by the caller's n >= k check);
//          rs = mu + z*sigma + 2 with mu = ns * k / V: expected exceedance count of the threshold in the row ~ k + z sigma (V / ns).
// Returns -FLT_MAX when no usable threshold exists (every element is then a candidate).  Contains block barriers.
constexpr int SMP_SPT = SMP_SAMPLE / SMP_THREADS;
__device__ __forceinline__ float sample_threshold(const uint32_t (&sk)[SMP_SPT], int ns, int V, int k, SampleScratch& sc, int warp, int lane) {
  float tlo;
  if (ns == V) {
    const int rs = k < ns ? k : ns;
    uint32_t prefix = 0;
    for (int bit = 30; bit >= 0; bit -= 2) {
      const uint32_t c1 = prefix | (1u << bit), c2 = prefix | (2u << bit), c3 = prefix | (3u << bit);
      int n1 = 0, n2 = 0, n3 = 0;
#pragma unroll
      for (int j = 0; j < SMP_SPT; ++j) { n1 += (sk[j] >= c1); n2 += (sk[j] >= c2); n3 += (sk[j] >= c3); }
      int t12, t3;
      block_sum2(n1 | (n2 << 16), n3, sc.red, warp, lane, t12, t3);
      const int t1 = t12 & 0xffff, t2 = t12 >> 16;
      if (t3 >= rs) prefix = c3; else if (t2 >= rs) prefix = c2; else if (t1 >= rs) prefix = c1;
    }
    tlo = key_to_float(prefix);
    if (prefix == 0) tlo = -FLT_MAX;
  } else {
    const float pf = (float)k / (float)V; const float mu = pf * ns;
    const int rs = (int)(mu + 4.0f * sqrtf(mu * (1.f - pf)) + 2.f);
    const int rw = (rs + SMP_THREADS / 32 - 1) / (SMP_THREADS / 32);
    uint32_t prefix = 0;
    for (int bit = 30; bit >= 12; bit -= 2) {                          // 20 key bits are plenty for a lower bound
      const uint32_t c1 = prefix | (1u << bit), c2 = prefix | (2u << bit), c3 = prefix | (3u << bit);
      int n = 0;
#pragma unroll
      for (int j = 0; j < SMP_SPT; ++j) n += (sk[j] >= c1) + ((sk[j] >= c2) << 10) + ((sk[j] >= c3) << 20);
      n = __reduce_add_sync(0xffffffffu, n);
      const int t1 = n & 1023, t2 = (n >> 10) & 1023, t3 = n >> 20;
      if (t3 >= rw) prefix = c3; else if (t2 >= rw) prefix = c2; else if (t1 >= rw) prefix = c1;
    }
    if (lane == 0) sc.redf[warp] = prefix ? key_to_float(prefix) : -FLT_MAX;
    __syncthreads();
    float acc = 0.f; bool bad = false;
#pragma unroll
    for (int w = 0; w < SMP_THREADS / 32; ++w) { const float t = sc.redf[w]; bad |= (t == -FLT_MAX) | !(t == t); acc += t; }
    tlo = bad ? -FLT_MAX : acc * (1.0f / (SMP_THREADS / 32));
    __syncthreads();
  }
  return tlo;
}

// max(temperature, 1e-10) of image b (muse_maskgit_pytorch.py:411): the per-image table when given, else the launcher's clamped scalar
__device__ __forceinline__ float image_tdiv(const mmg_logits_sample_args& a, int b, float tdiv) {
  if (!a.temperature_dev) return tdiv;
  const float t = a.temperature_dev[b];
  return t < 1e-10f ? 1e-10f : t;
}

// ---------------- phase C: perturbed argmax restricted to the exact top-k ----------------
// lval / lidx: the n candidates of the row (every element >= some threshold, n >= k or the complete exact top-k); (b, pos): the row.
// MODE 1 = injected-noise parity mode, MODE 2 = ATen-compatible in-kernel Philox (the stream a seeded torch.cuda run of the reference
// draws): IEEE division and accurate logf so the perturbed values match the reference's fp32 arithmetic as closely as a GPU can;
// MODE 0 (libmmg's own Philox keying) uses fast MUFU-based logs and a reciprocal multiply.
// Block argmax of the perturbed value, accepted iff the candidate's exact rank (#greater + #equal-with-lower-index) is < k, else
// excluded and repeated: equals argmax over torch.topk's kept set without ever forming the set.  Returns (token, its logit) to every
// thread; token < 0 for degenerate rows (all -inf / NaN).
template <int MODE>
__device__ __forceinline__ void sample_from_list(const mmg_logits_sample_args& a, float tdiv, const float* lval, const int* lidx, int n, int k, int V,
                                                 int b, int pos, SampleScratch& sc, int tid, int warp, int lane, int& win_v, float& win_x) {
  const int64_t grow = a.row_offset + (int64_t)b * a.n + pos;
  const uint64_t seed = a.seed + (a.seed_dev ? *a.seed_dev : 0ull);
  const float inv_t = 1.0f / tdiv;
  uint64_t aq0 = 0, aoff4 = 0; uint32_t ar0 = 0;
  if (MODE == 2) {            // flat index of logit (grow, v) in the reference's [B, n, V] noise tensor = grow * V + v = ar0 + v + S * aq0
    const uint64_t base = (uint64_t)grow * (uint64_t)V;
    aq0 = base / a.aten_stride; ar0 = (uint32_t)(base - aq0 * a.aten_stride);
    aoff4 = (a.aten_offset + (a.aten_offset_dev ? *a.aten_offset_dev : 0ull)) >> 2;
  }
  constexpr int PER = (SMP_CAP + SMP_THREADS - 1) / SMP_THREADS;
  float pv[PER];
  PhiloxRow prow;
  if (MODE == 0) prow = philox_row((uint32_t)a.step, (uint32_t)grow, (uint32_t)((uint64_t)grow >> 32), (uint32_t)seed, (uint32_t)(seed >> 32));
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int s = tid + j * SMP_THREADS;
    float p = -FLT_MAX;
    if (s < n) {
      const int v = lidx[s];
      if (MODE != 0) {
        float u;
        if (MODE == 1) u = a.u[((int64_t)b * a.n + pos) * V + v];
        else { const uint32_t r = ar0 + (uint32_t)v, dq = r / a.aten_stride; u = aten_uniform(r - dq * a.aten_stride, aq0 + dq, aoff4, seed); }
        const float l1 = logf(fmaxf(u, 1e-20f));
        p = __fdiv_rn(lval[s], tdiv) - logf(fmaxf(-l1, 1e-20f));
      } else {
        const float u = (float)(philox_first_row((uint32_t)v, prow) >> 8) * (1.0f / 16777216.0f);
        const float l1 = __logf(fmaxf(u, 1e-20f));
        p = fmaf(lval[s], inv_t, -__logf(fmaxf(-l1, 1e-20f)));
      }
    }
    pv[j] = p;
  }
  win_v = -1; win_x = 0.f;
  for (int iter = 0; iter < n; ++iter) {
    // block argmax of the perturbed value (ties -> lowest vocabulary index)
    float bv = -FLT_MAX; int bi = 0x7fffffff, bs = -1;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int s = tid + j * SMP_THREADS;
      if (s < n) { const int vi = lidx[s]; if (bs < 0 || better(pv[j], vi, bv, bi)) { bv = pv[j]; bi = vi; bs = s; } }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o); const int os = __shfl_xor_sync(0xffffffffu, bs, o);
      if (os >= 0 && (bs < 0 || better(ov, oi, bv, bi))) { bv = ov; bi = oi; bs = os; }
    }
    __syncthreads();
    if (lane == 0) { sc.redf[warp] = bv; sc.redi[warp] = bi; sc.redj[warp] = bs; }
    __syncthreads();
    bv = sc.redf[0]; bi = sc.redi[0]; bs = sc.redj[0];
#pragma unroll
    for (int w = 1; w < SMP_THREADS / 32; ++w) {
      const float ov = sc.redf[w]; const int oi = sc.redi[w], os = sc.redj[w];
      if (os >= 0 && (bs < 0 || better(ov, oi, bv, bi))) { bv = ov; bi = oi; bs = os; }
    }
    // exact rank of the candidate inside the row (the list covers everything >= its value)
    const float cx = lval[bs];
    int c = 0;
    for (int s = tid; s < n; s += SMP_THREADS) { const float x = lval[s]; c += (x > cx) || (x == cx && lidx[s] < bi); }
    int rank, dummy;
    block_sum2(c, 0, sc.red, warp, lane, rank, dummy);
    if (rank < k) { win_v = bi; win_x = cx; break; }
    // not in the kept set: drop its perturbed value (its logit stays in the list for later rank computations)
#pragma unroll
    for (int j = 0; j < PER; ++j) if (tid + j * SMP_THREADS == bs) pv[j] = -FLT_MAX;
  }
}

}  // namespace mmg

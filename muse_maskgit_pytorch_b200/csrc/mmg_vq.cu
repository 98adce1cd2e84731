// VQ codebook lookups (HBM-bound scans).  replaces vqgan_vae.py:424 (quantizer forward) and 429-435 (ids -> codes).
#include "mmg_common.cuh"
#include <float.h>

namespace mmg {

// LFQ encode: the nearest code of the implicit {+-1}^bits codebook is the sign pattern of the projected token.
// CUDA-core path (fp32 "parity" precision; bf16 inputs normally take the wgmma route below).  The projection [bits, D] sits in
// shared memory; a warp owns LFQ_TOK tokens at a time and a lane 4 channels of each (one 128-bit / 64-bit load per token), so one
// 128-bit shared-memory read of a weight quad feeds 4 x LFQ_TOK FMAs (0.06 shared reads per FMA instead of 1) and the token
// stream is fully coalesced.  Warp-shuffle reduction, then bit-pack (MSB first; x == 0 -> bit 0).
constexpr int LFQ_TOK = 4;
template <typename T> __device__ __forceinline__ float4 lfq_load4(const T* p);
template <> __device__ __forceinline__ float4 lfq_load4<float>(const float* p) {
  float4 v; asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p)); return v;
}
template <> __device__ __forceinline__ float4 lfq_load4<bf16>(const bf16* p) {
  uint32_t a, b; asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "l"(p));
  return make_float4(__uint_as_float(a << 16), __uint_as_float(a & 0xffff0000u), __uint_as_float(b << 16), __uint_as_float(b & 0xffff0000u));
}

template <typename T, int BITS_MAX>
__global__ void __launch_bounds__(256)
lfq_encode_kernel(const T* __restrict__ x, const float* __restrict__ w_in, const float* __restrict__ b_in, int64_t* __restrict__ ids,
                  int64_t tokens, int D, int bits) {
  extern __shared__ float ws[];                    // [bits][D]
  for (int i = threadIdx.x * 4; i < bits * D; i += blockDim.x * 4) *reinterpret_cast<float4*>(ws + i) = *reinterpret_cast<const float4*>(w_in + i);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t groups = (tokens + LFQ_TOK - 1) / LFQ_TOK;
  for (int64_t g = (int64_t)blockIdx.x * 8 + warp; g < groups; g += (int64_t)gridDim.x * 8) {
    const int64_t t0 = g * LFQ_TOK;
    float acc[LFQ_TOK][BITS_MAX];
#pragma unroll
    for (int k = 0; k < LFQ_TOK; ++k)
#pragma unroll
      for (int i = 0; i < BITS_MAX; ++i) acc[k][i] = 0.f;
#pragma unroll 2
    for (int c = lane * 4; c < D; c += 128) {
      float4 xv[LFQ_TOK];
#pragma unroll
      for (int k = 0; k < LFQ_TOK; ++k) xv[k] = (t0 + k < tokens) ? lfq_load4<T>(x + (t0 + k) * D + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int i = 0; i < BITS_MAX; ++i) {
        if (i < bits) {
          const float4 wv = *reinterpret_cast<const float4*>(ws + i * D + c);
#pragma unroll
          for (int k = 0; k < LFQ_TOK; ++k)
            acc[k][i] = fmaf(xv[k].x, wv.x, fmaf(xv[k].y, wv.y, fmaf(xv[k].z, wv.z, fmaf(xv[k].w, wv.w, acc[k][i]))));
        }
      }
    }
#pragma unroll
    for (int k = 0; k < LFQ_TOK; ++k) {
      int64_t id = 0;
#pragma unroll
      for (int i = 0; i < BITS_MAX; ++i) {
        if (i < bits) {
          const float s = warp_sum(acc[k][i]) + (b_in ? __ldg(b_in + i) : 0.f);
          if (s > 0.f) id |= (int64_t)1 << (bits - 1 - i);
        }
      }
      if (lane == 0 && t0 + k < tokens) ids[t0 + k] = id;
    }
  }
}

// generic shapes (D % 4 != 0, identity projection): one warp per token, scalar loads
template <typename T, int BITS_MAX>
__global__ void __launch_bounds__(256)
lfq_encode_generic_kernel(const T* __restrict__ x, const float* __restrict__ w_in, const float* __restrict__ b_in, int64_t* __restrict__ ids,
                          int64_t tokens, int D, int bits) {
  extern __shared__ float ws[];                    // [bits][D]
  if (w_in) for (int i = threadIdx.x; i < bits * D; i += blockDim.x) ws[i] = w_in[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < tokens; t += (int64_t)gridDim.x * 8) {
    const T* xr = x + t * D;
    float acc[BITS_MAX];
#pragma unroll
    for (int i = 0; i < BITS_MAX; ++i) acc[i] = 0.f;
    if (w_in) {
      for (int c = lane; c < D; c += 32) {
        const float xv = to_f(xr[c]);
#pragma unroll
        for (int i = 0; i < BITS_MAX; ++i) if (i < bits) acc[i] = fmaf(xv, ws[i * D + c], acc[i]);
      }
#pragma unroll
      for (int i = 0; i < BITS_MAX; ++i) { acc[i] = warp_sum(acc[i]); if (i < bits && b_in) acc[i] += b_in[i]; }
    } else {
#pragma unroll
      for (int i = 0; i < BITS_MAX; ++i) if (i < bits) acc[i] = to_f(xr[i]);
    }
    if (lane == 0) {
      int64_t id = 0;
#pragma unroll
      for (int i = 0; i < BITS_MAX; ++i) if (i < bits && acc[i] > 0.f) id |= (int64_t)1 << (bits - 1 - i);
      ids[t] = id;
    }
  }
}

// Explicit codebook: ids[t] = argmin_k ||x_t - e_k||^2 = argmin_k (||e_k||^2 - 2 x_t.e_k)   (||x_t||^2 is constant in k).
// Tiled scan: CTA = 64 tokens x 64 codes, the token and code tiles are staged through shared memory with coalesced loads
// (16 channels per step), 4x4 register micro-tiles, code norms accumulated on the fly; each row's best (distance, code) of
// the tile is merged across code tiles with one 64-bit atomicMin on (orderkey(distance) << 32 | code): lowest code wins ties.
__global__ void vq_init_kernel(unsigned long long* ids, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ids[i] = ~0ull;
}
__global__ void vq_finish_kernel(unsigned long long* ids, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ids[i] &= 0xffffffffull;
}
__global__ void __launch_bounds__(256)
vq_l2_argmin_kernel(const float* __restrict__ x, const float* __restrict__ cb, unsigned long long* __restrict__ best, int64_t tokens, int K, int D) {
  __shared__ float Xs[16][64 + 4];
  __shared__ float Es[16][64 + 4];
  __shared__ float Ds[64][64 + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t t0 = (int64_t)blockIdx.x * 64;
  const int k0 = blockIdx.y * 64;
  const int lr = tid >> 2, lk = (tid & 3) * 4;
  float acc[4][4] = {}; float e2[4] = {};
  for (int d0 = 0; d0 < D; d0 += 16) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int d = d0 + lk + j;
      Xs[lk + j][lr] = (t0 + lr < tokens && d < D) ? x[(t0 + lr) * D + d] : 0.f;
      Es[lk + j][lr] = (k0 + lr < K && d < D) ? __ldg(cb + (int64_t)(k0 + lr) * D + d) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = Xs[kk][ty * 4 + i]; b[i] = Es[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        e2[i] = fmaf(b[i], b[i], e2[i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) Ds[ty * 4 + i][tx * 4 + j] = e2[j] - 2.f * acc[i][j];
  __syncthreads();
  if (tid < 64 && t0 + tid < tokens) {
    unsigned long long bst = ~0ull;
    for (int j = 0; j < 64 && k0 + j < K; ++j) {
      const uint32_t u = __float_as_uint(Ds[tid][j]);
      const uint32_t key = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      const unsigned long long cand = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(k0 + j);
      bst = cand < bst ? cand : bst;
    }
    atomicMin(best + t0 + tid, bst);
  }
}

// ids -> +-1 codes -> project_out (LFQ.indices_to_codes): out[t, c] = b_out[c] + sum_i (+-1)_i w_out[c, i]
// A thread keeps the `bits` weights of two adjacent output channels in registers and walks a slice of DEC_TOK tokens (ids staged in
// shared memory, sign masks uniform across the block): the projection is read once per CTA instead of once per token.
constexpr int DEC_TOK = 64, DEC_MAXB = 24;
template <typename T>
__global__ void __launch_bounds__(256)
vq_decode_codes_kernel(const int64_t* __restrict__ ids, const float* __restrict__ w_out, const float* __restrict__ b_out, T* __restrict__ out,
                       int64_t tokens, int D, int bits) {
  __shared__ int64_t sid[DEC_TOK];
  const int64_t t0 = (int64_t)blockIdx.y * DEC_TOK;
  const int nt = (int)((tokens - t0) < DEC_TOK ? (tokens - t0) : DEC_TOK);
  if (threadIdx.x < nt) sid[threadIdx.x] = ids[t0 + threadIdx.x];
  __syncthreads();
  const int c = (blockIdx.x * 256 + threadIdx.x) * 2;
  if (c >= D) return;
  const bool two = c + 1 < D;
  if (!w_out) {                                  // identity projection (D == bits): the code itself
    for (int t = 0; t < nt; ++t) {
      const int64_t id = sid[t];
      out[(t0 + t) * D + c] = from_f<T>(((id >> (bits - 1 - c)) & 1) ? 1.f : -1.f);
      if (two) out[(t0 + t) * D + c + 1] = from_f<T>(((id >> (bits - 2 - c)) & 1) ? 1.f : -1.f);
    }
    return;
  }
  uint32_t w0[DEC_MAXB], w1[DEC_MAXB];
#pragma unroll
  for (int i = 0; i < DEC_MAXB; ++i) {
    w0[i] = i < bits ? __float_as_uint(__ldg(w_out + (int64_t)c * bits + i)) : 0u;
    w1[i] = (i < bits && two) ? __float_as_uint(__ldg(w_out + (int64_t)(c + 1) * bits + i)) : 0u;
  }
  const float b0 = b_out ? b_out[c] : 0.f, b1 = (b_out && two) ? b_out[c + 1] : 0.f;
  for (int t = 0; t < nt; ++t) {
    const uint32_t nid = ~(uint32_t)sid[t];       // bit set -> the code component is -1 -> flip the weight's sign
    float a0 = b0, a1 = b1;
#pragma unroll
    for (int i = 0; i < DEC_MAXB; ++i) {
      if (i < bits) {
        const uint32_t sg = ((nid >> (bits - 1 - i)) & 1u) << 31;
        a0 += __uint_as_float(w0[i] ^ sg); a1 += __uint_as_float(w1[i] ^ sg);
      }
    }
    T* o = out + (t0 + t) * D + c;
    if (two && (reinterpret_cast<uintptr_t>(o) % (2 * sizeof(T))) == 0) {
      if constexpr (sizeof(T) == 2) { __nv_bfloat162 v = __floats2bfloat162_rn(a0, a1); *reinterpret_cast<__nv_bfloat162*>(o) = v; }
      else *reinterpret_cast<float2*>(o) = make_float2(a0, a1);
    } else { o[0] = from_f<T>(a0); if (two) o[1] = from_f<T>(a1); }
  }
}

}  // namespace mmg

using namespace mmg;

template <typename T>
static int launch_lfq(const mmg_vq_lfq_encode_args* a, cudaStream_t st) {
  const size_t smem = a->w_in ? (size_t)a->bits * a->D * 4 : 0;
  MMG_CHECK_ARG(smem <= 200 * 1024, "mmg_vq_lfq_encode: projection does not fit in shared memory");
  const bool fast = a->w_in && a->D % 128 == 0 && (reinterpret_cast<uintptr_t>(a->x) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->w_in) & 15) == 0;
  const int per_block = fast ? 8 * LFQ_TOK : 8;
  int64_t grid = (a->T + per_block - 1) / per_block; if (grid > (int64_t)num_sms()) grid = num_sms();      // the projection is staged once per CTA
  auto launch = [&](auto kern) -> int {
    MMG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)grid, 256, smem, st>>>((const T*)a->x, a->w_in, a->b_in, a->ids, a->T, a->D, a->bits);
    MMG_LAUNCHED();
    return MMG_OK;
  };
  if (fast) return a->bits <= 16 ? launch(lfq_encode_kernel<T, 16>) : launch(lfq_encode_kernel<T, 24>);
  return launch(lfq_encode_generic_kernel<T, 24>);
}

extern "C" int mmg_vq_lfq_encode(const mmg_vq_lfq_encode_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->ids, "mmg_vq_lfq_encode: NULL pointer");
  MMG_CHECK_ARG(a->bits >= 1 && a->bits <= 24, "mmg_vq_lfq_encode: bits=%d not in [1,24]", a->bits);
  MMG_CHECK_ARG(a->w_in || a->D == a->bits, "mmg_vq_lfq_encode: identity projection needs D == bits");
  if (a->T == 0) return MMG_OK;
  if (a->dtype == MMG_BF16 && a->w_split && a->D % 64 == 0 && 3 * a->bits <= 64) {
    // bf16 tokens: the projection runs on wgmma as ONE HBM-bound TMA stream of the tokens against the 3-way bf16 split of project_in
    // ([hi | mid | lo] rows, hi + mid + lo == the fp32 weight), recombined in fp32 by the LFQ_IDS epilogue
    mmg_linear_args l{};
    l.a = a->x; l.w = a->w_split; l.M = a->T; l.N = 64; l.K = a->D; l.lda = a->D; l.ldw = a->D; l.dtype = MMG_BF16; l.epilogue = MMG_EPI_LFQ_IDS;
    l.epi.out = a->ids; l.epi.ldo = 1; l.epi.out_dtype = MMG_F32; l.epi.bias = a->b_in; l.epi.ln_width = a->bits;
    return mmg_linear(&l, stream);
  }
  return a->dtype == MMG_BF16 ? launch_lfq<bf16>(a, st) : launch_lfq<float>(a, st);
}

extern "C" int mmg_vq_l2_argmin(const mmg_vq_l2_argmin_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->codebook && a->ids, "mmg_vq_l2_argmin: NULL pointer");
  MMG_CHECK_ARG(a->K >= 1 && a->D >= 1, "mmg_vq_l2_argmin: K, D");
  if (a->T == 0) return MMG_OK;
  unsigned long long* best = reinterpret_cast<unsigned long long*>(a->ids);       // ids double as the packed (distance, code) keys
  const unsigned nb = (unsigned)((a->T + 255) / 256);
  vq_init_kernel<<<nb, 256, 0, st>>>(best, a->T);
  MMG_LAUNCHED();
  dim3 grid((unsigned)((a->T + 63) / 64), (unsigned)((a->K + 63) / 64));
  MMG_CHECK_ARG(grid.y < 65536, "mmg_vq_l2_argmin: K too large");
  vq_l2_argmin_kernel<<<grid, 256, 0, st>>>(a->x, a->codebook, best, a->T, a->K, a->D);
  MMG_LAUNCHED();
  vq_finish_kernel<<<nb, 256, 0, st>>>(best, a->T);
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_vq_decode_codes(const mmg_vq_decode_codes_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->ids && a->out, "mmg_vq_decode_codes: NULL pointer");
  MMG_CHECK_ARG(a->bits >= 1 && a->bits <= DEC_MAXB && (a->w_out || a->D == a->bits), "mmg_vq_decode_codes: bits (<= 24) / identity projection");
  if (a->T == 0) return MMG_OK;
  const dim3 grid((unsigned)((a->D + 511) / 512), (unsigned)((a->T + DEC_TOK - 1) / DEC_TOK));
  if (a->dtype == MMG_BF16) vq_decode_codes_kernel<bf16><<<grid, 256, 0, st>>>(a->ids, a->w_out, a->b_out, (bf16*)a->out, a->T, a->D, a->bits);
  else vq_decode_codes_kernel<float><<<grid, 256, 0, st>>>(a->ids, a->w_out, a->b_out, (float*)a->out, a->T, a->D, a->bits);
  MMG_LAUNCHED();
  return MMG_OK;
}

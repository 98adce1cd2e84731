// T5 text encoder kernels (HF T5EncoderModel, eval mode; the text step of MaskGit.generate, t5.py:60-99):
//   * mmg_t5_attention, dtype MMG_BF16 -> wgmma kernel below: relative-position-bias self-attention, d_kv = 64, no scaling, exact two-pass
//     softmax; q / k / v come by TMA straight out of the token-major output of the fused q|k|v projection;
//   * mmg_t5_attention, dtype MMG_F32  -> fp32 CUDA-core kernel with the same semantics (precision="fp32");
//   * mmg_rmsnorm: T5LayerNorm, fp32 statistics, optional zero-fill of padding rows.
#include "mmg_common.cuh"
#include "mmg_sm90.cuh"
#include "mmg_tmap.cuh"
#include <mutex>
#include <float.h>

namespace mmg {

constexpr int T5_MAX_T = 512;
constexpr int T5_KB = 64;                               // keys per block
constexpr int T5_LD = T5_KB + 4;                        // staging row stride (floats)
constexpr int T5_BIAS_N = 2 * T5_MAX_T + T5_KB;         // bias table: index key - query + T - 1, padded for the keys past T of the last block
constexpr size_t T5_SMEM = 1024 + 16384 + 2 * 8192 + 16384 + (size_t)128 * T5_LD * 4 + T5_BIAS_N * 4 + 64;
constexpr float T5_LOG2E = 1.4426950408889634f;

struct alignas(64) T5AttnParams {
  CUtensorMap tma_q;        // qkv as [B*T, 3*inner] bf16, boxes of 128 rows x 64 columns (one head of q for 128 queries)
  CUtensorMap tma_kv;       // the same matrix, boxes of 64 rows x 64 columns (one head of k or v for 64 keys)
  const uint8_t* key_mask;  // [B, T] or NULL
  const int32_t* rel_bucket; const float* rel_bias;
  bf16* out;
  int T, heads, inner, nb, KB_tail;   // nb blocks of 64 keys over [0, T); the last holds KB_tail (multiple of 32) of them
  int64_t ldo;
};

// One CTA = one (batch, head, 128-query tile); warps 0-3 are the softmax warpgroup (wgmma, then thread = query row), warp 4 issues the TMA
// loads.  The keys of the sequence are walked in blocks of 64, twice:
//   pass A:  S = Q K^T + bias -> per-row maximum;
//   pass B:  S again -> p = exp2((s - max) log2e) -> P (bf16, shared memory, K-major SWIZZLE_128B) -> O += P V (wgmma), row sums in fp32.
// Scores: s = q.k + bias[h, bucket(j - i)] for a live key, -FLT_MAX (HF's finfo.min, which swamps the bias) for a masked one; keys past the
// end of the sequence (rows of the next sequence in the projection output) are excluded by index.  A row with no live key therefore sees T
// equal scores and averages v, as HF does.
__global__ void __launch_bounds__(160, 1)
t5_attention_tc_kernel(const __grid_constant__ T5AttnParams p) {
  using namespace sm90;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;                    // 128 x 64 bf16
  uint8_t* sK = sQ + 16384;              // 64 x 64
  uint8_t* sV = sK + 8192;
  uint8_t* sP = sV + 8192;               // 128 x 64 bf16
  float* stg = reinterpret_cast<float*>(sP + 16384);     // 128 x T5_LD fp32: S of a block, finally O
  float* sbias = stg + 128 * T5_LD;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sbias + T5_BIAS_N);
  uint64_t* bar_q = bars + 0; uint64_t* bar_kv = bars + 1; uint64_t* bar_free = bars + 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg_role = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int bh = blockIdx.y, b = bh / p.heads, h = bh % p.heads;
  const int q0 = blockIdx.x * 128;
  const int T = p.T;
  const int row0 = b * T;

  if (warp == 4 && lane == 0) {
    prefetch_tmap(&p.tma_q); prefetch_tmap(&p.tma_kv);
    mbar_init(bar_q, 1); mbar_init(bar_kv, 1); mbar_init(bar_free, 4);
    fence_barrier_init();
  }
  // this head's bias as a function of d = key - query: sbias[d + T - 1] = rel_bias[bucket[d + T - 1], h]
  for (int i = threadIdx.x; i < T5_BIAS_N; i += blockDim.x)
    sbias[i] = i < 2 * T - 1 ? __ldg(p.rel_bias + (int64_t)__ldg(p.rel_bucket + i) * p.heads + h) : 0.f;
  __syncthreads();

  if (wg_role == 1) {
    if (elect_one()) {
      mbar_expect_tx(bar_q, 16384);
      tma_load_2d(sQ, &p.tma_q, bar_q, h * 64, row0 + q0);
      uint32_t ph_free = 0;
      int loads = 0;
      for (int pass = 0; pass < 2; ++pass) {
        for (int blk = 0; blk < p.nb; ++blk, ++loads) {
          if (loads) { mbar_wait(bar_free, ph_free); ph_free ^= 1; }
          const int krow = row0 + blk * T5_KB;
          mbar_expect_tx(bar_kv, pass == 0 ? 8192 : 16384);
          tma_load_2d(sK, &p.tma_kv, bar_kv, p.inner + h * 64, krow);
          if (pass == 1) tma_load_2d(sV, &p.tma_kv, bar_kv, 2 * p.inner + h * 64, krow);
        }
      }
    }
    __syncwarp();
  } else {
    const int r = warp * 32 + lane;
    const int qi = q0 + r;
    const int qc = qi < T ? qi : T - 1;                  // rows past T are computed (and dropped) with the last row's bias
    const float* srow = stg + r * T5_LD;
    const float* brow = sbias + (T - 1 - qc);            // brow[j] = bias(j - qc)
    const uint8_t* km = p.key_mask ? p.key_mask + row0 : nullptr;
    uint32_t ph_kv = 0;
    float row_max = -FLT_MAX, row_sum = 0.f;
    float o_acc[2][32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { o_acc[0][i] = 0.f; o_acc[1][i] = 0.f; }
    mbar_wait(bar_q, 0);
    const uint64_t qdesc = smem_desc_kmajor_sw128(smem_u32(sQ));
    const uint64_t kdesc = smem_desc_kmajor_sw128(smem_u32(sK));
    for (int pass = 0; pass < 2; ++pass) {
      for (int blk = 0; blk < p.nb; ++blk) {
        mbar_wait(bar_kv, ph_kv); ph_kv ^= 1;
        {   // S = Q K^T for the 128 query rows (two m64 halves), staged row-major
          float s_acc[2][32];
          wgmma_fence();
#pragma unroll
          for (int mh = 0; mh < 2; ++mh)
#pragma unroll
            for (int k = 0; k < 4; ++k) Wgmma<64>::template mma<0>(s_acc[mh], qdesc + (uint64_t)(mh * 512 + k * 2), kdesc + (uint64_t)(k * 2), k ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(s_acc[0]); reg_fence(s_acc[1]);
          named_sync(1, 128);                              // every row of the previous block's S has been read
          stage_acc<32, T5_LD>(s_acc[0], stg, 0, 64);
          stage_acc<32, T5_LD>(s_acc[1], stg + 64 * T5_LD, 0, 64);
          named_sync(1, 128);
        }
        const int kb_cur = blk == p.nb - 1 ? p.KB_tail : T5_KB;
        for (int c = 0; c < kb_cur; c += 32) {
          float s[32];
          stage_ld32(srow + c, s);
          const int j0 = blk * T5_KB + c;
          // keys of this chunk inside the sequence (inw) and live (livew), one ballot word each: lane l tests key j0 + l
          uint32_t inw = 0xffffffffu, livew = 0xffffffffu;
          if (km || j0 + 32 > T) {
            const int jl = j0 + lane;
            inw = __ballot_sync(0xffffffffu, jl < T);
            livew = __ballot_sync(0xffffffffu, jl < T && (!km || km[jl]));
          }
#pragma unroll
          for (int i = 0; i < 32; ++i) s[i] = ((livew >> i) & 1u) ? s[i] + brow[j0 + i] : -FLT_MAX;
          if (pass == 0) {
#pragma unroll
            for (int i = 0; i < 32; ++i) if ((inw >> i) & 1u) row_max = fmaxf(row_max, s[i]);
          } else {
            uint32_t packed[16];
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
              // (s - max) first: a masked score minus a finite maximum rounds to -FLT_MAX and its weight to 0; with every key masked the
              // difference is exactly 0 and every key weighs 1
              const float p0 = ((inw >> i) & 1u) ? ex2_fast((s[i] - row_max) * T5_LOG2E) : 0.f;
              const float p1 = ((inw >> (i + 1)) & 1u) ? ex2_fast((s[i + 1] - row_max) * T5_LOG2E) : 0.f;
              __nv_bfloat162 t = __floats2bfloat162_rn(p0, p1);
              packed[i >> 1] = *reinterpret_cast<uint32_t*>(&t);
              const float2 pr = __bfloat1622float2(t);       // normalise by the sum of the ROUNDED weights: O = sum(p~ v) / sum(p~)
              row_sum += pr.x + pr.y;
            }
            // P[r, c .. c+31] -> 16-byte chunks c / 8 .. +3 of row r, 128B swizzle: chunk ^= (r & 7)
            uint8_t* tile = sP + r * 128;
            const int ch0 = c >> 3;
#pragma unroll
            for (int q4 = 0; q4 < 4; ++q4) {
              const int ch = (ch0 + q4) ^ (r & 7);
              *reinterpret_cast<uint4*>(tile + ch * 16) = make_uint4(packed[q4 * 4], packed[q4 * 4 + 1], packed[q4 * 4 + 2], packed[q4 * 4 + 3]);
            }
          }
        }
        if (pass == 1) {
          fence_proxy_async();                 // generic-proxy smem writes of P -> visible to the tensor core (async proxy)
          named_sync(1, 128);
          const int ksteps = kb_cur / 16;
          for (int ks = 0; ks < ksteps; ++ks) {
            wgmma_fence();
            const uint32_t pa = smem_u32(sP) + ks * 32;
            const uint64_t vdesc = smem_desc_mnmajor_sw128(smem_u32(sV) + ks * 2048, 1024);
            Wgmma<64>::template mma<1>(o_acc[0], smem_desc_kmajor_sw128(pa), vdesc, 1u);
            Wgmma<64>::template mma<1>(o_acc[1], smem_desc_kmajor_sw128(pa + 8192), vdesc, 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(o_acc[0]); reg_fence(o_acc[1]);
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_free);    // K / V / P of this block are no longer needed
      }
    }
    named_sync(1, 128);
    stage_acc<32, T5_LD>(o_acc[0], stg, 0, 64);
    stage_acc<32, T5_LD>(o_acc[1], stg + 64 * T5_LD, 0, 64);
    named_sync(1, 128);
    if (qi < T) {
      const float inv = 1.f / row_sum;
      bf16* dst = p.out + (int64_t)(row0 + qi) * p.ldo + h * 64;
#pragma unroll
      for (int c = 0; c < 64; c += 32) {
        float o[32];
        stage_ld32(srow + c, o);
#pragma unroll
        for (int i = 0; i < 32; i += 8)
          *reinterpret_cast<uint4*>(dst + c + i) = make_uint4(pack_bf16(o[i] * inv, o[i + 1] * inv), pack_bf16(o[i + 2] * inv, o[i + 3] * inv),
                                                              pack_bf16(o[i + 4] * inv, o[i + 5] * inv), pack_bf16(o[i + 6] * inv, o[i + 7] * inv));
      }
    }
  }
}

// fp32 (precision="fp32"): one thread per query row, K / V tiles of 32 keys staged in shared memory, online softmax with expf.
__global__ void __launch_bounds__(128)
t5_attention_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, const uint8_t* __restrict__ key_mask,
                        const int32_t* __restrict__ rel_bucket, const float* __restrict__ rel_bias, int T, int heads, int64_t ldqkv, int64_t ldo) {
  __shared__ float Ks[32][64];
  __shared__ float Vs[32][64];
  __shared__ float Bs[2 * T5_MAX_T];
  __shared__ uint8_t Ms[32];
  const int bh = blockIdx.y, b = bh / heads, h = bh % heads, inner = heads * 64;
  const int qi = blockIdx.x * 128 + threadIdx.x;
  const bool active = qi < T;
  const int qc = active ? qi : T - 1;
  const int64_t row0 = (int64_t)b * T;
  for (int i = threadIdx.x; i < 2 * T - 1; i += blockDim.x) Bs[i] = rel_bias[(int64_t)rel_bucket[i] * heads + h];
  float qr[64], o[64];
  const float* qrow = qkv + (row0 + qc) * ldqkv + h * 64;
#pragma unroll
  for (int d = 0; d < 64; ++d) { qr[d] = qrow[d]; o[d] = 0.f; }
  float m = -FLT_MAX, l = 0.f;
  for (int j0 = 0; j0 < T; j0 += 32) {
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * 64; i += 128) {
      const int j = j0 + i / 64, d = i % 64;
      const float* kv = qkv + (row0 + j) * ldqkv + h * 64 + d;
      Ks[i / 64][d] = j < T ? kv[inner] : 0.f;
      Vs[i / 64][d] = j < T ? kv[2 * inner] : 0.f;
    }
    if (threadIdx.x < 32) {
      const int j = j0 + threadIdx.x;
      Ms[threadIdx.x] = j < T ? ((!key_mask || key_mask[row0 + j]) ? 1 : 0) : 2;     // 2: past the end of the sequence
    }
    __syncthreads();
    float s[32]; float tm = -FLT_MAX;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) acc = fmaf(qr[d], Ks[j][d], acc);
      acc = Ms[j] == 1 ? acc + Bs[j0 + j - qc + T - 1] : -FLT_MAX;      // HF: scores + (bias + finfo.min) == finfo.min for a masked key
      s[j] = acc;
      if (Ms[j] != 2) tm = fmaxf(tm, acc);
    }
    const float mn = fmaxf(m, tm);
    const float corr = expf(m - mn);
    l *= corr;
#pragma unroll
    for (int d = 0; d < 64; ++d) o[d] *= corr;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (Ms[j] == 2) continue;
      const float pj = expf(s[j] - mn);
      l += pj;
#pragma unroll
      for (int d = 0; d < 64; ++d) o[d] = fmaf(pj, Vs[j][d], o[d]);
    }
    m = mn;
  }
  if (active) {
    const float inv = 1.f / l;
    float* orow = out + (row0 + qi) * ldo + h * 64;
#pragma unroll
    for (int d = 0; d < 64; ++d) orow[d] = o[d] * inv;
  }
}

// RMSNorm: one warp per row, two sweeps over the row (sum of squares, then scale; the second reads from L1 / L2), 16-byte accesses.
template <typename TY> __device__ __forceinline__ void st4(TY* p, float a, float b, float c, float d);
template <> __device__ __forceinline__ void st4<float>(float* p, float a, float b, float c, float d) { *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d); }
template <> __device__ __forceinline__ void st4<bf16>(bf16* p, float a, float b, float c, float d) { *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16(a, b), pack_bf16(c, d)); }

template <typename TY>
__global__ void __launch_bounds__(256)
rmsnorm_kernel(const float* __restrict__ x, TY* __restrict__ y, const float* __restrict__ w, const uint8_t* __restrict__ row_mask,
               int64_t rows, int d, int64_t ldx, int64_t ldy, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  TY* yr = y + row * ldy;
  if (row_mask && !row_mask[row]) {
    for (int c = lane * 4; c < d; c += 128) st4<TY>(yr + c, 0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float* xr = x + row * ldx;
  float ss = 0.f;
  for (int c = lane * 4; c < d; c += 128) {
    const float4 t = *reinterpret_cast<const float4*>(xr + c);
    ss = fmaf(t.x, t.x, ss); ss = fmaf(t.y, t.y, ss); ss = fmaf(t.z, t.z, ss); ss = fmaf(t.w, t.w, ss);
  }
  ss = warp_sum(ss);
  const float r = rsqrtf(ss / (float)d + eps);
  for (int c = lane * 4; c < d; c += 128) {
    const float4 t = *reinterpret_cast<const float4*>(xr + c);
    const float4 g = __ldg(reinterpret_cast<const float4*>(w + c));
    st4<TY>(yr + c, g.x * (t.x * r), g.y * (t.y * r), g.z * (t.z * r), g.w * (t.w * r));
  }
}

}  // namespace mmg

using namespace mmg;

extern "C" int mmg_t5_attention(const mmg_t5_attention_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->qkv && a->out && a->rel_bucket && a->rel_bias, "mmg_t5_attention: NULL pointer");
  MMG_CHECK_ARG(a->B > 0 && a->heads > 0 && a->num_buckets > 0 && a->T >= 1 && a->T <= T5_MAX_T, "mmg_t5_attention: bad shape B=%d T=%d heads=%d (T <= %d)",
                a->B, a->T, a->heads, T5_MAX_T);
  MMG_CHECK_ARG((int64_t)a->B * a->heads < 65536 && (int64_t)a->B * a->T < (1ll << 31), "mmg_t5_attention: B * heads or B * T too large");
  const int inner = a->heads * 64;
  MMG_CHECK_ARG(a->ldqkv >= 3 * (int64_t)inner && a->ldo >= inner, "mmg_t5_attention: ldqkv >= 3 * heads * 64, ldo >= heads * 64");
  const dim3 grid((a->T + 127) / 128, (unsigned)(a->B * a->heads));
  if (a->dtype == MMG_F32) {
    t5_attention_f32_kernel<<<grid, 128, 0, st>>>((const float*)a->qkv, (float*)a->out, a->key_mask, a->rel_bucket, a->rel_bias, a->T, a->heads,
                                                  a->ldqkv, a->ldo);
    simt_launch_counter()++;
    MMG_LAUNCHED();
    return MMG_OK;
  }
  MMG_CHECK_ARG(a->dtype == MMG_BF16, "mmg_t5_attention: dtype %d", a->dtype);
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  MMG_CHECK_ARG(al(a->qkv) && al(a->out) && a->ldqkv % 8 == 0 && a->ldo % 8 == 0, "mmg_t5_attention: bf16 needs 16-byte aligned qkv / out and row strides %% 8");
  T5AttnParams p{};
  const int full = a->T / T5_KB, rem = a->T - full * T5_KB;
  p.nb = rem ? full + 1 : full; p.KB_tail = rem ? (rem + 31) / 32 * 32 : T5_KB;
  p.key_mask = a->key_mask; p.rel_bucket = a->rel_bucket; p.rel_bias = a->rel_bias; p.out = (bf16*)a->out;
  p.T = a->T; p.heads = a->heads; p.inner = inner; p.ldo = a->ldo;
  uint64_t dims[2] = {3 * (uint64_t)inner, (uint64_t)a->B * a->T}; uint64_t str[1] = {(uint64_t)a->ldqkv * 2};
  { uint32_t box[2] = {64, 128}; int rc = make_tmap_bf16(&p.tma_q, a->qkv, 2, dims, str, box); if (rc) return rc; }
  { uint32_t box[2] = {64, T5_KB}; int rc = make_tmap_bf16(&p.tma_kv, a->qkv, 2, dims, str, box); if (rc) return rc; }
  static std::once_flag once; static cudaError_t err = cudaSuccess;
  std::call_once(once, [] { err = cudaFuncSetAttribute(t5_attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T5_SMEM); });
  if (err != cudaSuccess) return fail(MMG_ECUDA, "cudaFuncSetAttribute(t5_attention_tc): %s", cudaGetErrorString(err));
  t5_attention_tc_kernel<<<grid, 160, T5_SMEM, st>>>(p);
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_rmsnorm(const mmg_rmsnorm_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->y && a->w, "mmg_rmsnorm: NULL pointer");
  MMG_CHECK_ARG(a->d > 0 && a->d % 4 == 0 && a->d < (1 << 30) && a->ldx % 4 == 0 && a->ldy % 4 == 0 && a->ldx >= a->d && a->ldy >= a->d,
                "mmg_rmsnorm: d %% 4, ldx %% 4, ldy %% 4, ld >= d");
  MMG_CHECK_ARG((reinterpret_cast<uintptr_t>(a->x) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->w) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(a->y) & (a->y_dtype == MMG_BF16 ? 7 : 15)) == 0, "mmg_rmsnorm: x / w / y alignment");
  MMG_CHECK_ARG(a->y_dtype == MMG_F32 || a->y_dtype == MMG_BF16, "mmg_rmsnorm: y_dtype %d", a->y_dtype);
  if (a->rows == 0) return MMG_OK;
  const unsigned grid = (unsigned)((a->rows + 7) / 8);
  if (a->y_dtype == MMG_BF16) rmsnorm_kernel<bf16><<<grid, 256, 0, st>>>(a->x, (bf16*)a->y, a->w, a->row_mask, a->rows, (int)a->d, a->ldx, a->ldy, a->eps);
  else rmsnorm_kernel<float><<<grid, 256, 0, st>>>(a->x, (float*)a->y, a->w, a->row_mask, a->rows, (int)a->d, a->ldx, a->ldy, a->eps);
  MMG_LAUNCHED();
  return MMG_OK;
}

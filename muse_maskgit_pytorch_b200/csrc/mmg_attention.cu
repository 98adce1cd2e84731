// Attention core (dh = 64): out = softmax(scale * q k^T + mask) v over keys [0, Tk), key 0 = learned null key.
// replaces Attend.forward / flash_attn (attend.py:66-140).
//   * mmg_attention with dtype MMG_F32  -> fp32 CUDA-core kernel (parity precision)
//   * mmg_attention with dtype MMG_BF16 -> wgmma kernel (mmg_attention_tc.cuh): S = Q K^T and O = P V on the tensor
//     cores; the softmax runs on the S accumulator fragments and feeds P to the P V product as a register operand, O stays in
//     registers through the epilogue; a producer warp keeps a ring of K / V stages loading under the math.
#include "mmg_common.cuh"
#include "mmg_attention_tc.cuh"
#include "mmg_attention_split.cuh"
#include "mmg_tmap.cuh"
#include <mutex>
#include <float.h>

namespace mmg {

// One thread per query row; K/V tiles of 32 keys staged in shared memory (broadcast reads); online softmax per tile.
template <typename T>
__global__ void __launch_bounds__(128)
attention_simt_kernel(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, T* __restrict__ out,
                      const uint8_t* __restrict__ key_mask, int heads, int Tq, int Tk, int Tk_alloc, int64_t ldo, int kv_shared, float scale) {
  __shared__ float Ks[32][64];
  __shared__ float Vs[32][64];
  __shared__ uint8_t Ms[32];
  const int bh = blockIdx.y, b = bh / heads, h = bh % heads;
  const int qi = blockIdx.x * 128 + threadIdx.x;
  const bool active = qi < Tq;
  const T* kb = k + (int64_t)(kv_shared ? h : bh) * Tk_alloc * 64;
  const T* vb = v + (int64_t)(kv_shared ? h : bh) * Tk_alloc * 64;
  float qr[64], o[64];
#pragma unroll
  for (int d = 0; d < 64; ++d) { qr[d] = active ? to_f(q[((int64_t)bh * Tq + qi) * 64 + d]) : 0.f; o[d] = 0.f; }
  float m = -FLT_MAX, l = 0.f;
  for (int j0 = 0; j0 < Tk; j0 += 32) {
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * 64; i += 128) {
      const int j = j0 + i / 64, d = i % 64;
      Ks[i / 64][d] = j < Tk ? to_f(kb[(int64_t)j * 64 + d]) : 0.f;
      Vs[i / 64][d] = j < Tk ? to_f(vb[(int64_t)j * 64 + d]) : 0.f;
    }
    if (threadIdx.x < 32) {
      const int j = j0 + threadIdx.x;
      // key 0 (null) is never masked: F.pad(mask, (1, 0), value=True)  muse_maskgit_pytorch.py:157
      Ms[threadIdx.x] = (j < Tk) ? ((j == 0 || !key_mask) ? 1 : key_mask[(int64_t)b * (Tk - 1) + (j - 1)]) : 2;
    }
    __syncthreads();
    float s[32]; float tm = -FLT_MAX;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) acc = fmaf(qr[d], Ks[j][d], acc);
      acc *= scale;
      if (Ms[j] == 0) acc = -FLT_MAX;          // masked_fill(~mask, -finfo.max)  attend.py:128-129
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
      const float p = expf(s[j] - mn);
      l += p;
#pragma unroll
      for (int d = 0; d < 64; ++d) o[d] = fmaf(p, Vs[j][d], o[d]);
    }
    m = mn;
  }
  if (active) {
    const float inv = 1.f / l;
    T* orow = out + ((int64_t)b * Tq + qi) * ldo + h * 64;
#pragma unroll
    for (int d = 0; d < 64; ++d) orow[d] = from_f<T>(o[d] * inv);
  }
}

template <int KB>
static int attn_launch(const AttnTcParams& p, dim3 grid, cudaStream_t st) {
  constexpr size_t smem = attn_smem_bytes(KB);
  static std::once_flag once; static cudaError_t err = cudaSuccess;
  std::call_once(once, [] { err = cudaFuncSetAttribute(attention_tc_kernel<KB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); });
  if (err != cudaSuccess) return fail(MMG_ECUDA, "cudaFuncSetAttribute(attention_tc): %s", cudaGetErrorString(err));
  MMG_CUDA(launch_pdl(attention_tc_kernel<KB>, grid, dim3(ATTN_THREADS), smem, st, p));
  MMG_LAUNCHED();
  return MMG_OK;
}

int attention_tc_launch(const mmg_attention_args* a, cudaStream_t st) {
  AttnTcParams p{};
  attn_blocks(a->Tk - 1, &p.nb, &p.KB, &p.KB_tail);         // blocks over the real keys 1 .. Tk-1; the null key (row 0) is handled by the softmax warps
  p.k = (const bf16*)a->k; p.v = (const bf16*)a->v;
  p.key_mask = a->key_mask; p.out = (bf16*)a->out; p.heads = a->heads; p.Tq = a->Tq; p.Tk = a->Tk; p.Tk_alloc = a->Tk_alloc;
  p.kv_shared = a->kv_batch_stride_zero; p.ldo = a->ldo; p.scale_log2e = a->scale * 1.4426950408889634f;
  // single-pass softmax when the caller bounds |q.k| and exp2((s - bound) * scale * log2e) cannot underflow the fp32 range
  p.smax = a->logit_bound;
  p.single_pass = (a->logit_bound > 0.f && a->scale > 0.f && 2.f * a->logit_bound * p.scale_log2e < 100.f) ? 1 : 0;
  const uint64_t BH = (uint64_t)a->B * a->heads;
  const uint64_t kv_heads = a->kv_batch_stride_zero ? (uint64_t)a->heads : BH;
  {
    uint64_t dims[2] = {64, BH * (uint64_t)a->Tq}; uint64_t str[1] = {128}; uint32_t box[2] = {64, 128};
    int rc = make_tmap_bf16(&p.tma_q, a->q, 2, dims, str, box); if (rc) return rc;
  }
  {
    uint64_t dims[2] = {64, kv_heads * (uint64_t)a->Tk_alloc}; uint64_t str[1] = {128}; uint32_t box[2] = {64, (uint32_t)p.KB};
    int rc = make_tmap_bf16(&p.tma_k, a->k, 2, dims, str, box); if (rc) return rc;
    rc = make_tmap_bf16(&p.tma_v, a->v, 2, dims, str, box); if (rc) return rc;
  }
  dim3 grid((a->Tq + 127) / 128, (unsigned)BH);
  if (p.KB == 64) return attn_launch<64>(p, grid, st);
  return attn_launch<128>(p, grid, st);
}

// fp32 parity on the tensor cores: q / k / v arrive as 3-way bf16 splits (384 columns per row), see mmg_attention_split.cuh
static int attention_split_launch(const mmg_attention_args* a, cudaStream_t st) {
  AttnSplitParams p{};
  const int full = a->Tk / AS_KB, rem = a->Tk - full * AS_KB;
  p.nb = rem ? full + 1 : full; p.KB_tail = rem ? (rem + 31) / 32 * 32 : AS_KB;
  p.key_mask = a->key_mask; p.out = (float*)a->out; p.heads = a->heads; p.Tq = a->Tq; p.Tk = a->Tk; p.Tk_alloc = a->Tk_alloc;
  p.kv_shared = a->kv_batch_stride_zero; p.ldo = a->ldo; p.scale_log2e = a->scale * 1.4426950408889634f;
  const uint64_t BH = (uint64_t)a->B * a->heads;
  const uint64_t kv_heads = a->kv_batch_stride_zero ? (uint64_t)a->heads : BH;
  uint64_t str[1] = {768};
  { uint64_t dims[2] = {384, BH * (uint64_t)a->Tq}; uint32_t box[2] = {64, 128};
    int rc = make_tmap_bf16(&p.tma_q, a->q, 2, dims, str, box); if (rc) return rc; }
  { uint64_t dims[2] = {384, kv_heads * (uint64_t)a->Tk_alloc}; uint32_t box[2] = {64, AS_KB};
    int rc = make_tmap_bf16(&p.tma_k, a->k, 2, dims, str, box); if (rc) return rc;
    rc = make_tmap_bf16(&p.tma_v, a->v, 2, dims, str, box); if (rc) return rc; }
  static std::once_flag once; static cudaError_t err = cudaSuccess;
  std::call_once(once, [] { err = cudaFuncSetAttribute(attention_tc_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM); });
  if (err != cudaSuccess) return fail(MMG_ECUDA, "cudaFuncSetAttribute(attention_tc_split): %s", cudaGetErrorString(err));
  dim3 grid((a->Tq + 127) / 128, (unsigned)BH);
  attention_tc_split_kernel<<<grid, 160, AS_SMEM, st>>>(p);
  MMG_LAUNCHED();
  return MMG_OK;
}

}  // namespace mmg

using namespace mmg;

extern "C" int mmg_attention(const mmg_attention_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->q && a->k && a->v && a->out, "mmg_attention: NULL pointer");
  MMG_CHECK_ARG(a->B > 0 && a->heads > 0 && a->Tq > 0 && a->Tk > 0 && a->Tk_alloc >= a->Tk, "mmg_attention: bad shape");
  if (a->split3) {
    MMG_CHECK_ARG(a->dtype == MMG_BF16 && attention_tc_supported(a) && (a->ldo % 4) == 0, "mmg_attention: split3 needs bf16 split operands, 16-byte aligned pointers, ldo %% 4");
    return attention_split_launch(a, st);
  }
  if (a->dtype == MMG_BF16 && attention_tc_supported(a)) return attention_tc_launch(a, st);
  dim3 grid((a->Tq + 127) / 128, a->B * a->heads);
  if (a->dtype == MMG_BF16)
    attention_simt_kernel<bf16><<<grid, 128, 0, st>>>((const bf16*)a->q, (const bf16*)a->k, (const bf16*)a->v, (bf16*)a->out, a->key_mask,
                                                        a->heads, a->Tq, a->Tk, a->Tk_alloc, a->ldo, a->kv_batch_stride_zero, a->scale);
  else
    attention_simt_kernel<float><<<grid, 128, 0, st>>>((const float*)a->q, (const float*)a->k, (const float*)a->v, (float*)a->out, a->key_mask,
                                                         a->heads, a->Tq, a->Tk, a->Tk_alloc, a->ldo, a->kv_batch_stride_zero, a->scale);
  simt_launch_counter()++;
  MMG_LAUNCHED();
  return MMG_OK;
}

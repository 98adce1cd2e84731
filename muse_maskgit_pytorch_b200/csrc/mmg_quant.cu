// mmg_quantize_e4m3_images: per-image e4m3 quantisation of a bf16 NHWC map (the A operand of the e4m3 convolutions, precision="fp8").
//   amax_b = max |x| over image b, taken as an integer max over the bits of |x| (order-independent, so bitwise reproducible);
//   inv = amax_b == 0 ? 0 : 448 / amax_b (IEEE division);  q = cvt.rn.satfinite.e4m3(x * inv);  scale_b = amax_b / 448.
// Three launches: the per-image maxima (atomicMax on the fp32 bits of |x|, kept in `scale`, which a memset zeroes first), the
// quantisation, and the conversion of the maxima into scales.
#include "mmg_common.cuh"

namespace mmg {

constexpr int QZ_THREADS = 256;

// |x| of eight bf16 -> the largest as fp32 bits (a bf16 is the top half of an fp32; non-negative floats order like their bits)
__device__ __forceinline__ uint32_t amax_bits8(const uint4 v) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) m = max(m, max(w[i] & 0x7fffu, (w[i] >> 16) & 0x7fffu));
  return m << 16;
}

__global__ void __launch_bounds__(QZ_THREADS)
image_amax_kernel(const uint4* __restrict__ x, uint32_t* __restrict__ amax_bits, int64_t n8) {
  pdl_wait(); pdl_trigger();
  const int b = blockIdx.y;
  const uint4* xb = x + (int64_t)b * n8;
  uint32_t m = 0;
  for (int64_t i = (int64_t)blockIdx.x * QZ_THREADS + threadIdx.x; i < n8; i += (int64_t)gridDim.x * QZ_THREADS) m = max(m, amax_bits8(__ldg(xb + i)));
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ uint32_t s_m[QZ_THREADS / 32];
  if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 1; i < QZ_THREADS / 32; ++i) m = max(m, s_m[i]);
    if (m) atomicMax(amax_bits + b, m);
  }
}

__global__ void __launch_bounds__(QZ_THREADS)
image_quant_kernel(const uint4* __restrict__ x, uint2* __restrict__ q, const uint32_t* __restrict__ amax_bits, int64_t n8) {
  pdl_wait(); pdl_trigger();
  const int b = blockIdx.y;
  const float amax = __uint_as_float(amax_bits[b]);
  const float inv = amax == 0.f ? 0.f : 448.f / amax;
  const uint4* xb = x + (int64_t)b * n8;
  uint2* qb = q + (int64_t)b * n8;
  for (int64_t i = (int64_t)blockIdx.x * QZ_THREADS + threadIdx.x; i < n8; i += (int64_t)gridDim.x * QZ_THREADS) {
    const uint4 v = __ldg(xb + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float2 lo = make_float2(__uint_as_float(w[2 * h] << 16) * inv, __uint_as_float(w[2 * h] & 0xffff0000u) * inv);
      const float2 hi = make_float2(__uint_as_float(w[2 * h + 1] << 16) * inv, __uint_as_float(w[2 * h + 1] & 0xffff0000u) * inv);
      o[h] = (uint32_t)__nv_cvt_float2_to_fp8x2(lo, __NV_SATFINITE, __NV_E4M3) | ((uint32_t)__nv_cvt_float2_to_fp8x2(hi, __NV_SATFINITE, __NV_E4M3) << 16);
    }
    qb[i] = make_uint2(o[0], o[1]);
  }
}

__global__ void image_scale_kernel(float* __restrict__ scale, int B) {
  pdl_wait(); pdl_trigger();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) scale[b] = scale[b] / 448.f;          // the slot holds amax_b (its bits) until here
}

}  // namespace mmg

using namespace mmg;

extern "C" int mmg_quantize_e4m3_images(const mmg_quantize_e4m3_images_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->q && a->scale, "mmg_quantize_e4m3_images: NULL operand");
  MMG_CHECK_ARG(a->B > 0 && a->B < 65536 && a->hw > 0 && a->C > 0 && a->C % 8 == 0,
                "mmg_quantize_e4m3_images: bad shape B=%lld hw=%lld C=%d (0 < B < 65536, C %% 8 == 0)", (long long)a->B, (long long)a->hw, a->C);
  MMG_CHECK_ARG((reinterpret_cast<uintptr_t>(a->x) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->q) & 15) == 0,
                "mmg_quantize_e4m3_images: x and q need 16-byte alignment");
  const int64_t n8 = a->hw * a->C / 8;                         // 16-byte chunks of one image
  int64_t bx = (n8 + 8 * QZ_THREADS - 1) / (8 * QZ_THREADS);   // >= 8 chunks per thread
  const int64_t cap = (4 * num_sms() + a->B - 1) / a->B;        // about four CTAs per SM over all images
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  const dim3 grid((unsigned)bx, (unsigned)a->B);
  uint32_t* bits = reinterpret_cast<uint32_t*>(a->scale);
  MMG_CUDA(cudaMemsetAsync(a->scale, 0, sizeof(float) * a->B, st));
  MMG_CUDA(launch_pdl(image_amax_kernel, grid, dim3(QZ_THREADS), 0, st, reinterpret_cast<const uint4*>(a->x), bits, n8));
  MMG_LAUNCHED();
  MMG_CUDA(launch_pdl(image_quant_kernel, grid, dim3(QZ_THREADS), 0, st, reinterpret_cast<const uint4*>(a->x), reinterpret_cast<uint2*>(a->q),
                      static_cast<const uint32_t*>(bits), n8));
  MMG_LAUNCHED();
  MMG_CUDA(launch_pdl(image_scale_kernel, dim3((unsigned)((a->B + 127) / 128)), dim3(128), 0, st, a->scale, (int)a->B));
  MMG_LAUNCHED();
  return MMG_OK;
}

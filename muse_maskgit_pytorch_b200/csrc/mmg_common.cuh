// Shared host/device helpers for libmmg (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <stdlib.h>
#include <utility>
#include "../../include/mmg.h"

namespace mmg {

typedef __nv_bfloat16 bf16;
typedef __nv_fp8_e4m3 fp8e4;

// ---- thread-local error string -------------------------------------------------------------------
inline char* err_buf() { static thread_local char buf[512] = {0}; return buf; }
inline int fail(int code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(err_buf(), 512, fmt, ap); va_end(ap);
  return code;
}
inline std::atomic<int64_t>& launch_counter() { static std::atomic<int64_t> c{0}; return c; }
// bf16 matrix products / convolutions that could not take the wgmma path (K or Cin % 64, N % 64, alignment, tile geometry) and ran on the
// CUDA-core kernel instead: a >100x performance cliff, so it is counted (mmg_simt_fallback_count) and, with MMG_VERBOSE=1, logged once per shape
inline std::atomic<int64_t>& simt_fallback_counter() { static std::atomic<int64_t> c{0}; return c; }
// every launch of the CUDA-core matrix-product / attention kernels (any dtype): the fp32 parity mode is expected to keep this at zero on
// tensor-core-eligible shapes (mmg_simt_launch_count)
inline std::atomic<int64_t>& simt_launch_counter() { static std::atomic<int64_t> c{0}; return c; }
inline void note_simt_fallback(const char* what, long long M, long long N, long long K) {
  simt_fallback_counter()++;
  static const bool verbose = [] { const char* e = getenv("MMG_VERBOSE"); return e && e[0] == '1'; }();
  if (verbose) fprintf(stderr, "[libmmg] %s M=%lld N=%lld K=%lld (bf16) runs on the CUDA-core kernel: shape / alignment outside the wgmma path\n", what, M, N, K);
}

#define MMG_CHECK_ARG(cond, ...) do { if (!(cond)) return ::mmg::fail(MMG_EINVAL, __VA_ARGS__); } while (0)
#define MMG_CUDA(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
    return ::mmg::fail(MMG_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)
// after a kernel launch: count it, surface launch-configuration errors (no sync)
#define MMG_LAUNCHED() do { ::mmg::launch_counter()++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) \
    return ::mmg::fail(MMG_ECUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

inline int num_sms() {
  static int n = 0;
  if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
  return n;
}

// ---- programmatic dependent launch (PDL) ------------------------------------------------------------
// Hot-loop kernels are launched with cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's CTAs become
// resident (and run their prologue) while the previous grid drains, then block in griddepcontrol.wait until that grid has
// completed and flushed.  Every kernel launched this way calls pdl_wait() before its first global access.  Opt-in with MMG_PDL=1:
// under CUDA-graph replay the launch gaps it hides are already small, so the default is off.
inline bool pdl_enabled() { static int v = -1; if (v < 0) { const char* e = getenv("MMG_PDL"); v = (e && e[0] == '1') ? 1 : 0; } return v != 0; }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- device helpers --------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<bf16>(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// exact-erf GELU (F.gelu default), ref muse_maskgit_pytorch.py:77
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float leaky01(float x) { return x > 0.f ? x : 0.1f * x; }

// one full 32-byte sector per lane as two adjacent 16-byte accesses (p 32-byte aligned)
__device__ __forceinline__ void st256(void* p, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t a4, uint32_t a5, uint32_t a6, uint32_t a7) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};\n\tst.global.v4.b32 [%0+16], {%5,%6,%7,%8};"
               :: "l"(p), "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(a4), "r"(a5), "r"(a6), "r"(a7) : "memory");
}
__device__ __forceinline__ void ld256(const void* p, uint32_t (&a)[8]) {
  asm volatile("ld.global.v4.b32 {%0,%1,%2,%3}, [%8];\n\tld.global.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]), "=r"(a[4]), "=r"(a[5]), "=r"(a[6]), "=r"(a[7]) : "l"(p));
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) { __nv_bfloat162 t = __floats2bfloat162_rn(a, b); return *reinterpret_cast<uint32_t*>(&t); }
__device__ __forceinline__ bool aligned32(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31) == 0; }

// load/store 64 consecutive elements of T from/to a 16B-aligned row chunk (whole 32-byte sectors per access pair when 32B-aligned)
template <typename T> struct Vec64;
template <> struct Vec64<float> {
  static __device__ __forceinline__ void store(float* p, const float (&v)[64]) {
    if (aligned32(p)) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        st256(p + 8 * i, __float_as_uint(v[8 * i]), __float_as_uint(v[8 * i + 1]), __float_as_uint(v[8 * i + 2]), __float_as_uint(v[8 * i + 3]),
              __float_as_uint(v[8 * i + 4]), __float_as_uint(v[8 * i + 5]), __float_as_uint(v[8 * i + 6]), __float_as_uint(v[8 * i + 7]));
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) reinterpret_cast<float4*>(p)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    }
  }
  static __device__ __forceinline__ void load(const float* p, float (&v)[64]) {
    if (aligned32(p)) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { uint32_t a[8]; ld256(p + 8 * i, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[8 * i + j] = __uint_as_float(a[j]); }
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) { float4 t = reinterpret_cast<const float4*>(p)[i]; v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w; }
    }
  }
};
template <> struct Vec64<bf16> {
  static __device__ __forceinline__ void store(bf16* p, const float (&v)[64]) {
    if (aligned32(p)) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        st256(p + 16 * i, pack_bf16(v[16 * i], v[16 * i + 1]), pack_bf16(v[16 * i + 2], v[16 * i + 3]), pack_bf16(v[16 * i + 4], v[16 * i + 5]), pack_bf16(v[16 * i + 6], v[16 * i + 7]),
              pack_bf16(v[16 * i + 8], v[16 * i + 9]), pack_bf16(v[16 * i + 10], v[16 * i + 11]), pack_bf16(v[16 * i + 12], v[16 * i + 13]), pack_bf16(v[16 * i + 14], v[16 * i + 15]));
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        uint4 t;
        t.x = pack_bf16(v[8 * i], v[8 * i + 1]); t.y = pack_bf16(v[8 * i + 2], v[8 * i + 3]);
        t.z = pack_bf16(v[8 * i + 4], v[8 * i + 5]); t.w = pack_bf16(v[8 * i + 6], v[8 * i + 7]);
        reinterpret_cast<uint4*>(p)[i] = t;
      }
    }
  }
  static __device__ __forceinline__ void load(const bf16* p, float (&v)[64]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint4 t = reinterpret_cast<const uint4*>(p)[i];
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
      for (int j = 0; j < 4; ++j) { float2 f = __bfloat1622float2(h[j]); v[8 * i + 2 * j] = f.x; v[8 * i + 2 * j + 1] = f.y; }
    }
  }
};

__device__ __forceinline__ float rcp_fast(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float ex2_fast(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// GLU output a * sigmoid(g) of the bf16 tensor-core epilogues (the register GLU and the GLU tile epilogue: the same instructions in both)
__device__ __forceinline__ float glu_fast(float a, float g) { return a * rcp_fast(1.0f + ex2_fast(-g * 1.4426950408889634f)); }
// exact-erf GELU for the bf16 tensor-core epilogues in 11 FP32 ops + one MUFU:  gelu(x) = max(x, 0) - 0.5 |x| erfc(|x| / sqrt 2), with
// log2 erfc(a / sqrt 2) as a degree-6 polynomial on [0, 6] (weighted minimax fit, scripts/fit_gelu.py); beyond 6 the correction term is
// below 1e-8 |x|.  Max abs error 6e-7 over all x (fp32 rounding included), relative error < 1e-4 in the negative tail — the output is
// rounded to bf16 (4e-3) next.  (The Abramowitz-Stegun form used before cost 2 MUFU + 18 ops per value; the GEGLU epilogue is issue-bound, DESIGN.md 8.)
__device__ __forceinline__ float gelu_fast(float x) {
  const float a = fabsf(x), aq = fminf(a, 6.0f);
  float q = fmaf(2.988134292536415e-05f, aq, -0.0007395807770080864f);
  q = fmaf(q, aq, 0.007976729422807693f); q = fmaf(q, aq, -0.053237367421388626f); q = fmaf(q, aq, -0.4589160978794098f);
  q = fmaf(q, aq, -1.1511470079421997f);
  const float e = ex2_fast(q * aq);
  return fmaf(-0.5f * a, e, fmaxf(x, 0.0f));
}

}  // namespace mmg

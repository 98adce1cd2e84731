// HBM-bound row kernels: LayerNorm, token embedding, final-LN + CFG combine, GroupNorm, first 5x5 conv, casts.
#include "mmg_common.cuh"

namespace mmg {

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, the row is held in registers (width <= 32*4*MAXV), two-pass mean/variance in fp32
// exactly as F.layer_norm (biased variance, eps 1e-5).  ref: muse_maskgit_pytorch.py:63-70
// ---------------------------------------------------------------------------------------------------------------
constexpr int LN_MAXV = 16;   // float4 chunks per lane -> width <= 2048

template <typename TX, typename TY>
__global__ void __launch_bounds__(256)
layernorm_kernel(const TX* __restrict__ x, TY* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ add,
                 float* __restrict__ x_out, float* __restrict__ zero_stats, int64_t add_from, int64_t rows, int width, int64_t ldx, int64_t ldy) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  if (zero_stats && lane == 0) *reinterpret_cast<float2*>(zero_stats + 2 * row) = make_float2(0.f, 0.f);
  if (row < add_from) { add = nullptr; x_out = nullptr; }
  const TX* xr = x + row * ldx;
  float v[LN_MAXV * 4];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = (i * 32 + lane) * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float t = 0.f;
      if (c + j < width) { t = to_f(xr[c + j]); if (add) t += __ldg(add + c + j); }
      v[i * 4 + j] = t; sum += t;
    }
  }
  sum = warp_sum(sum);
  const float mean = sum / (float)width;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = (i * 32 + lane) * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) if (c + j < width) { const float d = v[i * 4 + j] - mean; sq += d * d; }
  }
  sq = warp_sum(sq);
  const float rstd = rsqrtf(sq / (float)width + 1e-5f);
  TY* yr = y + row * ldy;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = (i * 32 + lane) * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c + j < width) {
        yr[c + j] = from_f<TY>((v[i * 4 + j] - mean) * rstd * __ldg(gamma + c + j));
        if (x_out) x_out[row * ldx + c + j] = v[i * 4 + j];
      } else if (c + j < ldy) {
        yr[c + j] = from_f<TY>(0.f);
      }
    }
  }
}

// Vectorised LayerNorm: every lane moves 16 bytes per access (4 fp32 or 8 bf16 columns), CH chunks per lane cover the row,
// statistics over the true width in fp32 (two-pass over registers, as F.layer_norm), columns in [width, ldy) written as 0.
template <typename T> struct VecIO;
template <> struct VecIO<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void ld(const float* p, float* v) { const float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
  static __device__ __forceinline__ void st(float* p, const float* v) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct VecIO<bf16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void ld(const bf16* p, float* v) {
    const uint4 t = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
  }
  static __device__ __forceinline__ void st(bf16* p, const float* v) {
    uint4 t; uint32_t* u = reinterpret_cast<uint32_t*>(&t);
#pragma unroll
    for (int j = 0; j < 4; ++j) { __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]); u[j] = *reinterpret_cast<uint32_t*>(&h); }
    *reinterpret_cast<uint4*>(p) = t;
  }
};
// store N fp32 values as TY starting at p (N = 4 or 8)
template <typename TY, int N> __device__ __forceinline__ void store_vec(TY* p, const float* v);
template <> __device__ __forceinline__ void store_vec<float, 4>(float* p, const float* v) { VecIO<float>::st(p, v); }
template <> __device__ __forceinline__ void store_vec<float, 8>(float* p, const float* v) { VecIO<float>::st(p, v); VecIO<float>::st(p + 4, v + 4); }
template <> __device__ __forceinline__ void store_vec<bf16, 8>(bf16* p, const float* v) { VecIO<bf16>::st(p, v); }
template <> __device__ __forceinline__ void store_vec<bf16, 4>(bf16* p, const float* v) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
  uint2 t; t.x = *reinterpret_cast<uint32_t*>(&a); t.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = t;
}

template <typename TX, typename TY, int CH>
__global__ void __launch_bounds__(256)
layernorm_vec_kernel(const TX* __restrict__ x, TY* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ add,
                     float* __restrict__ x_out, float* __restrict__ zero_stats, int64_t add_from, int64_t rows, int width, int64_t ldx, int64_t ldy) {
  constexpr int VN = VecIO<TX>::N;
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  if (zero_stats && lane == 0) *reinterpret_cast<float2*>(zero_stats + 2 * row) = make_float2(0.f, 0.f);
  if (row < add_from) { add = nullptr; x_out = nullptr; }
  const TX* xr = x + row * ldx;
  float v[CH][VN];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = (i * 32 + lane) * VN;
    if (c < width) {
      VecIO<TX>::ld(xr + c, v[i]);
      if (add) {
#pragma unroll
        for (int j = 0; j < VN; j += 4) { const float4 a = *reinterpret_cast<const float4*>(add + c + j); v[i][j] += a.x; v[i][j + 1] += a.y; v[i][j + 2] += a.z; v[i][j + 3] += a.w; }
      }
#pragma unroll
      for (int j = 0; j < VN; ++j) { if (c + j >= width) v[i][j] = 0.f; sum += v[i][j]; }
    } else {
#pragma unroll
      for (int j = 0; j < VN; ++j) v[i][j] = 0.f;
    }
  }
  float mean, rstd;
  if (sizeof(TY) == 2) {
    // bf16 output: one fused reduction of (sum, sum of squares) — the E[x^2] - mean^2 form is far inside bf16 output precision
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < CH; ++i)
#pragma unroll
      for (int j = 0; j < VN; ++j) sq = fmaf(v[i][j], v[i][j], sq);       // padded / out-of-width entries are 0
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); sq += __shfl_xor_sync(0xffffffffu, sq, o); }
    mean = sum / (float)width;
    rstd = rsqrtf(fmaxf(sq / (float)width - mean * mean, 0.f) + 1e-5f);
  } else {
    mean = warp_sum(sum) / (float)width;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int c = (i * 32 + lane) * VN;
#pragma unroll
      for (int j = 0; j < VN; ++j) if (c + j < width) { const float d = v[i][j] - mean; sq += d * d; }
    }
    rstd = rsqrtf(warp_sum(sq) / (float)width + 1e-5f);
  }
  TY* yr = y + row * ldy;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = (i * 32 + lane) * VN;
    if (c < ldy) {
      float o[VN];
#pragma unroll
      for (int j = 0; j < VN; ++j) o[j] = (c + j < width) ? (v[i][j] - mean) * rstd * __ldg(gamma + c + j) : 0.f;
      store_vec<TY, VN>(yr + c, o);
      if (x_out && c < width) {
#pragma unroll
        for (int j = 0; j < VN; j += 4) *reinterpret_cast<float4*>(x_out + row * ldx + c + j) = make_float4(v[i][j], v[i][j + 1], v[i][j + 2], v[i][j + 3]);
      }
    }
  }
}

// The hot LayerNorm of the transformer blocks (fp32 residual stream -> bf16 GEMM operand, width = CH * 128 exactly, dense rows): a warp
// normalises TWO rows, with the 2 * CH 128-bit loads of both rows issued before any arithmetic (twice the bytes in flight per warp: the
// one-row kernel sat at 34 % of the HBM rate with 44 % of the issue slots busy) and gamma read as float4.
template <int CH>
__global__ void __launch_bounds__(256)
layernorm_rows2_kernel(const float* __restrict__ x, bf16* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ add,
                       float* __restrict__ x_out, float* __restrict__ zero_stats, int64_t add_from, int64_t rows) {
  constexpr int W = CH * 128;
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t r0 = ((int64_t)blockIdx.x * 8 + (threadIdx.x >> 5)) * 2;
  if (r0 >= rows) return;
  const bool two = r0 + 1 < rows;
  float4 v[2][CH];
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < CH; ++i)
      v[q][i] = (q == 0 || two) ? reinterpret_cast<const float4*>(x + (r0 + q) * W)[i * 32 + lane] : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 g[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) g[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i * 32 + lane);
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int64_t row = r0 + q;
    if (q == 1 && !two) break;
    if (zero_stats && lane == 0) *reinterpret_cast<float2*>(zero_stats + 2 * row) = make_float2(0.f, 0.f);
    const bool do_add = add && row >= add_from;
    if (do_add) {
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(add) + i * 32 + lane);
        v[q][i].x += a.x; v[q][i].y += a.y; v[q][i].z += a.z; v[q][i].w += a.w;
        if (x_out) reinterpret_cast<float4*>(x_out + row * W)[i * 32 + lane] = v[q][i];
      }
    }
    float sum = 0.f, sq = 0.f;
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      sum += (v[q][i].x + v[q][i].y) + (v[q][i].z + v[q][i].w);
      sq = fmaf(v[q][i].x, v[q][i].x, fmaf(v[q][i].y, v[q][i].y, fmaf(v[q][i].z, v[q][i].z, fmaf(v[q][i].w, v[q][i].w, sq))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); sq += __shfl_xor_sync(0xffffffffu, sq, o); }
    const float mean = sum * (1.0f / W);
    const float rstd = rsqrtf(fmaxf(sq * (1.0f / W) - mean * mean, 0.f) + 1e-5f);
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const float o0 = (v[q][i].x - mean) * rstd * g[i].x, o1 = (v[q][i].y - mean) * rstd * g[i].y;
      const float o2 = (v[q][i].z - mean) * rstd * g[i].z, o3 = (v[q][i].w - mean) * rstd * g[i].w;
      uint2 t; t.x = pack_bf16(o0, o1); t.y = pack_bf16(o2, o3);
      reinterpret_cast<uint2*>(y + row * W)[i * 32 + lane] = t;
    }
  }
}

// x[copy][r, :] = token_emb[ids[r]] + pos_emb[r % n]        ref: muse_maskgit_pytorch.py:322-323 (and 316 with use_pos = 0)
__global__ void embed_kernel(const int64_t* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                             float* __restrict__ x, int64_t rows, int64_t n, int64_t dim, int copies, int use_pos) {
  pdl_wait(); pdl_trigger();
  const int64_t row = blockIdx.x;
  const int64_t id = ids[row];
  const float4* t = reinterpret_cast<const float4*>(tok + id * dim);
  const float4* p = reinterpret_cast<const float4*>(pos + (row % n) * dim);
  for (int c = threadIdx.x; c < dim / 4; c += blockDim.x) {
    float4 a = __ldg(t + c);
    if (use_pos) { const float4 b = __ldg(p + c); a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
    for (int k = 0; k < copies; ++k) reinterpret_cast<float4*>(x + ((int64_t)k * rows + row) * dim)[c] = a;
  }
}

// e[j] = LNn + (LNc - LNn) * s on the masked rows; one warp per masked row; dim <= 128 * NV (NV float4 per lane: the register arrays are
// sized for the row width actually used — the one-size LN_MAXV version needed 255 registers and spilled).
template <typename TE, int NV>
__global__ void __launch_bounds__(256)
final_embed_kernel(const float* __restrict__ xc, const float* __restrict__ xn, const float* __restrict__ gamma,
                   const int32_t* __restrict__ masked_pos, TE* __restrict__ e, int B, int n, int num_masked, int dim, float s) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t j = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (j >= (int64_t)B * num_masked) return;
  const int b = (int)(j / num_masked);
  const int64_t row = (int64_t)b * n + masked_pos[j];
  float out[NV * 4];
#pragma unroll
  for (int i = 0; i < NV * 4; ++i) out[i] = 0.f;
  for (int pass = 0; pass < 2; ++pass) {
    const float* xr = (pass == 0 ? xc : xn);
    if (!xr) continue;
    xr += row * dim;
    float v[NV * 4]; float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
#pragma unroll
      if (c + 3 < dim) {                 // rows are 16-byte aligned whenever dim % 4 == 0 (checked by the launcher)
        const float4 t = *reinterpret_cast<const float4*>(xr + c);
        v[i * 4] = t.x; v[i * 4 + 1] = t.y; v[i * 4 + 2] = t.z; v[i * 4 + 3] = t.w; sum += (t.x + t.y) + (t.z + t.w);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float t = (c + k < dim) ? xr[c + k] : 0.f; v[i * 4 + k] = t; sum += t; }
      }
    }
    const float mean = warp_sum(sum) / (float)dim;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) if (c + k < dim) { const float d = v[i * 4 + k] - mean; sq += d * d; }
    }
    const float rstd = rsqrtf(warp_sum(sq) / (float)dim + 1e-5f);
    // cond pass contributes s * LNc, null pass (1 - s) * LNn:  LNn + (LNc - LNn) * s
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) if (c + k < dim) {
        const float ln = (v[i * 4 + k] - mean) * rstd * __ldg(gamma + c + k);
        // keep the reference's association: null + (cond - null) * scale
        if (pass == 0) out[i * 4 + k] = ln; else out[i * 4 + k] = ln + (out[i * 4 + k] - ln) * s;
      }
    }
  }
  TE* er = e + j * dim;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
#pragma unroll
    if (c + 3 < dim) {
      if constexpr (sizeof(TE) == 2) *reinterpret_cast<uint2*>(er + c) = make_uint2(pack_bf16(out[i * 4], out[i * 4 + 1]), pack_bf16(out[i * 4 + 2], out[i * 4 + 3]));
      else *reinterpret_cast<float4*>(er + c) = make_float4(out[i * 4], out[i * 4 + 1], out[i * 4 + 2], out[i * 4 + 3]);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) if (c + k < dim) er[c + k] = from_f<TE>(out[i * 4 + k]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm over NHWC [B, HW, C]: one CTA per (b, group); mean, then centred variance, then apply (3 passes over an
// L2-resident slab).  eps 1e-5, affine, optional LeakyReLU(0.1).   ref: vqgan_vae.py:257,260,272-276
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < nw) ? red[l] : 0.f;
  t = warp_sum(t);
  return t;
}

template <typename T>
__global__ void __launch_bounds__(256)
groupnorm_kernel(T* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int C, int groups, int act) {
  __shared__ float red[32];
  const int b = blockIdx.x / groups, g = blockIdx.x % groups;
  const int cg = C / groups;
  T* base = x + (int64_t)b * HW * C + g * cg;
  const int total = HW * cg;
  float s = 0.f;
  for (int i = threadIdx.x; i < total; i += blockDim.x) s += to_f(base[(int64_t)(i / cg) * C + (i % cg)]);
  const float mean = block_sum(s, red) / (float)total;
  float q = 0.f;
  for (int i = threadIdx.x; i < total; i += blockDim.x) { const float d = to_f(base[(int64_t)(i / cg) * C + (i % cg)]) - mean; q += d * d; }
  const float rstd = rsqrtf(block_sum(q, red) / (float)total + 1e-5f);
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    const int c = i % cg; T* p = base + (int64_t)(i / cg) * C + c;
    float v = (to_f(*p) - mean) * rstd * __ldg(gamma + g * cg + c) + __ldg(beta + g * cg + c);
    if (act) v = leaky01(v);
    *p = from_f<T>(v);
  }
}

// First encoder conv: 5x5 pad 2, Cin = C (<= 4), fp32 NCHW image -> NHWC activations.  K = 25*C is tiny; persistent
// CTAs keep the transposed weights [K][Cout] in shared memory and sweep groups of 8 pixels (patches staged in smem,
// broadcast reads), thread = output channel, stores coalesced along Cout.   ref: vqgan_vae.py:231
constexpr int CI_PIX = 8;
template <typename T>
__global__ void __launch_bounds__(256)
conv_in_kernel(const float* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias, T* __restrict__ out,
               int B, int C, int H, int W, int Cout, int ks) {
  extern __shared__ float ws[];                   // [K][Cout] then patches [CI_PIX][K]
  const int kk = ks * ks, pad = ks / 2;
  const int K = C * kk;
  float* patch = ws + (size_t)K * Cout;
  for (int i = threadIdx.x; i < Cout * K; i += blockDim.x) { const int co = i / K, k = i - co * K; ws[k * Cout + co] = w[i]; }
  const int64_t pixels = (int64_t)B * H * W;
  for (int64_t p0 = (int64_t)blockIdx.x * CI_PIX; p0 < pixels; p0 += (int64_t)gridDim.x * CI_PIX) {
    __syncthreads();
    for (int i = threadIdx.x; i < CI_PIX * K; i += blockDim.x) {
      const int pi = i / K, k = i - pi * K; const int64_t pix = p0 + pi;
      float v = 0.f;
      if (pix < pixels) {
        const int b = (int)(pix / ((int64_t)H * W)); const int rem = (int)(pix - (int64_t)b * H * W); const int y = rem / W, xx = rem - y * W;
        const int c = k / kk, r = (k % kk) / ks, sx = k % ks; const int iy = y + r - pad, ix = xx + sx - pad;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(img + (((int64_t)b * C + c) * H + iy) * W + ix);
      }
      patch[i] = v;
    }
    __syncthreads();
    for (int co = threadIdx.x; co < Cout; co += blockDim.x) {
      float acc[CI_PIX];
      const float bv = bias ? bias[co] : 0.f;
#pragma unroll
      for (int pi = 0; pi < CI_PIX; ++pi) acc[pi] = bv;
      for (int k = 0; k < K; ++k) {
        const float wv = ws[k * Cout + co];
#pragma unroll
        for (int pi = 0; pi < CI_PIX; ++pi) acc[pi] = fmaf(patch[pi * K + k], wv, acc[pi]);
      }
#pragma unroll
      for (int pi = 0; pi < CI_PIX; ++pi) if (p0 + pi < pixels) out[(p0 + pi) * Cout + co] = from_f<T>(acc[pi]);
    }
  }
}

template <typename S, typename D>
__global__ void cast_kernel(const S* __restrict__ s, D* __restrict__ d, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) d[i] = from_f<D>(to_f(s[i]));
}

// fp32 -> three bf16 terms (hi = bf16(x), mid = bf16(x - hi), lo = bf16(x - hi - mid): 24 mantissa bits in all), laid out so that ONE
// bf16 tensor-core product over 6K columns accumulates the six significant cross terms of the fp32 product in fp32, smallest first:
//   A side [lo | hi | mid | mid | hi | hi ]  x  W side [hi | lo | mid | hi | mid | hi]  =  lo*hi + hi*lo + mid*mid + mid*hi + hi*mid + hi*hi
// (the dropped mid*lo, lo*mid, lo*lo terms are below 2^-24 of the product).  precision="fp32" runs its matrix products through this.
__global__ void split3_kernel(const float* __restrict__ src, bf16* __restrict__ dst, int64_t rows, int64_t K, int64_t lds, int side) {
  const int64_t kv = K >> 3;                       // 8 columns per thread
  const int64_t total = rows * kv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / kv, c = (i - r * kv) * 8;
    const float4 a = *reinterpret_cast<const float4*>(src + r * lds + c), b = *reinterpret_cast<const float4*>(src + r * lds + c + 4);
    const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t hi[4], mid[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float h[2], m[2], l[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = x[2 * j + e];
        h[e] = __bfloat162float(__float2bfloat16_rn(v));
        const float r1 = v - h[e];                                   // exact
        m[e] = __bfloat162float(__float2bfloat16_rn(r1));
        l[e] = r1 - m[e];                                            // exact; rounded to bf16 by the pack below
      }
      hi[j] = pack_bf16(h[0], h[1]); mid[j] = pack_bf16(m[0], m[1]); lo[j] = pack_bf16(l[0], l[1]);
    }
    const uint4 H = make_uint4(hi[0], hi[1], hi[2], hi[3]), M = make_uint4(mid[0], mid[1], mid[2], mid[3]), L = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    bf16* d = dst + r * 6 * K + c;
    const uint4 t0 = side ? H : L, t1 = side ? L : H, t3 = side ? H : M, t4 = side ? M : H;
    *reinterpret_cast<uint4*>(d) = t0; *reinterpret_cast<uint4*>(d + K) = t1; *reinterpret_cast<uint4*>(d + 2 * K) = M;
    *reinterpret_cast<uint4*>(d + 3 * K) = t3; *reinterpret_cast<uint4*>(d + 4 * K) = t4; *reinterpret_cast<uint4*>(d + 5 * K) = H;
  }
}

}  // namespace mmg

using namespace mmg;

extern "C" int mmg_layernorm(const mmg_layernorm_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->y && a->gamma, "mmg_layernorm: NULL pointer");
  MMG_CHECK_ARG(a->width > 0 && a->width <= LN_MAXV * 128, "mmg_layernorm: width %lld not in (0, %d]", (long long)a->width, LN_MAXV * 128);
  MMG_CHECK_ARG(a->ldy >= a->width && a->ldx >= a->width, "mmg_layernorm: leading dims");
  MMG_CHECK_ARG(!a->x_out || a->x_dtype == MMG_F32, "mmg_layernorm: x_out requires fp32 x");
  if (a->rows == 0) return MMG_OK;
  const unsigned grid = (unsigned)((a->rows + 7) / 8);
  const int w = (int)a->width;
  const int vn = a->x_dtype == MMG_BF16 ? 8 : 4;                      // columns per 16-byte access of the input
  const int64_t span = a->ldy > w ? a->ldy : w;
  const bool vec = (a->ldx % vn == 0) && (a->ldy % vn == 0) && ((reinterpret_cast<uintptr_t>(a->x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(a->y) & 15) == 0) &&
                   (!a->add || (w % vn == 0 && (reinterpret_cast<uintptr_t>(a->add) & 15) == 0)) && (!a->x_out || w % vn == 0) &&
                   ((w + vn - 1) / vn * vn <= a->ldx) && span <= 16 * 32 * vn;
#define LNV(TX, TY, CH) launch_pdl(layernorm_vec_kernel<TX, TY, CH>, dim3(grid), dim3(256), 0, st, (const TX*)a->x, (TY*)a->y, a->gamma, a->add, a->x_out, a->zero_stats, a->add_from, a->rows, w, a->ldx, a->ldy)
#define LNV_DISPATCH(TX, TY) do { const int64_t per = 32 * vn; const int ch = (int)((span + per - 1) / per); \
    if (ch <= 4) LNV(TX, TY, 4); else if (ch <= 6) LNV(TX, TY, 6); else if (ch <= 8) LNV(TX, TY, 8); else LNV(TX, TY, 16); } while (0)
#define LN_LAUNCH(TX, TY) layernorm_kernel<TX, TY><<<grid, 256, 0, st>>>((const TX*)a->x, (TY*)a->y, a->gamma, a->add, a->x_out, a->zero_stats, a->add_from, a->rows, w, a->ldx, a->ldy)
  // dense fp32 -> bf16 rows of exactly CH * 128 columns: two rows per warp
  const bool rows2 = a->x_dtype == MMG_F32 && a->y_dtype == MMG_BF16 && vec && a->ldx == w && a->ldy == w && (w == 512 || w == 256 || w == 128) &&
                     (!a->x_out || a->x_out == (const float*)a->x) && ((reinterpret_cast<uintptr_t>(a->gamma) & 15) == 0);
  if (rows2) {
    const unsigned g2 = (unsigned)((a->rows + 15) / 16);
#define LN2(CH) launch_pdl(layernorm_rows2_kernel<CH>, dim3(g2), dim3(256), 0, st, (const float*)a->x, (bf16*)a->y, a->gamma, a->add, a->x_out, a->zero_stats, a->add_from, a->rows)
    if (w == 512) MMG_CUDA(LN2(4)); else if (w == 256) MMG_CUDA(LN2(2)); else MMG_CUDA(LN2(1));
#undef LN2
    MMG_LAUNCHED();
    return MMG_OK;
  }
  if (a->x_dtype == MMG_F32 && a->y_dtype == MMG_F32) { if (vec) LNV_DISPATCH(float, float); else LN_LAUNCH(float, float); }
  else if (a->x_dtype == MMG_F32 && a->y_dtype == MMG_BF16) { if (vec) LNV_DISPATCH(float, bf16); else LN_LAUNCH(float, bf16); }
  else if (a->x_dtype == MMG_BF16 && a->y_dtype == MMG_BF16) { if (vec) LNV_DISPATCH(bf16, bf16); else LN_LAUNCH(bf16, bf16); }
  else return fail(MMG_EINVAL, "mmg_layernorm: unsupported dtype pair %d -> %d", a->x_dtype, a->y_dtype);
#undef LNV
#undef LNV_DISPATCH
#undef LN_LAUNCH
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_embed(const mmg_embed_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->ids && a->token_emb && a->x && (a->pos_emb || !a->use_pos), "mmg_embed: NULL pointer");
  MMG_CHECK_ARG(a->dim % 4 == 0 && a->copies >= 1 && a->n > 0, "mmg_embed: dim %% 4, copies, n");
  if (a->rows == 0) return MMG_OK;
  MMG_CUDA(launch_pdl(embed_kernel, dim3((unsigned)a->rows), dim3(128), 0, st, a->ids, a->token_emb, a->use_pos ? a->pos_emb : a->token_emb, a->x, a->rows, a->n, a->dim, a->copies, a->use_pos));
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_final_embed(const mmg_final_embed_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x_cond && a->gamma && a->masked_pos && a->e, "mmg_final_embed: NULL pointer");
  MMG_CHECK_ARG(a->dim > 0 && a->dim <= LN_MAXV * 128, "mmg_final_embed: dim");
  const int64_t R = (int64_t)a->B * a->num_masked;
  if (R == 0) return MMG_OK;
  const unsigned grid = (unsigned)((R + 7) / 8);
  MMG_CHECK_ARG(a->dim % 4 == 0 && (reinterpret_cast<uintptr_t>(a->x_cond) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->x_null) & 15) == 0, "mmg_final_embed: dim %% 4, 16-byte aligned rows");
  MMG_CHECK_ARG((reinterpret_cast<uintptr_t>(a->e) & 15) == 0, "mmg_final_embed: e must be 16-byte aligned");
#define MMG_FE(TE, NV) MMG_CUDA(launch_pdl(final_embed_kernel<TE, NV>, dim3(grid), dim3(256), 0, st, a->x_cond, a->x_null, a->gamma, a->masked_pos, (TE*)a->e, a->B, a->n, a->num_masked, a->dim, a->cond_scale))
  const int nv = a->dim <= 128 ? 1 : a->dim <= 256 ? 2 : a->dim <= 512 ? 4 : a->dim <= 1024 ? 8 : LN_MAXV;
  if (a->e_dtype == MMG_BF16) { switch (nv) { case 1: MMG_FE(bf16, 1); break; case 2: MMG_FE(bf16, 2); break; case 4: MMG_FE(bf16, 4); break; case 8: MMG_FE(bf16, 8); break; default: MMG_FE(bf16, LN_MAXV); } }
  else { switch (nv) { case 1: MMG_FE(float, 1); break; case 2: MMG_FE(float, 2); break; case 4: MMG_FE(float, 4); break; case 8: MMG_FE(float, 8); break; default: MMG_FE(float, LN_MAXV); } }
#undef MMG_FE
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_groupnorm(const mmg_groupnorm_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->gamma && a->beta, "mmg_groupnorm: NULL pointer");
  MMG_CHECK_ARG(a->groups > 0 && a->C % a->groups == 0, "mmg_groupnorm: C %% groups");
  const unsigned grid = (unsigned)(a->B * a->groups);
  if (a->dtype == MMG_BF16) groupnorm_kernel<bf16><<<grid, 256, 0, st>>>((bf16*)a->x, a->gamma, a->beta, a->HW, a->C, a->groups, a->act);
  else groupnorm_kernel<float><<<grid, 256, 0, st>>>((float*)a->x, a->gamma, a->beta, a->HW, a->C, a->groups, a->act);
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_conv_in(const mmg_conv_in_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->img && a->w && a->out, "mmg_conv_in: NULL pointer");
  MMG_CHECK_ARG(a->C >= 1 && a->C <= 4, "mmg_conv_in: channels %d not in [1,4]", a->C);
  const int ks = a->ksize ? a->ksize : 5;
  MMG_CHECK_ARG(ks >= 1 && ks <= 9 && (ks & 1), "mmg_conv_in: kernel size %d must be odd and <= 9", ks);
  const size_t smem = ((size_t)a->Cout + CI_PIX) * a->C * ks * ks * sizeof(float);
  MMG_CHECK_ARG(smem <= 200 * 1024, "mmg_conv_in: Cout x kernel too large for shared memory");
  int64_t pixels = ((int64_t)a->B * a->H * a->W + CI_PIX - 1) / CI_PIX;
  if (pixels > (int64_t)num_sms() * 2) pixels = (int64_t)num_sms() * 2;
  if (a->out_dtype == MMG_BF16) {
    MMG_CUDA(cudaFuncSetAttribute(conv_in_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    conv_in_kernel<bf16><<<(unsigned)pixels, 256, smem, st>>>(a->img, a->w, a->bias, (bf16*)a->out, a->B, a->C, a->H, a->W, a->Cout, ks);
  } else {
    MMG_CUDA(cudaFuncSetAttribute(conv_in_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    conv_in_kernel<float><<<(unsigned)pixels, 256, smem, st>>>(a->img, a->w, a->bias, (float*)a->out, a->B, a->C, a->H, a->W, a->Cout, ks);
  }
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_cast(const mmg_cast_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->src && a->dst, "mmg_cast: NULL pointer");
  if (a->n == 0) return MMG_OK;
  const unsigned grid = (unsigned)((a->n + 255) / 256 < num_sms() * 16 ? (a->n + 255) / 256 : num_sms() * 16);
  if (a->src_dtype == MMG_F32 && a->dst_dtype == MMG_BF16) cast_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)a->src, (bf16*)a->dst, a->n);
  else if (a->src_dtype == MMG_BF16 && a->dst_dtype == MMG_F32) cast_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)a->src, (float*)a->dst, a->n);
  else return fail(MMG_EINVAL, "mmg_cast: unsupported dtype pair");
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_split3(const mmg_split3_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->src && a->dst, "mmg_split3: NULL pointer");
  MMG_CHECK_ARG(a->rows >= 0 && a->K > 0 && a->K % 8 == 0 && a->lds >= a->K && a->lds % 4 == 0, "mmg_split3: K %% 8, lds %% 4 (rows %lld, K %lld, lds %lld)",
                (long long)a->rows, (long long)a->K, (long long)a->lds);
  MMG_CHECK_ARG((reinterpret_cast<uintptr_t>(a->src) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->dst) & 15) == 0, "mmg_split3: 16-byte alignment");
  if (a->rows == 0) return MMG_OK;
  const int64_t work = a->rows * (a->K / 8);
  const unsigned grid = (unsigned)((work + 255) / 256 < num_sms() * 16 ? (work + 255) / 256 : num_sms() * 16);
  split3_kernel<<<grid, 256, 0, st>>>(a->src, reinterpret_cast<bf16*>(a->dst), a->rows, a->K, a->lds, a->side);
  MMG_LAUNCHED();
  return MMG_OK;
}

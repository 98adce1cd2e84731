// Fused GEMM epilogues, shared by the wgmma kernel (mmg_gemm_tc.cuh) and the fp32 CUDA-core kernel
// (mmg_gemm_simt.cu).  One thread owns one output row and walks it in chunks of 64 accumulator columns.
#pragma once
#include "mmg_common.cuh"

namespace mmg {

struct Epilogue {
  mmg_epilogue_args p;
  int kind;
  int fast;                 // 1: tensor-core (bf16) path — MUFU-based erf/sigmoid are accurate far beyond bf16 output precision
  int64_t M, N;
  float rgb_acc[4];
  float st_a, st_b;         // LNFOLD: (mean, rstd) of the row
  int r_b, r_t;             // QKV: (batch, token) of the row; CONVT*: (batch, y * W + x)
  template <typename T>
  static __device__ __forceinline__ void store_n(T* dst, const float (&v)[64], int n, bool vec_ok) {
    if (vec_ok && n == 64) {
      Vec64<T>::store(dst, v);
    } else {
#pragma unroll
      for (int i = 0; i < 64; ++i) if (i < n) dst[i] = from_f<T>(v[i]);
    }
  }
  static __device__ __forceinline__ void store32_bf16(bf16* dst, const float* v) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint4 t;
      __nv_bfloat162 a = __floats2bfloat162_rn(v[8 * i], v[8 * i + 1]), b = __floats2bfloat162_rn(v[8 * i + 2], v[8 * i + 3]);
      __nv_bfloat162 c = __floats2bfloat162_rn(v[8 * i + 4], v[8 * i + 5]), d = __floats2bfloat162_rn(v[8 * i + 6], v[8 * i + 7]);
      t.x = *reinterpret_cast<uint32_t*>(&a); t.y = *reinterpret_cast<uint32_t*>(&b);
      t.z = *reinterpret_cast<uint32_t*>(&c); t.w = *reinterpret_cast<uint32_t*>(&d);
      reinterpret_cast<uint4*>(dst)[i] = t;
    }
  }

  __device__ __forceinline__ void begin_row(int64_t row) {
    if (kind == MMG_EPI_QKV) { const uint32_t r = (uint32_t)row, d = (uint32_t)p.tokens; r_b = (int)(r / d); r_t = (int)(r - (uint32_t)r_b * d); }
    if (kind == MMG_EPI_CONVT || kind == MMG_EPI_CONVT_RGB) { const uint32_t r = (uint32_t)row, d = (uint32_t)(p.H * p.W); r_b = (int)(r / d); r_t = (int)(r - (uint32_t)r_b * d); }
    if (kind == MMG_EPI_LNFOLD_RESIDUAL) {
      // the row's (sum, sumsq) = its per-chunk partials added in ascending chunk order: the same bits whichever CTA wrote which partial when
      const float2* sp = reinterpret_cast<const float2*>(p.row_stats) + row * (int64_t)p.stats_slots;
      float sx = 0.f, sq = 0.f;
      for (int i = 0; i < p.stats_slots; ++i) { const float2 t = __ldg(sp + i); sx += t.x; sq += t.y; }
      const float mean = sx / (float)p.ln_width;
      st_a = mean; st_b = rsqrtf(fmaxf(sq / (float)p.ln_width - mean * mean, 0.f) + 1e-5f);
    }
    if (kind == MMG_EPI_CONVT_RGB) {
#pragma unroll
      for (int c = 0; c < 4; ++c) rgb_acc[c] = (c < p.rgb_channels) ? p.rgb_b[c] : 0.f;
    }
  }

  // row: global output row (< M). col0: first accumulator column of this chunk (multiple of 64). nvalid: columns < N.
  // QKV: which output a 64-column chunk belongs to (0 q, 1 k, 2 v), its head, and the l2-normalisation * scale of q / k in place
  //   F.normalize(dim=-1, eps=1e-12) then * scale   (muse_maskgit_pytorch.py:151-153)
  template <bool FAST>
  __device__ __forceinline__ int qkv_chunk(int col0, float (&v)[64], int& h) const {
    const int hc = col0 >> 6;
    const int which = hc < p.nq_heads ? 0 : (hc < p.nq_heads + p.nk_heads ? 1 : 2);
    h = which == 0 ? hc : (which == 1 ? hc - p.nq_heads : hc - p.nq_heads - p.nk_heads);
    const float* sc = which == 0 ? p.q_scale : (which == 1 ? p.k_scale : nullptr);
    if (sc) {
      float s4[4] = {0.f, 0.f, 0.f, 0.f};                    // four partial sums: 16-deep dependency chains instead of 64
#pragma unroll
      for (int i = 0; i < 64; ++i) s4[i & 3] = fmaf(v[i], v[i], s4[i & 3]);
      const float ss = (s4[0] + s4[1]) + (s4[2] + s4[3]);
      const float inv = FAST ? rsqrtf(fmaxf(ss, 1e-24f)) : 1.0f / fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
      for (int i = 0; i < 64; ++i) v[i] = v[i] * inv * sc[i];
    }
    return which;
  }
  // the learned null key / value -> key row 0 of (b, h), written by the thread that owns token 0 (muse_maskgit_pytorch.py:145-149)
  __device__ __forceinline__ void qkv_null_row(int which, int64_t b, int h) const {
    const void* nsrc = which == 1 ? p.null_k : p.null_v;
    if (!nsrc) return;
    void* dst = which == 1 ? p.k_out : p.v_out;
    const int64_t noff = ((b * p.heads + h) * (int64_t)p.kv_rows) * 64;
    if (p.out_dtype == MMG_BF16) {
      const uint4* sp = reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(nsrc) + h * 64);
      uint4* dp = reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(dst) + noff);
#pragma unroll
      for (int i = 0; i < 8; ++i) dp[i] = sp[i];
    } else {
      const float4* sp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(nsrc) + h * 64);
      float4* dp = reinterpret_cast<float4*>(reinterpret_cast<float*>(dst) + noff);
#pragma unroll
      for (int i = 0; i < 16; ++i) dp[i] = sp[i];
    }
  }

  // GEGLU of one 64-column accumulator chunk [x(32) | gate(32)] -> 32 outputs.  With row_stats: this chunk's (sum, sumsq) of the outputs goes
  // to its own slot row_stats[row][col0 / 64] (no atomics: the folded LayerNorm adds the slots in a fixed order, so bf16 generate() is bitwise
  // reproducible whatever the tile schedule).  The statistics are those of the bf16-ROUNDED outputs when the output is bf16 — the values the
  // second product consumes.
  template <bool FAST>
  __device__ __forceinline__ void geglu_chunk(const float (&v)[64], float (&o)[32], int64_t row, int col0, bool write_stats) const {
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = v[32 + i] * (FAST ? gelu_fast(v[i]) : gelu_erf(v[i]));
    if (p.row_stats && write_stats) {
      float sx = 0.f, sq = 0.f;
      if (p.out_dtype == MMG_BF16) {
#pragma unroll
        for (int i = 0; i < 32; ++i) { const float t = __bfloat162float(__float2bfloat16_rn(o[i])); sx += t; sq = fmaf(t, t, sq); }
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) { sx += o[i]; sq = fmaf(o[i], o[i], sq); }
      }
      reinterpret_cast<float2*>(p.row_stats)[row * (int64_t)p.stats_slots + (col0 >> 6)] = make_float2(sx, sq);
    }
  }

  template <bool FAST>
  __device__ __forceinline__ void apply(int64_t row, int col0, float (&v)[64], int nvalid) {
    const bool bf = (p.out_dtype == MMG_BF16);
    switch (kind) {
      case MMG_EPI_LFQ_IDS: {
        const int bits = p.ln_width;                 // 3 * bits <= 64: columns [hi | mid | lo] of the split projection
        long long id = 0;
#pragma unroll
        for (int i = 0; i < 21; ++i) {
          if (i < bits) {
            float s3 = 0.f;
#pragma unroll
            for (int j = 0; j < 64; ++j) if (j == i || j == i + bits || j == i + 2 * bits) s3 += v[j];
            if (s3 + (p.bias ? __ldg(p.bias + i) : 0.f) > 0.f) id |= 1ll << (bits - 1 - i);
          }
        }
        if (col0 == 0) reinterpret_cast<long long*>(p.out)[row] = id;
        break;
      }
      case MMG_EPI_ARGMIN: {
        unsigned long long best = ~0ull;
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          if (i < nvalid) {
            const float d = __ldg(p.bias + col0 + i) - 2.f * v[i];
            const uint32_t u = __float_as_uint(d);
            const uint32_t key = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
            const unsigned long long cand = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(col0 + i);
            best = cand < best ? cand : best;
          }
        }
        atomicMin(reinterpret_cast<unsigned long long*>(p.out) + row, best);
        break;
      }
      case MMG_EPI_LNFOLD_RESIDUAL: {
#pragma unroll
        for (int i = 0; i < 64; ++i) v[i] = st_b * (v[i] - st_a * __ldg(p.bias + col0 + i));
        float* o = reinterpret_cast<float*>(p.out) + row * p.ldo + col0;
        const float* r = reinterpret_cast<const float*>(p.resid) + row * p.ldr + col0;
        float t[64]; Vec64<float>::load(r, t);
#pragma unroll
        for (int i = 0; i < 64; ++i) v[i] += t[i];
        Vec64<float>::store(o, v);
        break;
      }
      case MMG_EPI_STORE:
      case MMG_EPI_RESIDUAL: {
        if (p.bias) {
#pragma unroll
          for (int i = 0; i < 64; ++i) if (i < nvalid) v[i] += __ldg(p.bias + col0 + i);
        }
        const bool vec_ok = (nvalid == 64) && ((p.ldo & 7) == 0);
        if (kind == MMG_EPI_RESIDUAL) {
          const bool rvec = vec_ok && ((p.ldr & 7) == 0);
          if (bf) {
            const bf16* r = reinterpret_cast<const bf16*>(p.resid) + row * p.ldr + col0;
            if (rvec) { float t[64]; Vec64<bf16>::load(r, t);
#pragma unroll
              for (int i = 0; i < 64; ++i) v[i] += t[i];
            } else {
#pragma unroll
              for (int i = 0; i < 64; ++i) if (i < nvalid) v[i] += to_f(r[i]);
            }
          } else {
            const float* r = reinterpret_cast<const float*>(p.resid) + row * p.ldr + col0;
            if (rvec) { float t[64]; Vec64<float>::load(r, t);
#pragma unroll
              for (int i = 0; i < 64; ++i) v[i] += t[i];
            } else {
#pragma unroll
              for (int i = 0; i < 64; ++i) if (i < nvalid) v[i] += r[i];
            }
          }
        }
        if (p.act == 1) {
#pragma unroll
          for (int i = 0; i < 64; ++i) v[i] = leaky01(v[i]);
        }
        if (bf) store_n(reinterpret_cast<bf16*>(p.out) + row * p.ldo + col0, v, nvalid, vec_ok);
        else    store_n(reinterpret_cast<float*>(p.out) + row * p.ldo + col0, v, nvalid, vec_ok);
        break;
      }
      case MMG_EPI_GEGLU:
      case MMG_EPI_GLU: {
        float o[32];
        if (kind == MMG_EPI_GEGLU) {
          geglu_chunk<FAST>(v, o, row, col0, true);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            float a = v[i] + (p.bias ? __ldg(p.bias + col0 + i) : 0.f);
            float g = v[32 + i] + (p.bias ? __ldg(p.bias + col0 + 32 + i) : 0.f);
            o[i] = FAST ? a * rcp_fast(1.0f + ex2_fast(-g * 1.4426950408889634f)) : a * (1.0f / (1.0f + expf(-g)));
          }
        }
        const int oc = col0 >> 1;
        if (bf) {
          bf16* d = reinterpret_cast<bf16*>(p.out) + row * p.ldo + oc;
          if ((p.ldo & 7) == 0) store32_bf16(d, o);
          else {
#pragma unroll
            for (int i = 0; i < 32; ++i) d[i] = from_f<bf16>(o[i]);
          }
        } else {
          float* d = reinterpret_cast<float*>(p.out) + row * p.ldo + oc;
          if ((p.ldo & 3) == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) reinterpret_cast<float4*>(d)[i] = make_float4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) d[i] = o[i];
          }
        }
        break;
      }
      case MMG_EPI_QKV: {
        const int64_t b = r_b, t = r_t;
        int h;
        const int which = qkv_chunk<FAST>(col0, v, h);
        void* dst = which == 0 ? p.q_out : (which == 1 ? p.k_out : p.v_out);
        const int64_t off = which == 0 ? ((b * p.heads + h) * (int64_t)p.q_rows + t) * 64 : ((b * p.heads + h) * (int64_t)p.kv_rows + p.key_off + t) * 64;
        if (bf) Vec64<bf16>::store(reinterpret_cast<bf16*>(dst) + off, v);
        else    Vec64<float>::store(reinterpret_cast<float*>(dst) + off, v);
        if (t == 0 && which != 0) qkv_null_row(which, b, h);
        break;
      }
      case MMG_EPI_CONVT:
      case MMG_EPI_CONVT_RGB: {
#pragma unroll
        for (int i = 0; i < 64; ++i) v[i] = leaky01(v[i] + (p.bias ? __ldg(p.bias + col0 + i) : 0.f));
        if (kind == MMG_EPI_CONVT) {
          const int64_t b = r_b; const int rem = r_t; const int y = rem / p.W, x = rem - y * p.W;
          const int64_t opix = (b * 2 * p.H + 2 * y + p.py) * (int64_t)(2 * p.W) + 2 * x + p.px;
          const bool vec_ok = (nvalid == 64) && ((p.ldo & 7) == 0);
          if (bf) store_n(reinterpret_cast<bf16*>(p.out) + opix * p.ldo + col0, v, nvalid, vec_ok);
          else    store_n(reinterpret_cast<float*>(p.out) + opix * p.ldo + col0, v, nvalid, vec_ok);
        } else {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (c < p.rgb_channels) {
              const float* w = p.rgb_w + (int64_t)c * N + col0;
              float s = 0.f;
#pragma unroll
              for (int i = 0; i < 64; ++i) if (i < nvalid) s += v[i] * __ldg(w + i);
              rgb_acc[c] += s;
            }
          }
        }
        break;
      }
    }
  }

  // ---- residual epilogues with the residual chunk prefetched by the caller (tensor-core kernel) -------------------------
  __device__ __forceinline__ bool can_prefetch_resid() const {
    if (kind == MMG_EPI_LNFOLD_RESIDUAL) return true;
    return kind == MMG_EPI_RESIDUAL && p.out_dtype == MMG_F32 && (p.ldo & 7) == 0 && (p.ldr & 7) == 0 && p.act == 0;
  }
  __device__ __forceinline__ void load_resid(int64_t row, int col0, float (&r)[64]) const {
    Vec64<float>::load(reinterpret_cast<const float*>(p.resid) + row * p.ldr + col0, r);
  }
  // v <- epilogue(v) + r   (r = resid[row, col0 .. col0+63]); the caller stores v with store_f32
  __device__ __forceinline__ void fuse_resid(int col0, float (&v)[64], const float (&r)[64]) const {
    if (kind == MMG_EPI_LNFOLD_RESIDUAL) {
#pragma unroll
      for (int i = 0; i < 64; ++i) v[i] = fmaf(st_b, v[i] - st_a * __ldg(p.bias + col0 + i), r[i]);
    } else {
#pragma unroll
      for (int i = 0; i < 64; ++i) v[i] += r[i] + (p.bias ? __ldg(p.bias + col0 + i) : 0.f);
    }
  }
  // residual epilogues as an in-place reduction (out == resid): v <- the term added to the row; the caller pushes it with
  // cp.reduce.async.bulk (fp32 add in L2), so the residual row is never read and nothing goes through the L1 wavefront path
  __device__ __forceinline__ bool can_reduce_in_place() const {
    return can_prefetch_resid() && p.out == p.resid && p.ldo == p.ldr && p.out_dtype == MMG_F32 && (p.ldo & 3) == 0 &&
           (reinterpret_cast<uintptr_t>(p.out) & 15) == 0;
  }
  __device__ __forceinline__ void resid_term(int col0, float (&v)[64]) const {
    if (kind == MMG_EPI_LNFOLD_RESIDUAL) {
#pragma unroll
      for (int i = 0; i < 64; ++i) v[i] = st_b * (v[i] - st_a * __ldg(p.bias + col0 + i));
    } else if (p.bias) {
#pragma unroll
      for (int i = 0; i < 64; ++i) v[i] += __ldg(p.bias + col0 + i);
    }
  }
  __device__ __forceinline__ void store_f32(int64_t row, int col0, const float (&v)[64]) const {
    Vec64<float>::store(reinterpret_cast<float*>(p.out) + row * p.ldo + col0, v);
  }

  __device__ __forceinline__ void end_row(int64_t row) {
    if (kind == MMG_EPI_CONVT_RGB) {
      const int64_t b = r_b; const int rem = r_t; const int y = rem / p.W, x = rem - y * p.W;
      const int oy = 2 * y + p.py, ox = 2 * x + p.px;
      float* o = reinterpret_cast<float*>(p.out);
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < p.rgb_channels) o[((b * p.rgb_channels + c) * (int64_t)(2 * p.H) + oy) * (2 * p.W) + ox] = rgb_acc[c];
    }
  }
};

// host-side validation shared by the launchers
inline int validate_epilogue(int kind, const mmg_epilogue_args& e, int64_t N) {
  switch (kind) {
    case MMG_EPI_STORE: MMG_CHECK_ARG(e.out, "epilogue STORE: out is NULL"); break;
    case MMG_EPI_RESIDUAL: MMG_CHECK_ARG(e.out && e.resid, "epilogue RESIDUAL: out/resid NULL"); break;
    case MMG_EPI_LFQ_IDS: MMG_CHECK_ARG(e.out && N == 64 && e.ln_width >= 1 && 3 * e.ln_width <= 64, "epilogue LFQ_IDS: N must be 64 and 3*bits <= 64"); break;
    case MMG_EPI_ARGMIN: MMG_CHECK_ARG(e.out && e.bias, "epilogue ARGMIN: out / code norms NULL"); break;
    case MMG_EPI_LNFOLD_RESIDUAL:
      MMG_CHECK_ARG(e.out && e.resid && e.bias && e.row_stats && e.ln_width > 0 && e.stats_slots >= 1, "epilogue LNFOLD_RESIDUAL: out/resid/cvec/row_stats/ln_width/stats_slots");
      MMG_CHECK_ARG(e.out_dtype == MMG_F32 && (N % 64) == 0 && (e.ldo % 4) == 0 && (e.ldr % 4) == 0, "epilogue LNFOLD_RESIDUAL: fp32 out, N %% 64, ld %% 4");
      break;
    case MMG_EPI_GEGLU: case MMG_EPI_GLU:
      MMG_CHECK_ARG(e.out && (N % 64) == 0, "epilogue GEGLU/GLU: N %% 64 != 0 or out NULL");
      MMG_CHECK_ARG(!e.row_stats || (int64_t)e.stats_slots * 64 >= N, "epilogue GEGLU: row_stats needs stats_slots >= N / 64 (%d slots for N = %lld)", e.stats_slots, (long long)N);
      break;
    case MMG_EPI_QKV:
      MMG_CHECK_ARG((N % 64) == 0 && N / 64 == e.nq_heads + e.nk_heads + e.nv_heads, "epilogue QKV: N != 64*(nq+nk+nv)");
      MMG_CHECK_ARG(e.tokens > 0 && e.heads > 0, "epilogue QKV: tokens/heads");
      MMG_CHECK_ARG((!e.nq_heads || (e.q_out && e.q_scale)) && (!e.nk_heads || (e.k_out && e.k_scale)) && (!e.nv_heads || e.v_out), "epilogue QKV: NULL output");
      break;
    case MMG_EPI_CONVT: MMG_CHECK_ARG(e.out && e.H > 0 && e.W > 0, "epilogue CONVT: geometry"); break;
    case MMG_EPI_CONVT_RGB: MMG_CHECK_ARG(e.out && e.rgb_w && e.rgb_b && e.rgb_channels >= 1 && e.rgb_channels <= 4, "epilogue CONVT_RGB: args"); break;
    default: return fail(MMG_EINVAL, "unknown epilogue %d", kind);
  }
  return MMG_OK;
}

}  // namespace mmg

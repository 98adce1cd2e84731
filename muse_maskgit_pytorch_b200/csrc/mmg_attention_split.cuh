// fp32-parity attention on the tensor cores (precision="fp32"): the same wgmma S = Q K^T / O = P V structure as mmg_attention_tc.cuh, with every
// operand carried as three bf16 terms (hi + mid + lo = the fp32 value to 2^-24, mmg_split3) and the six significant cross terms of each product
// accumulated in fp32 registers, smallest first:
//   S  = sum over the 6 x 64 split columns of q (left-operand order) and k (right-operand order)          -> 24 MMAs (K = 16) per key block
//   O += P_lo V_hi + P_hi V_lo + P_mid V_mid + P_mid V_hi + P_hi V_mid + P_hi V_hi                          -> 6 x KB / 16 MMAs per key block
// P is split by the softmax warps as they write it; V's terms are the column chunks 0 (hi), 1 (lo), 2 (mid) of its right-operand split.
// Exact two-pass softmax (true row maximum, attend.py:131), fp32 output.  One CTA = (batch, head, 128 queries), key blocks of 64.
// replaces: attention_simt_kernel on the token-identical parity path (attend.py:123-138 arithmetic).
#pragma once
#include "mmg_common.cuh"
#include "mmg_sm90.cuh"
#include <cudaTypedefs.h>
#include <float.h>

namespace mmg {

struct alignas(64) AttnSplitParams {
  CUtensorMap tma_q, tma_k, tma_v;      // [rows, 384] bf16, boxes of 64 columns x 128 (q) / 64 (k, v) rows
  const uint8_t* key_mask;
  float* out;
  int heads, Tq, Tk, Tk_alloc, nb, KB_tail, kv_shared;
  int64_t ldo;
  float scale_log2e;
};

constexpr int AS_KB = 64;
constexpr int AS_LD = 68;                  // fp32 staging row stride of S / O: it lives in the K tiles, free once S is computed
constexpr int AS_SMEM = 1024 + 6 * 16384 + 6 * 8192 + 3 * 8192 + 3 * 16384 + 128;
static_assert(128 * AS_LD * 4 <= 6 * 8192, "staging must fit the K tiles");

__global__ void __launch_bounds__(160, 1)
attention_tc_split_kernel(const __grid_constant__ AttnSplitParams p) {
  using namespace sm90;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;                         // 6 x (128 x 64 bf16)
  uint8_t* sK = sQ + 6 * 16384;               // 6 x (64 x 64)
  uint8_t* sV = sK + 6 * 8192;                // 3 x (64 x 64): hi, lo, mid
  uint8_t* sP = sV + 3 * 8192;                // 3 x (128 x 64): hi, mid, lo
  float* stg = reinterpret_cast<float*>(sK);  // 128 x AS_LD fp32: S of a block once its product is done, finally O
  uint64_t* bars = reinterpret_cast<uint64_t*>(sP + 3 * 16384);
  uint64_t* bar_q = bars + 0; uint64_t* bar_kv = bars + 1; uint64_t* bar_free = bars + 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // warpgroup index broadcast from lane 0: provably uniform, so the wgmma of the softmax warpgroup are not treated as divergent code
  const int wg_role = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int bh = blockIdx.y, b = bh / p.heads, h = bh % p.heads;
  const int q0 = blockIdx.x * 128;
  const int kvh = p.kv_shared ? h : bh;

  if (warp == 4 && lane == 0) {
    prefetch_tmap(&p.tma_q); prefetch_tmap(&p.tma_k); prefetch_tmap(&p.tma_v);
    mbar_init(bar_q, 1); mbar_init(bar_kv, 1); mbar_init(bar_free, 4);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg_role == 1) {
    if (elect_one()) {
      mbar_expect_tx(bar_q, 6 * 16384);
      for (int c = 0; c < 6; ++c) tma_load_2d(sQ + c * 16384, &p.tma_q, bar_q, c * 64, bh * p.Tq + q0);
      uint32_t ph_free = 0;
      for (int pass = 0; pass < 2; ++pass) {
        for (int blk = 0; blk < p.nb; ++blk) {
          if (pass | blk) { mbar_wait(bar_free, ph_free); ph_free ^= 1; }    // the previous block is done with K / V / P (and the staging)
          const int krow = kvh * p.Tk_alloc + blk * AS_KB;
          mbar_expect_tx(bar_kv, (pass == 0 ? 6 : 9) * 8192);
          for (int c = 0; c < 6; ++c) tma_load_2d(sK + c * 8192, &p.tma_k, bar_kv, c * 64, krow);
          if (pass == 1) for (int c = 0; c < 3; ++c) tma_load_2d(sV + c * 8192, &p.tma_v, bar_kv, c * 64, krow);
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== softmax warpgroup: wgmma, then thread = query row =====================
    const int r = warp * 32 + lane;
    const int qi = q0 + r;
    const float* srow = stg + r * AS_LD;
    const uint8_t* km = p.key_mask ? p.key_mask + (int64_t)b * (p.Tk - 1) : nullptr;
    uint32_t ph_kv = 0;
    float row_max = -FLT_MAX, row_sum = 0.f, mneg = 0.f;
    float o_acc[2][32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { o_acc[0][i] = 0.f; o_acc[1][i] = 0.f; }
    mbar_wait(bar_q, 0);
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 1) mneg = row_max * p.scale_log2e;
      for (int blk = 0; blk < p.nb; ++blk) {
        mbar_wait(bar_kv, ph_kv); ph_kv ^= 1;
        {   // S = sum over the 6 split chunks of Q_c K_c^T, staged row-major over the (now consumed) K tiles
          float s_acc[2][32];
#pragma unroll
          for (int c = 0; c < 6; ++c) {
            wgmma_fence();
            const uint64_t qd = smem_desc_kmajor_sw128(smem_u32(sQ + c * 16384)), kd = smem_desc_kmajor_sw128(smem_u32(sK + c * 8192));
#pragma unroll
            for (int mh = 0; mh < 2; ++mh)
#pragma unroll
              for (int k = 0; k < 4; ++k) Wgmma<AS_KB>::template mma<0>(s_acc[mh], qd + (uint64_t)(mh * 512 + k * 2), kd + (uint64_t)(k * 2), (c | k) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(s_acc[0]); reg_fence(s_acc[1]);
          named_sync(1, 128);                                    // every warp's wgmma has read K before the staging overwrites it
          stage_acc<32, AS_LD>(s_acc[0], stg, 0, AS_KB);
          stage_acc<32, AS_LD>(s_acc[1], stg + 64 * AS_LD, 0, AS_KB);
          named_sync(1, 128);
        }
        const int kb_cur = blk == p.nb - 1 ? p.KB_tail : AS_KB;
        for (int c = 0; c < kb_cur; c += 32) {
          float s[32];
          stage_ld32(srow + c, s);
          const int j0 = blk * AS_KB + c;
          if (pass == 0) {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const int j = j0 + i;
              const bool live = j < p.Tk && (j == 0 || !km || km[j - 1]);     // key 0 (null) is never masked
              if (live) row_max = fmaxf(row_max, s[i]);
            }
          } else {
            uint32_t ph[16], pm[16], pl[16];
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
              float hi[2], mid[2], lo[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int j = j0 + i + e;
                const bool live = j < p.Tk && (j == 0 || !km || km[j - 1]);
                const float pv = live ? ex2_fast(fmaf(s[i + e], p.scale_log2e, -mneg)) : 0.f;
                row_sum += pv;
                hi[e] = __bfloat162float(__float2bfloat16_rn(pv));
                const float r1 = pv - hi[e];
                mid[e] = __bfloat162float(__float2bfloat16_rn(r1));
                lo[e] = r1 - mid[e];
              }
              ph[i >> 1] = pack_bf16(hi[0], hi[1]); pm[i >> 1] = pack_bf16(mid[0], mid[1]); pl[i >> 1] = pack_bf16(lo[0], lo[1]);
            }
            // P[r, c .. c+31] -> 16-byte chunks (c % 64) / 8 .. +3 of row r, 128B swizzle: chunk ^= (r & 7); three term tiles
            const int ch0 = (c & 63) >> 3;
#pragma unroll
            for (int q4 = 0; q4 < 4; ++q4) {
              const int ch = (ch0 + q4) ^ (r & 7);
              uint8_t* dst = sP + r * 128 + ch * 16;
              *reinterpret_cast<uint4*>(dst) = make_uint4(ph[q4 * 4], ph[q4 * 4 + 1], ph[q4 * 4 + 2], ph[q4 * 4 + 3]);
              *reinterpret_cast<uint4*>(dst + 16384) = make_uint4(pm[q4 * 4], pm[q4 * 4 + 1], pm[q4 * 4 + 2], pm[q4 * 4 + 3]);
              *reinterpret_cast<uint4*>(dst + 32768) = make_uint4(pl[q4 * 4], pl[q4 * 4 + 1], pl[q4 * 4 + 2], pl[q4 * 4 + 3]);
            }
          }
        }
        if (pass == 1) {
          fence_proxy_async();                 // generic-proxy smem writes of P -> visible to the tensor core (async proxy)
          named_sync(1, 128);
          const int ksteps = (blk == p.nb - 1 ? p.KB_tail : AS_KB) / 16;
          // (P term, V term): P tiles hi = 0, mid = 1, lo = 2; V tiles hi = 0, lo = 1, mid = 2
          const int pt[6] = {2, 0, 1, 1, 0, 0}, vt[6] = {0, 1, 2, 0, 2, 0};
          for (int t = 0; t < 6; ++t)
            for (int ks = 0; ks < ksteps; ++ks) {
              wgmma_fence();
              const uint32_t pa = smem_u32(sP + pt[t] * 16384) + ks * 32;
              const uint64_t vdesc = smem_desc_mnmajor_sw128(smem_u32(sV + vt[t] * 8192) + ks * 2048, 1024);
              Wgmma<64>::template mma<1>(o_acc[0], smem_desc_kmajor_sw128(pa), vdesc, 1u);
              Wgmma<64>::template mma<1>(o_acc[1], smem_desc_kmajor_sw128(pa + 8192), vdesc, 1u);
            }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(o_acc[0]); reg_fence(o_acc[1]);
        }
        named_sync(1, 128);                    // every row of this block's S has been read before K is reloaded over the staging
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_free);
      }
    }
    const float inv = 1.f / row_sum;
    named_sync(1, 128);
    stage_acc<32, AS_LD>(o_acc[0], stg, 0, 64);
    stage_acc<32, AS_LD>(o_acc[1], stg + 64 * AS_LD, 0, 64);
    named_sync(1, 128);
#pragma unroll
    for (int c = 0; c < 64; c += 32) {
      float o[32];
      stage_ld32(srow + c, o);
      if (qi < p.Tq) {
        float* dst = p.out + ((int64_t)b * p.Tq + qi) * p.ldo + h * 64 + c;
#pragma unroll
        for (int i = 0; i < 32; i += 4) *reinterpret_cast<float4*>(dst + i) = make_float4(o[i] * inv, o[i + 1] * inv, o[i + 2] * inv, o[i + 3] * inv);
      }
    }
  }
}

}  // namespace mmg

// wgmma attention for dh = 64 (bf16 operands, fp32 softmax statistics).
//
// One CTA = one (batch, head, 128-query tile).  Key 0 of every (batch, head) is the learned null key: it is never masked, and it is handled
// OUTSIDE the tensor-core blocks — each softmax thread computes its row's q . k_null with 64 FMAs, its weight joins the row sum and
// p_null * v_null is added to O in the epilogue — so that the n = 256 (1 024, 32) real keys are exactly 4 (8, 1) blocks instead of 4 + a block
// that holds one key.  The real keys 1 .. Tk-1 are walked in nb blocks of KB (64 or 128) keys (the last block
// may be shorter: KB_tail), twice (or once, see single_pass):
//   pass A:  S = Q K^T (wgmma, 2 x m64nKBk16, 4 k-steps) -> shared-memory staging -> per-row running max        (no P, no V traffic)
//   pass B:  S again -> p = exp2((s - max) * scale*log2e) in registers (masked / out-of-range keys -> 0), row sums in fp32,
//            P (bf16) written to shared memory in the K-major SWIZZLE_128B operand layout, O += P V (wgmma, 2 x m64n64k16,
//            KB_tail/16 k-steps, V consumed MN-major straight from its TMA tile) accumulating in registers across blocks.
//   finally: O / rowsum -> bf16 -> out[b, t, h*64 : (h+1)*64].
// The exact two-pass softmax (true row max, as attend.py:131) avoids the rescaling chain of an online softmax; the second
// Q K^T costs 4 extra MMAs per block.  Warps 0-3 are one warpgroup: they issue the wgmma and own the query rows (thread = row once the
// accumulators are staged); warp 4 (one elected lane) issues the TMA loads of the next block as soon as a block is done with K / V.
#pragma once
#include "mmg_common.cuh"
#include "mmg_sm90.cuh"
#include <cudaTypedefs.h>
#include <float.h>

namespace mmg {

struct alignas(64) AttnTcParams {
  CUtensorMap tma_q, tma_k, tma_v;
  const uint8_t* key_mask;
  bf16* out;
  const bf16* k; const bf16* v;   // [kv heads, Tk_alloc, 64]: row 0 of a head = the null key / value (read directly by the softmax warps)
  int heads, Tq, Tk, Tk_alloc, nb, KB, KB_tail, kv_shared;   // nb blocks over the Tk - 1 real keys: nb-1 of KB keys, the last of KB_tail (<= KB, multiple of 32)
  int64_t ldo;
  float scale_log2e;
  float smax;              // > 0: caller-guaranteed bound on |q.k| -> single-pass softmax with a fixed reference maximum
  int single_pass;
};

// Shared memory of one CTA (launcher and kernel agree on it): Q, K, V, P tiles and the fp32 staging of S / O
__host__ __device__ constexpr int attn_stg_ld(int KB) { return (KB > 64 ? KB : 64) + 4; }
__host__ __device__ constexpr size_t attn_smem_bytes(int KB) {
  return 1024 + 16384 + 2 * (size_t)((KB * 128 + 1023) & ~1023) + (size_t)((KB + 63) / 64) * 16384 + (size_t)128 * attn_stg_ld(KB) * 4 + 128;
}

template <int KB>
__global__ void __launch_bounds__(160, 1)
attention_tc_kernel(const __grid_constant__ AttnTcParams p) {
  using namespace sm90;
  constexpr int LD = attn_stg_ld(KB);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  constexpr int kv_bytes = KB * 128;
  uint8_t* sQ = smem;                         // 128 x 64 bf16
  uint8_t* sK = sQ + 16384;                   // KB x 64
  uint8_t* sV = sK + ((kv_bytes + 1023) & ~1023);
  uint8_t* sP = sV + ((kv_bytes + 1023) & ~1023);      // ceil(KB/64) sub-tiles of 128 x 64 bf16
  constexpr int p_tiles = (KB + 63) / 64;
  float* stg = reinterpret_cast<float*>(sP + p_tiles * 16384);    // 128 x LD fp32: S of a block, finally O
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg + 128 * LD);
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
  pdl_wait();
  pdl_trigger();

  if (wg_role == 1) {
    if (elect_one()) {
      // one K (pass A) or K + V (pass B) load per block, each after the softmax warpgroup is done with the previous block's tiles
      mbar_expect_tx(bar_q, 16384);
      tma_load_2d(sQ, &p.tma_q, bar_q, 0, bh * p.Tq + q0);
      uint32_t ph_free = 0;
      int loads = 0;
      for (int pass = p.single_pass ? 1 : 0; pass < 2; ++pass) {
        for (int blk = 0; blk < p.nb; ++blk, ++loads) {
          if (loads) { mbar_wait(bar_free, ph_free); ph_free ^= 1; }
          const int krow = kvh * p.Tk_alloc + 1 + blk * KB;                 // real keys start at row 1
          mbar_expect_tx(bar_kv, pass == 0 ? kv_bytes : 2 * kv_bytes);
          tma_load_2d(sK, &p.tma_k, bar_kv, 0, krow);
          if (pass == 1) tma_load_2d(sV, &p.tma_v, bar_kv, 0, krow);
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== softmax warpgroup: wgmma, then thread = query row =====================
    const int r = warp * 32 + lane;
    const int qi = q0 + r;
    const float* srow = stg + r * LD;
    const uint8_t* km = p.key_mask ? p.key_mask + (int64_t)b * (p.Tk - 1) : nullptr;   // one byte per REAL key
    const int Tr = p.Tk - 1;                                     // real keys
    uint32_t ph_kv = 0;
    float row_sum = 0.f;
    float mneg = 0.f;
    // the null key: s0 = q_r . k_null (Q tile: row r at r * 128 bytes, 16-byte chunk c at position c ^ (r & 7))
    const bf16* knull = p.k + (int64_t)kvh * p.Tk_alloc * 64;
    float s0 = 0.f;
    mbar_wait(bar_q, 0);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const uint4 qv = *reinterpret_cast<const uint4*>(sQ + r * 128 + ((c ^ (r & 7)) * 16));
      const uint4 kv4 = __ldg(reinterpret_cast<const uint4*>(knull) + c);
      const __nv_bfloat162* qh = reinterpret_cast<const __nv_bfloat162*>(&qv);
      const __nv_bfloat162* kh = reinterpret_cast<const __nv_bfloat162*>(&kv4);
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float2 a = __bfloat1622float2(qh[e]), b2 = __bfloat1622float2(kh[e]); s0 = fmaf(a.x, b2.x, s0); s0 = fmaf(a.y, b2.y, s0); }
    }
    float row_max = s0;                                         // the null key is always live
    float p_null = 0.f;
    float o_acc[2][32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { o_acc[0][i] = 0.f; o_acc[1][i] = 0.f; }
    const uint64_t qdesc = smem_desc_kmajor_sw128(smem_u32(sQ));
    const uint64_t kdesc = smem_desc_kmajor_sw128(smem_u32(sK));
    for (int pass = p.single_pass ? 1 : 0; pass < 2; ++pass) {
      if (pass == 1) {
        mneg = (p.single_pass ? p.smax : row_max) * p.scale_log2e;
        p_null = ex2_fast(fmaf(s0, p.scale_log2e, -mneg));
        row_sum = p_null;
      }
      for (int blk = 0; blk < p.nb; ++blk) {
        mbar_wait(bar_kv, ph_kv); ph_kv ^= 1;
        {   // S = Q K^T for the 128 query rows (two m64 halves), staged row-major
          float s_acc[2][KB / 2];
          wgmma_fence();
#pragma unroll
          for (int mh = 0; mh < 2; ++mh)
#pragma unroll
            for (int k = 0; k < 4; ++k) Wgmma<KB>::template mma<0>(s_acc[mh], qdesc + (uint64_t)(mh * 512 + k * 2), kdesc + (uint64_t)(k * 2), k ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(s_acc[0]); reg_fence(s_acc[1]);
          named_sync(1, 128);                                    // every row of the previous block's S has been read
          stage_acc<KB / 2, LD>(s_acc[0], stg, 0, KB);
          stage_acc<KB / 2, LD>(s_acc[1], stg + 64 * LD, 0, KB);
          named_sync(1, 128);
        }
        const int kb_cur = blk == p.nb - 1 ? p.KB_tail : KB;
        for (int c = 0; c < kb_cur; c += 32) {
          float s[32];
          stage_ld32(srow + c, s);
          const int j0 = blk * KB + c;
          // liveness of the 32 keys of this chunk as one ballot word (lane l tests key j0 + l: ONE coalesced mask byte per lane instead of 32
          // byte loads per thread; key 0, the null key, is never masked)
          uint32_t livew = 0xffffffffu;
          if (km || j0 + 32 > Tr) {
            const int jl = j0 + lane;
            livew = __ballot_sync(0xffffffffu, jl < Tr && (!km || km[jl]));
          }
          if (pass == 0) {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              // masked keys take the value -FLT_MAX in the reference; they only matter for the max if every key is masked,
              // which cannot happen
              if ((livew >> i) & 1u) row_max = fmaxf(row_max, s[i]);
            }
          } else {
            uint32_t packed[16];
            if (!km && j0 + 32 <= Tr) {
              // fast path (self-attention, chunk fully inside the key range): no per-key liveness tests
#pragma unroll
              for (int i = 0; i < 32; i += 2) {
                const float p0 = ex2_fast(fmaf(s[i], p.scale_log2e, -mneg)), p1 = ex2_fast(fmaf(s[i + 1], p.scale_log2e, -mneg));
                packed[i >> 1] = pack_bf16(p0, p1);
                // denominator from the unrounded weights: the bf16 rounding of P is unbiased, so sum(p~ v) / sum(p) differs from the exactly
                // normalised sum(p~ v) / sum(p~) by ~2^-9 / sqrt(keys) relative, far below the bf16 rounding of the output (and saves the
                // unpack + add pair per element in this issue-limited loop)
                row_sum += p0 + p1;
              }
            } else {
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
              float pv[2];
#pragma unroll
              for (int e = 0; e < 2; ++e)
                pv[e] = ((livew >> (i + e)) & 1u) ? ex2_fast(fmaf(s[i + e], p.scale_log2e, -mneg)) : 0.f;
              __nv_bfloat162 t = __floats2bfloat162_rn(pv[0], pv[1]);
              packed[i >> 1] = *reinterpret_cast<uint32_t*>(&t);
              const float2 pr = __bfloat1622float2(t);     // masked / ragged chunks (few live keys, no averaging): normalise by the sum of the
              row_sum += pr.x + pr.y;                      // ROUNDED weights, O = sum(p~ v) / sum(p~): a row whose only live key is the null key gets exactly null_v
            }
            }
            // P[r, c .. c+31] -> sub-tile (c / 64), 16-byte chunks (c % 64) / 8 .. +3, 128B swizzle: chunk ^= (r & 7)
            uint8_t* tile = sP + (c >> 6) * 16384 + r * 128;
            const int ch0 = (c & 63) >> 3;
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
          const int ksteps = (blk == p.nb - 1 ? p.KB_tail : KB) / 16;
          for (int ks = 0; ks < ksteps; ++ks) {
            wgmma_fence();
            const uint32_t pa = smem_u32(sP) + (ks >> 2) * 16384 + (ks & 3) * 32;
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
        if (lane == 0) mbar_arrive(bar_free);                    // K / V / P of this block are no longer needed
      }
    }
    named_sync(1, 128);
    stage_acc<32, LD>(o_acc[0], stg, 0, 64);
    stage_acc<32, LD>(o_acc[1], stg + 64 * LD, 0, 64);
    named_sync(1, 128);
    const float inv = 1.f / row_sum;
    const bf16* vnull = p.v + (int64_t)kvh * p.Tk_alloc * 64;
#pragma unroll
    for (int c = 0; c < 64; c += 32) {
      float o[32];
      stage_ld32(srow + c, o);                                     // no real key at all (nb == 0): zero, the output is the null value
#pragma unroll
      for (int i = 0; i < 32; i += 8) {                          // + p_null * v_null (fp32; p_null unrounded in numerator and denominator)
        const uint4 vv = __ldg(reinterpret_cast<const uint4*>(vnull + c + i));
        const __nv_bfloat162* vh = reinterpret_cast<const __nv_bfloat162*>(&vv);
#pragma unroll
        for (int e = 0; e < 4; ++e) { const float2 f = __bfloat1622float2(vh[e]); o[i + 2 * e] = fmaf(p_null, f.x, o[i + 2 * e]); o[i + 2 * e + 1] = fmaf(p_null, f.y, o[i + 2 * e + 1]); }
      }
      if (qi < p.Tq) {
        bf16* dst = p.out + ((int64_t)b * p.Tq + qi) * p.ldo + h * 64 + c;
#pragma unroll
        for (int i = 0; i < 32; i += 8) {
          uint4 t;
          __nv_bfloat162 a0 = __floats2bfloat162_rn(o[i] * inv, o[i + 1] * inv), a1 = __floats2bfloat162_rn(o[i + 2] * inv, o[i + 3] * inv);
          __nv_bfloat162 a2 = __floats2bfloat162_rn(o[i + 4] * inv, o[i + 5] * inv), a3 = __floats2bfloat162_rn(o[i + 6] * inv, o[i + 7] * inv);
          t.x = *reinterpret_cast<uint32_t*>(&a0); t.y = *reinterpret_cast<uint32_t*>(&a1);
          t.z = *reinterpret_cast<uint32_t*>(&a2); t.w = *reinterpret_cast<uint32_t*>(&a3);
          *reinterpret_cast<uint4*>(dst + i) = t;
        }
      }
    }
  }
}

// ---- host side -------------------------------------------------------------------------------------------------
inline bool attention_tc_supported(const mmg_attention_args* a) {
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return al(a->q) && al(a->k) && al(a->v) && al(a->out) && (a->ldo % 8 == 0) && a->Tk >= 2 && a->Tk <= 4096;
}

// Key blocking: nb-1 blocks of KB keys and a last block of KB_tail keys (multiple of 32).  KB = 64 keeps a CTA at ~84 KB of shared memory,
// so two CTAs share an SM and hide each other's MMA -> softmax -> MMA round trips; long sequences use 128-key blocks (fewer round trips per CTA).
inline void attn_blocks(int Tk, int* nb, int* KB, int* KB_tail) {
  const int kb = Tk <= 640 ? 64 : 128;
  const int full = Tk / kb, rem = Tk - full * kb;
  *KB = kb;
  if (rem == 0) { *nb = full; *KB_tail = kb; }
  else { *nb = full + 1; *KB_tail = (rem + 31) / 32 * 32; }
}

int attention_tc_launch(const mmg_attention_args* a, cudaStream_t st);

}  // namespace mmg

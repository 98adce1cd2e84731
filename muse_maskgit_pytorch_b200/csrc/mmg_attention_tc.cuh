// wgmma attention for dh = 64 and dh = 128 (bf16 operands, fp32 softmax statistics).
//
// One CTA = one (batch, head, 128-query tile).  Key 0 of every (batch, head) is the learned null key: it is never masked, and it is handled
// OUTSIDE the tensor-core blocks — each consumer thread computes q . k_null for its two rows with 64 FMAs each, its weight joins the row
// sum and p_null * v_null is added to O in the epilogue — so that the n = 256 (1 024, 32) real keys are exactly 4 (8, 1) blocks instead of
// 4 + a block that holds one key.  The real keys 1 .. Tk-1 are walked in nb blocks of KB (64 or 128) keys (the last block may be shorter:
// KB_tail), twice (or once, see single_pass), 64 keys at a time:
//   pass A:  S = Q K^T (wgmma m64n64k16, 4 k-steps) -> per-row max over the fragment, two shfl.xor steps across the lane quad at the end
//   pass B:  S again -> p = exp2(s * scale*log2e - max * scale*log2e) on the fragment (masked / out-of-range keys -> 0), row sums in fp32,
//            P packed to bf16 in registers is the A operand of O += P V (wgmma m64n64k16 with A from registers, KB_tail/16 k-steps in
//            the last block, V consumed MN-major straight from its TMA tile), O accumulating in registers across blocks.
//   finally: O / rowsum -> bf16 -> a swizzled 64-row box in the warpgroup's Q rows -> 16-byte rows of out[b, t, h*64 : (h+1)*64].
// The exact two-pass softmax (true row max, as attend.py:131) avoids the rescaling chain of an online softmax; the second Q K^T costs 4
// extra MMAs per 64 keys.  Warps 0-3 and 4-7 are two consumer warpgroups of 64 query rows each, sharing the K / V tiles; warp 8 (one
// elected lane) keeps a ring of K / V stages filled ahead of them.
// dh = 128 (attention_tc_d128_kernel) is the same body with every 256-byte row split into two 64-column SW128 panels: the Q tile and each
// K / V stage hold two panels, S = Q K^T takes 8 k16 steps (4 per panel), O = P V runs two m64n64 register-A MMAs per k-step (one per V
// panel) into the two 32-register halves of O, and the output box is the warpgroup's rows of both Q panels.
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
  const bf16* k; const bf16* v;   // [kv heads, Tk_alloc, dh]: row 0 of a head = the null key / value (read directly by the consumer warps)
  int heads, Tq, Tk, Tk_alloc, nb, KB, KB_tail, kv_shared;   // nb blocks over the Tk - 1 real keys: nb-1 of KB keys, the last of KB_tail (<= KB, multiple of 32)
  int64_t ldo;
  float scale_log2e;
  float smax;              // > 0: caller-guaranteed bound on |q.k| -> single-pass softmax with a fixed reference maximum
  int single_pass;
};

// Block and ring of one CTA (launcher and kernel agree on them): warps 0-7 are two consumer warpgroups, each owning 64 of the 128 query
// rows; warp 8 issues the TMA loads.  Shared memory: the Q tile, then a ring of K + V stages holding 256 keys in all (4 x 64 or
// 2 x 128: every C3 self-attention block in flight at once), then the mbarriers: 81 KB at dh = 64, so two CTAs share an SM; 161 KB at
// dh = 128 (one CTA per SM, which its 64 O registers per thread ask for anyway).
constexpr int ATTN_THREADS = 288;
__host__ __device__ constexpr int attn_stages(int KB) { return 256 / KB; }
__host__ __device__ constexpr size_t attn_smem_bytes(int KB, int HD = 64) {
  return 1024 + (size_t)HD * 256 + (size_t)attn_stages(KB) * 2 * KB * HD * 2 + (size_t)(2 * attn_stages(KB) + 1) * 8;
}

template <int KB, int HD>
__device__ __forceinline__ void attention_tc_body(const AttnTcParams& p) {
  using namespace sm90;
  constexpr int NP = HD / 64;                           // 64-column SW128 panels per row
  constexpr int NS = attn_stages(KB), panel_bytes = KB * 128, kv_bytes = NP * panel_bytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;                                   // NP panels of 128 x 64 bf16; each consumer warpgroup's 64 rows become its output box
  uint8_t* sKV = sQ + NP * 16384;                       // stage s: K (NP panels of KB x 64) at sKV + 2 s kv_bytes, V right after it
  uint64_t* full = reinterpret_cast<uint64_t*>(sKV + NS * 2 * kv_bytes);
  uint64_t* empty = full + NS;
  uint64_t* bar_q = empty + NS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // warpgroup index broadcast from lane 0: provably uniform, so the wgmma of the consumer warpgroups are not treated as divergent code
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int bh = blockIdx.y, b = bh / p.heads, h = bh % p.heads;
  const int q0 = blockIdx.x * 128;
  const int kvh = p.kv_shared ? h : bh;

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&p.tma_q); prefetch_tmap(&p.tma_k); prefetch_tmap(&p.tma_v);
    for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(bar_q, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (wg == 2) {
    // producer: load n fills stage n % NS once all 8 consumer warps have released its previous contents.  Two-pass: loads 0 .. nb-1 are
    // K only (the row-max pass), loads nb .. 2 nb - 1 are K + V.
    if (elect_one()) {
      mbar_expect_tx(bar_q, NP * 16384);
#pragma unroll
      for (int pp = 0; pp < NP; ++pp) tma_load_2d(sQ + pp * 16384, &p.tma_q, bar_q, 64 * pp, bh * p.Tq + q0);
      const int loads = (p.single_pass ? 1 : 2) * p.nb;
      for (int n = 0; n < loads; ++n) {
        const int s = n % NS, blk = n % p.nb;
        const bool with_v = p.single_pass || n >= p.nb;
        if (n >= NS) mbar_wait(&empty[s], (n / NS - 1) & 1);
        const int krow = kvh * p.Tk_alloc + 1 + blk * KB;                 // real keys start at row 1
        uint8_t* sK = sKV + s * 2 * kv_bytes;
        mbar_expect_tx(&full[s], with_v ? 2 * kv_bytes : kv_bytes);
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) {
          tma_load_2d(sK + pp * panel_bytes, &p.tma_k, &full[s], 64 * pp, krow);
          if (with_v) tma_load_2d(sK + kv_bytes + pp * panel_bytes, &p.tma_v, &full[s], 64 * pp, krow);
        }
      }
    }
    __syncwarp();
    return;
  }

  // ===================== consumer warpgroup wg: query rows 64 wg .. 64 wg + 63 of the tile, softmax on the accumulator fragments =====
  // thread (warp w, lane l) holds rows wr and wr + 8 (fragment index i: row wr + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2)
  const int wr = 16 * (warp & 3) + (lane >> 2), lq = lane & 3;
  const uint8_t* km = p.key_mask ? p.key_mask + (int64_t)b * (p.Tk - 1) : nullptr;   // one byte per REAL key
  const int Tr = p.Tk - 1;                                     // real keys
  const float sl = p.scale_log2e;
  uint8_t* sQw = sQ + wg * 8192;                             // panel pp of the warpgroup's rows at sQw + pp * 16384
  // the null key: s0 = q_r . k_null for both rows (Q panel: row r at r * 128 bytes, 16-byte chunk c at position c ^ (r & 7))
  const bf16* knull = p.k + (int64_t)kvh * p.Tk_alloc * HD;
  float s0[2] = {0.f, 0.f};
  mbar_wait(bar_q, 0);
#pragma unroll
  for (int c = 0; c < 8 * NP; ++c) {
    const uint4 kv4 = __ldg(reinterpret_cast<const uint4*>(knull) + c);
    const __nv_bfloat162* kh = reinterpret_cast<const __nv_bfloat162*>(&kv4);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = wr + 8 * rr;
      const uint4 qv = *reinterpret_cast<const uint4*>(sQw + (c >> 3) * 16384 + r * 128 + (((c & 7) ^ (r & 7)) * 16));
      const __nv_bfloat162* qh = reinterpret_cast<const __nv_bfloat162*>(&qv);
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float2 a = __bfloat1622float2(qh[e]), b2 = __bfloat1622float2(kh[e]); s0[rr] = fmaf(a.x, b2.x, s0[rr]); s0[rr] = fmaf(a.y, b2.y, s0[rr]); }
    }
  }
  float mx[2] = {s0[0], s0[1]};                              // pass A: this thread's share of the row max (the null key is always live)
  float mneg[2] = {0.f, 0.f};
  float lsum[2] = {0.f, 0.f};                                // pass B: this thread's share of the real keys' row sum
  float o_acc[NP][32];                                       // O columns 64 pp .. 64 pp + 63 in o_acc[pp]
#pragma unroll
  for (int pp = 0; pp < NP; ++pp)
#pragma unroll
    for (int i = 0; i < 32; ++i) o_acc[pp][i] = 0.f;
  int n = 0;                                                  // load index: stage n % NS, phase n / NS
  for (int pass = p.single_pass ? 1 : 0; pass < 2; ++pass) {
    if (pass == 1) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        float m = mx[rr];                                      // max over the lane quad that shares the row: exact in any order
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        mneg[rr] = (p.single_pass ? p.smax : m) * sl;
      }
    }
    for (int blk = 0; blk < p.nb; ++blk, ++n) {
      const int s = n % NS;
      mbar_wait(&full[s], (n / NS) & 1);
      const uint32_t sK = smem_u32(sKV + s * 2 * kv_bytes), sV = sK + kv_bytes;
      const int kb_cur = blk == p.nb - 1 ? p.KB_tail : KB;
#pragma unroll
      for (int sub = 0; sub < KB / 64; ++sub) {              // 64 keys at a time: S of a sub-block is one m64n64 fragment per warpgroup
        if (sub * 64 >= kb_cur) break;
        float s_acc[32];
        wgmma_fence();
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) {
          const uint64_t qdesc = smem_desc_kmajor_sw128(smem_u32(sQw) + pp * 16384);
          const uint64_t kdesc = smem_desc_kmajor_sw128(sK + pp * panel_bytes + sub * 8192);
#pragma unroll
          for (int k = 0; k < 4; ++k) Wgmma<64>::template mma<0>(s_acc, qdesc + (uint64_t)(k * 2), kdesc + (uint64_t)(k * 2), (pp | k) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(s_acc);
        // liveness of each 32-key chunk as one ballot word (lane l tests key j0 + l: ONE coalesced mask byte per lane; key 0, the null
        // key, is never masked); a chunk without mask that ends inside the key range is `fast`: every key live, no tests
        uint32_t livew[2];
        bool fast[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int j0 = blk * KB + sub * 64 + 32 * c;
          fast[c] = !km && j0 + 32 <= Tr;
          const int jl = j0 + lane;
          livew[c] = fast[c] ? 0xffffffffu : __ballot_sync(0xffffffffu, jl < Tr && (!km || km[jl]));
        }
        if (pass == 0) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            // masked keys take the value -FLT_MAX in the reference; they only matter for the max if every key is masked, which cannot
            // happen (the null key is live)
            if ((livew[i >> 4] >> (8 * ((i >> 2) & 3) + 2 * lq + (i & 1))) & 1u) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s_acc[i]);
          }
        } else {
          uint32_t pk[16];                                     // P as bf16 pairs: pk[4 k .. 4 k + 3] is the A fragment of k16 step k
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (fast[c]) {
#pragma unroll
              for (int i = 16 * c; i < 16 * c + 16; i += 2) {
                const int rr = (i >> 1) & 1;
                const float p0 = ex2_fast(fmaf(s_acc[i], sl, -mneg[rr])), p1 = ex2_fast(fmaf(s_acc[i + 1], sl, -mneg[rr]));
                pk[i >> 1] = pack_bf16(p0, p1);
                // denominator from the unrounded weights: the bf16 rounding of P is unbiased, so sum(p~ v) / sum(p) differs from the
                // exactly normalised sum(p~ v) / sum(p~) by ~2^-9 / sqrt(keys) relative, far below the bf16 rounding of the output
                lsum[rr] += p0 + p1;
              }
            } else {
#pragma unroll
              for (int i = 16 * c; i < 16 * c + 16; i += 2) {
                const int rr = (i >> 1) & 1, bit = 8 * ((i >> 2) & 3) + 2 * lq;
                const float p0 = ((livew[c] >> bit) & 1u) ? ex2_fast(fmaf(s_acc[i], sl, -mneg[rr])) : 0.f;
                const float p1 = ((livew[c] >> (bit + 1)) & 1u) ? ex2_fast(fmaf(s_acc[i + 1], sl, -mneg[rr])) : 0.f;
                __nv_bfloat162 t = __floats2bfloat162_rn(p0, p1);
                pk[i >> 1] = *reinterpret_cast<uint32_t*>(&t);
                // masked / ragged chunks (few live keys, no averaging): normalise by the sum of the ROUNDED weights, O = sum(p~ v) / sum(p~):
                // a row whose only live key is the null key gets exactly null_v
                const float2 pr = __bfloat1622float2(t);
                lsum[rr] += pr.x + pr.y;
              }
            }
          }
          // O += P V: the k16 steps of this sub-block that hold keys (V consumed MN-major straight from its TMA tile)
          const int ksteps = min(4, (kb_cur - sub * 64) / 16);
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            if (ks < ksteps) {
              const uint32_t a[4] = {pk[4 * ks], pk[4 * ks + 1], pk[4 * ks + 2], pk[4 * ks + 3]};
#pragma unroll
              for (int pp = 0; pp < NP; ++pp)
                WgmmaRS64::mma(o_acc[pp], a, smem_desc_mnmajor_sw128(sV + pp * panel_bytes + sub * 8192 + ks * 2048, 1024));
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
#pragma unroll
          for (int pp = 0; pp < NP; ++pp) reg_fence(o_acc[pp]);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);                  // this warp is done with the stage's K / V
    }
  }

  // ---- epilogue from the fragments: O / row_sum (+ p_null v_null) -> bf16 -> this warpgroup's 64-row box (its Q rows, no longer read)
  // -> 16-byte coalesced rows of out[b, t, h*dh : (h+1)*dh]
  float pnull[2], inv[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float t = lsum[rr];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    pnull[rr] = ex2_fast(fmaf(s0[rr], sl, -mneg[rr]));       // unrounded in numerator and denominator
    inv[rr] = 1.f / (pnull[rr] + t);
  }
  const bf16* vnull = p.v + (int64_t)kvh * p.Tk_alloc * HD;
#pragma unroll
  for (int pp = 0; pp < NP; ++pp) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int rr = (i >> 1) & 1, r = wr + 8 * rr, col = 8 * (i >> 2) + 2 * lq;
      const float2 f = __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(vnull + 64 * pp + col)));
      const float a0 = fmaf(pnull[rr], f.x, o_acc[pp][i]), a1 = fmaf(pnull[rr], f.y, o_acc[pp][i + 1]);
      *reinterpret_cast<uint32_t*>(sQw + pp * 16384 + r * 128 + (((col >> 3) ^ (r & 7)) << 4) + (col & 7) * 2) = pack_bf16(a0 * inv[rr], a1 * inv[rr]);
    }
  }
  named_sync(1 + wg, 128);
  const int t = threadIdx.x & 127;
#pragma unroll
  for (int it = 0; it < 4 * NP; ++it) {                       // 16 / NP rows of 8 NP 16-byte chunks per iteration
    const int r = (16 / NP) * it + t / (8 * NP), ch = t % (8 * NP);
    const int qi = q0 + 64 * wg + r;
    if (qi < p.Tq) {
      const uint4 val = *reinterpret_cast<const uint4*>(sQw + (ch >> 3) * 16384 + r * 128 + (((ch & 7) ^ (r & 7)) << 4));
      *reinterpret_cast<uint4*>(p.out + ((int64_t)b * p.Tq + qi) * p.ldo + h * HD + ch * 8) = val;
    }
  }
}

template <int KB>
__global__ void __launch_bounds__(ATTN_THREADS, 2)
attention_tc_kernel(const __grid_constant__ AttnTcParams p) { attention_tc_body<KB, 64>(p); }

template <int KB>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_tc_d128_kernel(const __grid_constant__ AttnTcParams p) { attention_tc_body<KB, 128>(p); }

// ---- host side -------------------------------------------------------------------------------------------------
inline bool attention_tc_supported(const mmg_attention_args* a) {
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return al(a->q) && al(a->k) && al(a->v) && al(a->out) && (a->ldo % 8 == 0) && a->Tk >= 2 && a->Tk <= 4096;
}

// Key blocking: nb-1 blocks of KB keys and a last block of KB_tail keys (multiple of 32).  Short sequences use 64-key blocks (a ring of
// four, a ragged tail wastes at most 32 keys); long sequences use 128-key blocks (half the TMA loads and barrier round trips per key).
inline void attn_blocks(int Tk, int* nb, int* KB, int* KB_tail) {
  const int kb = Tk <= 640 ? 64 : 128;
  const int full = Tk / kb, rem = Tk - full * kb;
  *KB = kb;
  if (rem == 0) { *nb = full; *KB_tail = kb; }
  else { *nb = full + 1; *KB_tail = (rem + 31) / 32 * 32; }
}

int attention_tc_launch(const mmg_attention_args* a, int head_dim, cudaStream_t st);

}  // namespace mmg

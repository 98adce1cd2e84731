// mmg_logits_fused: to_logits + top-k filter + gumbel argmax + confidence of one decode step WITHOUT materialising the
// [rows, V] fp32 logits (muse_maskgit_pytorch.py:576-609; SURVEY.md 7.5).
//
//   1. sample GEMM     S[r, j] = e_r . W[j * stride]      ns = min(V, 4096) evenly spaced vocabulary rows (the wgmma GEMM on a strided view of W)
//   2. threshold       t_lo[r] = sample quantile whose expected exceedance count in the full row is k + 4 sigma (exact k-th value when ns == V)
//   3. fused GEMM      the wgmma logits GEMM, 128 x 128 tiles, whose epilogue keeps per-row online-softmax partials (max, sum exp) in registers
//                      and appends the candidates {x >= t_lo[r]} (12 % of the logits) to per-(row, split, chunk) lists: each epilogue thread owns
//                      one row for a whole work item (an M-tile x a contiguous range of N-tiles), compacts its candidates through a private
//                      shared-memory FIFO and writes them as full 32-byte sectors.  The logits themselves never leave the SM.
//   4. finish          per row: merge the partials, gather the lists (n candidates; the exact top-k is inside iff n >= k), then the same exact-rank
//                      perturbed argmax as the materialised-logits sampler (mmg_sampler.cuh: sample_from_list) -> ids, scores.
//   5./6. fallback     rows whose sampled threshold missed (n < k: ~3e-5 of the rows) or whose lists overflowed are redone through the
//                      materialised path on at most LF_FB_CAP rows: a skippable logits GEMM + mmg_logits_sample on an index list.  More such rows than
//                      LF_FB_CAP in one step (constant logits rows ...) raises status[1]; the host then repeats the call on the materialised path.
//
// HBM traffic per row: ~62 KB of candidates written + read instead of 2 x 256 KB of logits; the Philox / gumbel work happens on the lists only.
#include <cuda_fp16.h>
#include "mmg_sm90.cuh"
#include "mmg_tmap.cuh"
#include "mmg_sampler.cuh"
#include <mutex>
#include <type_traits>

namespace mmg {

int linear_impl(const mmg_linear_args* a, const int* skip_if_zero, void* stream);      // mmg_gemm.cu

constexpr int LF_BM = 128, LF_BN = 128, LF_BK = 64;
constexpr int LF_EPI_WARPS = 8, LF_THREADS = 128 + 32 * LF_EPI_WARPS;   // warpgroup 0: TMA; 2 consumer warpgroups (wgmma + epilogue)
constexpr int LF_SEGS = 2;                  // list segments per (row, split): warps of column half h take the 64-column chunk h of every tile
constexpr int LF_FIFO = 32;                 // candidate entries of the per-thread shared-memory FIFO (drained 4 at a time after every 64 columns)
constexpr int LF_FB_CAP = 128;              // rows per step that may take the materialised fallback
constexpr int LF_MAX_SPLITS = 64;
constexpr int LF_A_BYTES = LF_BM * LF_BK * 2, LF_B_BYTES = LF_BN * LF_BK * 2;
constexpr int LF_SLICES = 5;                // epilogue slices of a tile run between the next tile's k-blocks (4 x 16 columns, then the drains)

// Shared memory: the epilogue runs from the accumulator registers, so next to the candidate FIFOs (64 KB) there is room for four 32 KB
// operand stages within the 227 KB of a block: 1 KB alignment + 128 KB ring + 8 KB barriers / padding + 64 KB FIFOs = 201 KB.
// The cross-entropy epilogue (XENT, mmg_logits_xent) keeps no candidates: its 64 KB go to two more stages, 1 + 192 + 8 = 201 KB.
template <bool XENT>
struct LfCfg {
  static constexpr int STAGE_BYTES = LF_A_BYTES + LF_B_BYTES;
  static constexpr int FIFO_BYTES = XENT ? 0 : LF_EPI_WARPS * LF_FIFO * 32 * 8;
  static constexpr int STAGES = XENT ? 6 : 4;
  // [<= 1 KB to align][operand ring][barriers + padding up to the next 8 KB boundary][FIFO region, 8 KB aligned like its per-warp stride]
  static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 8192 + FIFO_BYTES;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

// Fragment -> chunk hand-over.  In the m64n128k16 accumulator fragment the lane quad q = lane % 4 of a row group holds rows r0 and r0 + 8
// (r0 = 16 warp + lane / 4) x both 64-column halves, 16 values of each (row, half) chunk per lane: columns 8 j + 2 q + e (j < 8, e < 2) of
// the half.  Chunk c = 2 half + (row == r0 + 8) belongs to lane c of the quad.  Block (s, kk) below is the 16 values kk = 2 j + e of chunk
// (or, after the exchange, source lane) s: fragment register lf_frag(s, kk).
__host__ __device__ constexpr int lf_frag(int s, int kk) { return 32 * (s >> 1) + 4 * (kk >> 1) + 2 * (s & 1) + (kk & 1); }

// blocks s <-> s ^ x for every s (a lane-dependent permutation: two selects per pair of registers)
__device__ __forceinline__ void lf_xor_blocks(float (&d)[64], int x) {
#pragma unroll
  for (int bit = 1; bit <= 2; bit <<= 1) {
    const bool sw = (x & bit) != 0;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      if (s & bit) continue;
#pragma unroll
      for (int kk = 0; kk < 16; ++kk) {
        const float a = d[lf_frag(s, kk)], b = d[lf_frag(s | bit, kk)];
        d[lf_frag(s, kk)] = sw ? b : a; d[lf_frag(s | bit, kk)] = sw ? a : b;
      }
    }
  }
}

// 4 x 4 block transpose inside the quad, from the accumulators acc (left as they are: the next tile's wgmma owns them) into v: afterwards
// block s of v holds chunk q's 16 values from source lane s, so that the chunk's column i = 8 j + 2 s + e is v[lf_frag(s, 2 j + e)]
// (lf_col below).  Block m first holds the lane's share of chunk q ^ m (sent to lane q ^ m by the xor-m shuffle, which brings back lane
// q ^ m's share of chunk q), then block s takes the share of lane s.
__device__ __forceinline__ void lf_quad_transpose(const float (&acc)[64], float (&v)[64], int q) {
#pragma unroll
  for (int i = 0; i < 64; ++i) v[i] = acc[i];
  lf_xor_blocks(v, q);
#pragma unroll
  for (int m = 1; m < 4; ++m)
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) v[lf_frag(m, kk)] = __shfl_xor_sync(0xffffffffu, v[lf_frag(m, kk)], m);
  lf_xor_blocks(v, q);
}
// register of column i (0..63) of the lane's chunk after lf_quad_transpose
__host__ __device__ constexpr int lf_col(int i) { return lf_frag((i >> 1) & 3, 2 * (i >> 3) + (i & 1)); }

struct alignas(64) LfParams {
  CUtensorMap tma_a, tma_b;
  int64_t R;                      // rows (sampled positions of the step)
  int num_kb, num_m_tiles, num_pm, S, npt, cap;
  const float* thr;               // [R] candidate threshold per row
  float4* parts;                  // [R][S][2]: (running max, sum of exp(x - max), candidate count as int bits, overflow flag as int bits)
                                  // XENT: (running max, sum of exp(x - max), logit at the label column, 1 as int bits if the segment saw the label)
  uint2* lists;                   // [R][S][2][cap]: (logit bits, vocabulary index)
  const int32_t* labels;          // XENT: [R] label column per row
};

// XENT = false: the candidate / softmax epilogue of the fused sampling tail.  XENT = true: the cross-entropy epilogue of mmg_logits_xent,
// which keeps the softmax partials only and takes the label's logit from the one 64-column chunk that holds it.
template <bool XENT>
__global__ void __launch_bounds__(LF_THREADS, 1)
tc_logits_kernel(const __grid_constant__ LfParams p) {
  using namespace sm90;
  using Cfg = LfCfg<XENT>;
  constexpr int STAGES = Cfg::STAGES, STAGE_BYTES = Cfg::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  // FIFO region: aligned (in the shared-memory window) to its 8 KB per-warp stride, so that a thread's slot address is base | slot << 8
  uint8_t* fifo_all = smem + STAGES * STAGE_BYTES + 256;
  fifo_all += (8192u - (smem_u32(fifo_all) & 8191u)) & 8191u;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_items = p.num_pm * p.S;
  const int unit0 = (int)blockIdx.x, unit_step = (int)gridDim.x;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&p.tma_a); prefetch_tmap(&p.tma_b);
    for (int i = 0; i < STAGES; ++i) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, LF_EPI_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && elect_one()) {
      // ===================== TMA producer =====================
      int stage = 0; uint32_t phase = 0;
      for (int item = unit0; item < num_items; item += unit_step) {
        const int m_blk = item % p.num_pm, sp = item / p.num_pm;
        for (int j = 0; j < p.npt; ++j) {
          const int n_blk = sp * p.npt + j;
          for (int kb = 0; kb < p.num_kb; ++kb) {
            mbar_wait(empty_bar + stage, phase ^ 1);
            uint8_t* sa = smem + stage * STAGE_BYTES;
            uint8_t* sb = sa + LF_A_BYTES;
            mbar_expect_tx(full_bar + stage, STAGE_BYTES);
            tma_load_2d(sa, &p.tma_a, full_bar + stage, kb * LF_BK, m_blk * LF_BM);
            tma_load_2d(sb, &p.tma_b, full_bar + stage, kb * LF_BK, n_blk * LF_BN);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===================== consumer warpgroups: wgmma on 64 rows each, then one thread = one row x one 64-column chunk per tile =====================
    constexpr float LOG2E = 1.4426950408889634f;
    const int wg = (warp - 4) >> 2, wq = warp & 3;
    const int q = lane & 3;                       // the lane's chunk of its quad's rows (lf_quad_transpose)
    const int half = q >> 1;                      // the 64-column chunk of every tile this thread takes
    const int r_in_tile = wg * 64 + wq * 16 + (lane >> 2) + 8 * (q & 1);
    // FIFO slot s of this thread lives at fifo | s << 8 (the warp's 8 KB region is 8 KB aligned, a slot row is 32 lanes x 8 bytes)
    const uint32_t fifo = smem_u32(fifo_all) + (uint32_t)(warp - 4) * (LF_FIFO * 256) + (uint32_t)lane * 8u;
    int stage = 0; uint32_t phase = 0;
    float acc[LF_BN / 2];
#pragma unroll
    for (int i = 0; i < LF_BN / 2; ++i) acc[i] = 0.f;
    for (int item = unit0; item < num_items; item += unit_step) {
      const int m_blk = item % p.num_pm, sp = item / p.num_pm;
      const int64_t row = (int64_t)m_blk * LF_BM + r_in_tile;
      const bool valid = row < p.R;
      const float tlo = (!XENT && valid) ? __ldg(p.thr + row) : FLT_MAX;            // rows past R never produce a candidate
      const int lab = (XENT && valid) ? __ldg(p.labels + row) : -1;
      float xl = 0.f; int has_label = 0;
      uint2* seg = p.lists + ((row * p.S + sp) * LF_SEGS + half) * (int64_t)p.cap;
      float m_run = -1e30f, s_run = 0.f;
      uint32_t pos8 = 0;                          // appended entries << 8 (slot byte offset before wrapping)
      int flushed = 0, ovf = 0;
      // the wgmma main loop of tile n_blk into acc; between(kb) runs after k-block kb's group is issued and the previous stage released,
      // while the tensor pipe works on it
      auto mainloop = [&](int n_blk, auto&& between) {
        int prev_stage = -1;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(full_bar + stage, phase);
          const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
          const uint64_t adesc = smem_desc_kmajor_sw128(sa + (uint32_t)wg * 8192u);
          const uint64_t bdesc = smem_desc_kmajor_sw128(sa + LF_A_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < LF_BK / 16; ++k)
            Wgmma<LF_BN>::template mma<0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev_stage >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + prev_stage); }
          prev_stage = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          between(kb);
        }
        wgmma_wait<0>();
        reg_fence(acc);
        if (prev_stage >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + prev_stage); }
      };
      mainloop(sp * p.npt, [](int) {});
      for (int j = 0; j < p.npt; ++j) {
        const int n_blk = sp * p.npt + j;
        const int c = half;
        // the tile's chunk leaves the accumulators (which the next tile's wgmma then owns): column i in v[lf_col(i)]
        float v[64];
        lf_quad_transpose(acc, v, q);
        if constexpr (XENT) {
          const uint32_t off = (uint32_t)lab - (uint32_t)(n_blk * LF_BN + c * 64);      // one chunk of the row holds the label column
          if (off < 64u) {
#pragma unroll
            for (int i = 0; i < 64; ++i) if ((uint32_t)i == off) xl = v[lf_col(i)];
            has_label = 1;
          }
        }
        // ---- online softmax statistics of the row ----
        float lm = fmaxf(v[lf_col(0)], v[lf_col(1)]);
#pragma unroll
        for (int i = 2; i < 64; i += 2) lm = fmaxf(lm, fmaxf(v[lf_col(i)], v[lf_col(i + 1)]));
        if (lm > m_run) { s_run *= ex2_approx((m_run - lm) * LOG2E); m_run = lm; }
        const float mb = m_run * LOG2E;
        float s0 = 0.f, s1 = 0.f;
        const uint32_t col0 = (uint32_t)(n_blk * LF_BN + c * 64);
        const uint32_t pos8_before = pos8;
        // slices 0..3: the exp sums (even / odd column chains, in column order) and the candidate appends of 16 columns each;
        // slice 4: overflow check and the sector drains, after all 64 appends as before
        auto slice = [&](auto sc) {
          constexpr int SL = decltype(sc)::value;
          if constexpr (SL < 4) {
#pragma unroll
            for (int i = 16 * SL; i < 16 * SL + 16; i += 2) { s0 += ex2_approx(fmaf(v[lf_col(i)], LOG2E, -mb)); s1 += ex2_approx(fmaf(v[lf_col(i + 1)], LOG2E, -mb)); }
            if constexpr (!XENT) {
              // ---- candidates >= t_lo -> private FIFO (predicated, no branch) ----
#pragma unroll
              for (int i = 16 * SL; i < 16 * SL + 16; ++i) {
                if (v[lf_col(i)] >= tlo) {
                  const uint32_t a = fifo | (pos8 & ((LF_FIFO - 1) << 8));
                  asm volatile("st.shared.b32 [%0], %1;\n\tst.shared.b32 [%0+4], %2;" :: "r"(a), "r"(__float_as_uint(v[lf_col(i)])), "r"(col0 + (uint32_t)i) : "memory");
                  pos8 += 256u;
                }
              }
            }
          } else if constexpr (XENT) {
            s_run += s0 + s1;
          } else {
            s_run += s0 + s1;
            // more than LF_FIFO - 3 candidates in 64 columns wrapped over unflushed entries (12 % are expected: never on real rows) -> fallback row
            if (pos8 - pos8_before > (uint32_t)((LF_FIFO - 3) << 8)) ovf = 1;
            // ---- drain whole 32-byte sectors: most lanes have one or two to write, all at the same point ----
            while ((int)(pos8 >> 8) - flushed >= 4) {
              if (flushed + 4 <= p.cap) {
                const uint32_t b0 = fifo | (((uint32_t)flushed << 8) & ((LF_FIFO - 1) << 8));      // flushed % 4 == 0: the four slots do not wrap
                uint32_t w[8];
#pragma unroll
                for (int i = 0; i < 4; ++i)
                  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(w[2 * i]), "=r"(w[2 * i + 1]) : "r"(b0 + (uint32_t)(i * 256)));
                st256(seg + flushed, w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
              } else {
                ovf = 1;
              }
              flushed += 4;
            }
          }
        };
        auto slice_at = [&](int s) {
          switch (s) {
            case 0: slice(std::integral_constant<int, 0>{}); break;
            case 1: slice(std::integral_constant<int, 1>{}); break;
            case 2: slice(std::integral_constant<int, 2>{}); break;
            case 3: slice(std::integral_constant<int, 3>{}); break;
            case 4: slice(std::integral_constant<int, 4>{}); break;
          }
        };
        if (j + 1 < p.npt) {
          // the next tile of the item runs on the tensor pipe while this one's epilogue is sliced in between its k-blocks
          mainloop(n_blk + 1, [&](int kb) { if (kb < LF_SLICES) slice_at(kb); });
          for (int s = p.num_kb; s < LF_SLICES; ++s) slice_at(s);
        } else {
          // the item's last tile: finish its epilogue before the next item switches rows
          slice(std::integral_constant<int, 0>{}); slice(std::integral_constant<int, 1>{}); slice(std::integral_constant<int, 2>{});
          slice(std::integral_constant<int, 3>{}); slice(std::integral_constant<int, 4>{});
        }
      }
      if constexpr (XENT) {
        if (valid) p.parts[(row * p.S + sp) * LF_SEGS + half] = make_float4(m_run, s_run, xl, __int_as_float(has_label));
        continue;
      }
      // ---- end of the work item: the last (< 4) entries as one padded sector, then the partial record ----
      const int pos = (int)(pos8 >> 8);
      if (valid) {
        if (pos > flushed) {
          if (flushed + 4 <= p.cap) {
            const uint32_t b0 = fifo | (((uint32_t)flushed << 8) & ((LF_FIFO - 1) << 8));
            uint32_t w[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              w[2 * i] = 0xff7fffffu; w[2 * i + 1] = 0xffffffffu;                      // (-FLT_MAX, no index) padding
              if (flushed + i < pos)
                asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(w[2 * i]), "=r"(w[2 * i + 1]) : "r"(b0 + (uint32_t)(i * 256)));
            }
            st256(seg + flushed, w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
          } else {
            ovf = 1;
          }
        }
        p.parts[(row * p.S + sp) * LF_SEGS + half] = make_float4(m_run, s_run, __int_as_float(pos), __int_as_float(ovf));
      }
    }
  }

  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------------------------
// threshold: one WARP per row, no shared memory, no block barrier.
//   ns < V (sampled rows): the lane keeps its 1/32 of the ns = 4096 sampled logits as 64 half2 registers and the warp walks the 16 bits of
//     the order-preserving fp16 key, one bit per round: count(x >= candidate) is two packed instructions per PAIR of samples (HSET2.GE +
//     HADD2, exact: a lane counts at most 128) and one shuffle reduction.  fp16 resolves the threshold to ~5e-4 near the 90th percentile
//     of a logits row, i.e. to less than one sample; the threshold only has to put the sample rank at
//       rs = mu + 4 sigma + 2   (mu = ns k / V, sigma^2 = mu (1 - k / V))  ->  expected exceedance count in the full row ~ k + 4 sigma V / ns
//     and the exact candidate count is checked by the finishing kernel anyway.
//   ns == V (V <= 4096): the exact k-th largest logit by the same walk over the 32 bits of the fp32 key.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int THR_WARPS = 8, THR_KEYS = SMP_SAMPLE / 32;
__device__ __forceinline__ uint32_t half_key(uint32_t h) { return (h & 0x8000u) ? (~h & 0xffffu) : (h | 0x8000u); }      // fp16 bits -> monotone 16-bit key
__device__ __forceinline__ uint32_t key_half(uint32_t k) { return (k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu); }      // and back

__global__ void __launch_bounds__(THR_WARPS * 32)
logits_threshold_exact_kernel(const float* __restrict__ S, int ns, int k, float* __restrict__ thr, int64_t R, int* __restrict__ fb_count) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (blockIdx.x == 0 && threadIdx.x == 0) *fb_count = 0;
  const int64_t r = (int64_t)blockIdx.x * THR_WARPS + warp;
  if (r >= R) return;
  const float* row = S + r * ns;
  uint32_t sk[THR_KEYS];
#pragma unroll
  for (int j = 0; j < THR_KEYS; ++j) { const int i = lane + j * 32; sk[j] = i < ns ? fkey(ld_stream(row + i)) : 0u; }
  const int rs = k < ns ? k : ns;
  uint32_t prefix = 0;
  for (int bit = 31; bit >= 0; --bit) {
    const uint32_t c = prefix | (1u << bit);
    int n = 0;
#pragma unroll
    for (int j = 0; j < THR_KEYS; ++j) n += (sk[j] >= c);
    if ((int)__reduce_add_sync(0xffffffffu, n) >= rs) prefix = c;
  }
  if (lane == 0) thr[r] = prefix ? key_to_float(prefix) : -FLT_MAX;
}

__global__ void __launch_bounds__(THR_WARPS * 32)
logits_threshold_kernel(const float* __restrict__ S, int ns, int V, int k, float* __restrict__ thr, int64_t R, int* __restrict__ fb_count) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (blockIdx.x == 0 && threadIdx.x == 0) *fb_count = 0;   // per-step fallback counter (the previous step's fallback kernels are done: stream order)
  const int64_t r = (int64_t)blockIdx.x * THR_WARPS + warp;
  if (r >= R) return;
  const float* row = S + r * ns;
  // sampled rows: ns == SMP_SAMPLE (lf_supported), 128 samples per lane as 64 half2 (float4 loads: lane owns 4 consecutive samples per 128)
  __half2 x2[THR_KEYS / 2];
#pragma unroll
  for (int j = 0; j < THR_KEYS / 4; ++j) {
    const float4 v = ld_stream4(reinterpret_cast<const float4*>(row) + j * 32 + lane);
    x2[2 * j] = __floats2half2_rn(v.x, v.y); x2[2 * j + 1] = __floats2half2_rn(v.z, v.w);
  }
  const float pf = (float)k / (float)V, mu = pf * ns;
  const int rs = (int)(mu + 4.0f * sqrtf(mu * (1.f - pf)) + 2.f);
  uint32_t prefix = 0;
  for (int bit = 15; bit >= 0; --bit) {
    const uint32_t c = prefix | (1u << bit);
    const __half t = __ushort_as_half((unsigned short)key_half(c));
    const __half2 t2 = __half2half2(t);
    __half2 cnt = __float2half2_rn(0.f);
#pragma unroll
    for (int j = 0; j < THR_KEYS / 2; ++j) cnt = __hadd2(cnt, __hge2(x2[j], t2));          // 1.0 per sample >= t; NaN thresholds / samples count as 0
    const int n = (int)(__low2float(cnt) + __high2float(cnt));
    if ((int)__reduce_add_sync(0xffffffffu, n) >= rs) prefix = c;
  }
  // prefix = the largest fp16 key with at least rs samples >= it (0: fewer than rs comparable samples -> no usable threshold)
  if (lane == 0) thr[r] = prefix ? __half2float(__ushort_as_half((unsigned short)key_half(prefix))) : -FLT_MAX;
}

// ---------------------------------------------------------------------------------------------------------------------------
// finish: merge partials, gather the candidate lists, sample
// ---------------------------------------------------------------------------------------------------------------------------
struct LfFinish {
  const float4* parts; const uint2* lists; int S, cap;
  const bf16* e; int K;                       // the step's embeddings [R, K] (copied to e_fb for fallback rows)
  int* fb_count; int* fb_rows; bf16* e_fb; int fb_cap;
  int* status;                                // [0] += fallback rows, [1] = 1 when more rows than fb_cap needed the fallback
};

// Finisher.  One CTA of LFN_THREADS per row, nothing but a few words of shared memory, so 6-8 CTAs share an SM and one row's memory round trips
// hide under the others' Philox / gumbel arithmetic.  The row's candidate segments (~62 KB of interleaved (logit, index) pairs) are STREAMED:
//   pass 1  every candidate: noise -> perturbed value, each thread keeps only its best; block argmax -> winner (ties -> lowest vocabulary index)
//   pass 2  (the same bytes again, now L2 hits) exact rank of the winner's logit inside the row: the list covers everything >= it
// and if the winner fails the rank test (it lies between the candidate threshold and the true k-th value: the list holds ~ k + 4 sigma
// entries) its index joins a small exclusion list and pass 1 is repeated — the noise is a pure function of (row, vocabulary index), so the
// repeat reproduces the same values and the result equals sample_from_list's on the gathered list.  (First version: one 512-thread CTA per row
// gathered the list into 74 KB of shared memory with per-lane 8-byte loads, two CTAs per SM: 0.86 TB/s, 15 % of a generate().)
constexpr int LFN_THREADS = 256;
constexpr int LFN_MAX_EXCL = 24;

// candidate traversal shared by both passes: warp w of NW takes segments w, w + NW, ... when there are at least NW segments, otherwise
// NW / nseg warps share a segment; a lane reads two entries (16 bytes) per load, two loads in flight
template <typename F>
__device__ __forceinline__ void lfn_for_each(const uint2* __restrict__ row_lists, const int* s_cnt, int nseg, int cap, int warp, int lane, F&& fn) {
  constexpr int NW = LFN_THREADS / 32;
  const int g = nseg >= NW ? 1 : NW / nseg;                      // warps per segment (nseg = 2 x a power of two)
  const int sub = warp % g, stride = 64 * g;
  for (int sgi = warp / g; sgi < nseg; sgi += NW / g) {
    const int c = s_cnt[sgi];
    const uint2* src = row_lists + (int64_t)sgi * cap;
    for (int i = (sub * 32 + lane) * 2; i < c; i += 2 * stride) {
      uint4 e0, e1 = make_uint4(0u, 0u, 0u, 0u);
      const int i1 = i + stride;
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(e0.x), "=r"(e0.y), "=r"(e0.z), "=r"(e0.w) : "l"(src + i));
      if (i1 < c) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(e1.x), "=r"(e1.y), "=r"(e1.z), "=r"(e1.w) : "l"(src + i1));
      fn(e0.x, e0.y); if (i + 1 < c) fn(e0.z, e0.w);
      if (i1 < c) { fn(e1.x, e1.y); if (i1 + 1 < c) fn(e1.z, e1.w); }
    }
  }
}

// MINB = CTAs per SM the register budget is sized for: 6 (39 registers: the Philox round keys are re-derived per candidate) or 4 (64 registers,
// keys kept).  The kernel is issue-bound (ncu: 71 % issue slots, ALU pipe 53 %), so fewer instructions beat more resident warps; MMG_FINISH_MINB=6
// selects the other build.
template <int MODE, int MINB>
__global__ void __launch_bounds__(LFN_THREADS, MINB)
logits_finish_kernel(const mmg_logits_sample_args a, float tdiv, const LfFinish f) {
  __shared__ int s_cnt[LF_SEGS * LF_MAX_SPLITS];
  __shared__ float s_m[LF_SEGS * LF_MAX_SPLITS], s_s[LF_SEGS * LF_MAX_SPLITS];
  __shared__ float s_max, s_sum;
  __shared__ int s_n, s_bad, s_slot;
  __shared__ int s_excl[LFN_MAX_EXCL];
  __shared__ float s_rv[LFN_THREADS / 32]; __shared__ int s_ri[LFN_THREADS / 32]; __shared__ uint32_t s_rx[LFN_THREADS / 32]; __shared__ int s_rc[LFN_THREADS / 32];
  constexpr float LOG2E = 1.4426950408889634f;
  constexpr int NW = LFN_THREADS / 32;

  pdl_wait(); pdl_trigger();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int V = a.V, k = a.k;
  const int64_t r = blockIdx.x;
  const int b = (int)(r / a.num_masked);
  const int pos = a.masked_pos[r];
  const int nseg = LF_SEGS * f.S;
  if (tid == 0) s_bad = 0;
  __syncthreads();
  if (tid < nseg) {
    const float4 pt = f.parts[r * nseg + tid];
    s_m[tid] = pt.x; s_s[tid] = pt.y; s_cnt[tid] = __float_as_int(pt.z);
    if (__float_as_int(pt.w) || __float_as_int(pt.z) > f.cap) s_bad = 1;
  }
  __syncthreads();
  if (warp == 0) {                                                // merge the softmax partials of the segments
    float M = -FLT_MAX;
    for (int i = lane; i < nseg; i += 32) M = fmaxf(M, s_m[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, o));
    float sm = 0.f; int tot = 0;
    for (int i = lane; i < nseg; i += 32) { sm += s_s[i] * ex2_approx((s_m[i] - M) * LOG2E); tot += s_cnt[i]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { sm += __shfl_xor_sync(0xffffffffu, sm, o); tot += __shfl_xor_sync(0xffffffffu, tot, o); }
    if (lane == 0) { s_max = M; s_sum = sm; s_n = tot; }
  }
  __syncthreads();
  const int n = s_n;
  bool fallback = s_bad || n < k;
  if (!fallback) {
    const uint2* row_lists = f.lists + r * (int64_t)nseg * f.cap;
    const int64_t grow = a.row_offset + (int64_t)b * a.n + pos;
    const uint64_t seed = a.seed + (a.seed_dev ? *a.seed_dev : 0ull);
    tdiv = image_tdiv(a, b, tdiv);
    const float inv_t = 1.0f / tdiv;
    uint64_t aq0 = 0, aoff4 = 0; uint32_t ar0 = 0;
    if (MODE == 2) {            // flat index of logit (grow, v) in the reference's [B, n, V] noise tensor = grow * V + v = ar0 + v + S * aq0
      const uint64_t base = (uint64_t)grow * (uint64_t)V;
      aq0 = base / a.aten_stride; ar0 = (uint32_t)(base - aq0 * a.aten_stride);
      aoff4 = (a.aten_offset + (a.aten_offset_dev ? *a.aten_offset_dev : 0ull)) >> 2;
    }
    PhiloxRow prow;
    if (MODE == 0) prow = philox_row((uint32_t)a.step, (uint32_t)grow, (uint32_t)((uint64_t)grow >> 32), (uint32_t)seed, (uint32_t)(seed >> 32));
    int win_v = -1; float win_x = 0.f;
    for (int nex = 0; ; ++nex) {
      // ---- pass 1: perturbed argmax over the candidates that have not failed the rank test
      float bv = -FLT_MAX; int bi = 0x7fffffff; uint32_t bx = 0;
      lfn_for_each(row_lists, s_cnt, nseg, f.cap, warp, lane, [&](uint32_t xb, uint32_t vb) {
        const int v = (int)vb;
        bool skip = false;
        for (int e = 0; e < nex; ++e) skip |= s_excl[e] == v;
        if (skip) return;
        const float x = __uint_as_float(xb);
        float p;
        if (MODE != 0) {
          float u;
          if (MODE == 1) u = a.u[((int64_t)b * a.n + pos) * V + v];
          else { const uint32_t q = ar0 + (uint32_t)v, dq = q / a.aten_stride; u = aten_uniform(q - dq * a.aten_stride, aq0 + dq, aoff4, seed); }
          const float l1 = logf(fmaxf(u, 1e-20f));
          p = __fdiv_rn(x, tdiv) - logf(fmaxf(-l1, 1e-20f));
        } else {
          const float u = (float)(philox_first_row((uint32_t)v, prow) >> 8) * (1.0f / 16777216.0f);
          const float l1 = __logf(fmaxf(u, 1e-20f));
          p = fmaf(x, inv_t, -__logf(fmaxf(-l1, 1e-20f)));
        }
        if (bi == 0x7fffffff || better(p, v, bv, bi)) { bv = p; bi = v; bx = xb; }
      });
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o); const uint32_t ox = __shfl_xor_sync(0xffffffffu, bx, o);
        if (oi != 0x7fffffff && (bi == 0x7fffffff || better(ov, oi, bv, bi))) { bv = ov; bi = oi; bx = ox; }
      }
      __syncthreads();                                           // previous round's readers of the scratch are done
      if (lane == 0) { s_rv[warp] = bv; s_ri[warp] = bi; s_rx[warp] = bx; }
      __syncthreads();
      bv = s_rv[0]; bi = s_ri[0]; bx = s_rx[0];
#pragma unroll
      for (int w = 1; w < NW; ++w) {
        const float ov = s_rv[w]; const int oi = s_ri[w];
        if (oi != 0x7fffffff && (bi == 0x7fffffff || better(ov, oi, bv, bi))) { bv = ov; bi = oi; bx = s_rx[w]; }
      }
      if (bi == 0x7fffffff) break;                               // nothing left (degenerate row): win_v stays -1
      // ---- pass 2: exact rank of the winner's logit inside the row
      const float cx = __uint_as_float(bx);
      int c = 0;
      lfn_for_each(row_lists, s_cnt, nseg, f.cap, warp, lane, [&](uint32_t xb, uint32_t vb) {
        const float x = __uint_as_float(xb);
        c += (x > cx) || (x == cx && (int)vb < bi);
      });
      c = __reduce_add_sync(0xffffffffu, c);
      if (lane == 0) s_rc[warp] = c;
      __syncthreads();
      int rank = 0;
#pragma unroll
      for (int w = 0; w < NW; ++w) rank += s_rc[w];
      if (rank < k) { win_v = bi; win_x = cx; break; }
      if (nex == LFN_MAX_EXCL) { fallback = true; break; }
      if (tid == 0) s_excl[nex] = bi;
      __syncthreads();
    }
    if (!fallback) {
      if (tid == 0) {
        if (win_v < 0) { const uint2 e0 = row_lists[0]; win_v = (int)e0.y; win_x = __uint_as_float(e0.x); }    // degenerate rows (NaN logits)
        const float pr = expf(win_x - s_max) / s_sum;
        if (!a.only_masked || a.ids[(int64_t)b * a.n + pos] == a.mask_id) a.ids[(int64_t)b * a.n + pos] = win_v;
        a.scores[(int64_t)b * a.n + pos] = 1.0f - pr;
      }
      return;
    }
  }
  // the sampled threshold missed, a list overflowed, or too many winners failed the rank test: this row goes through the materialised path
  // (fallback kernels of this step)
  if (tid == 0) {
    const int slot = atomicAdd(f.fb_count, 1);
    atomicAdd(f.status, 1);
    if (slot < f.fb_cap) f.fb_rows[slot] = (int)r; else f.status[1] = 1;
    s_slot = slot;
  }
  __syncthreads();
  const int slot = s_slot;
  if (slot < f.fb_cap)
    for (int i = tid; i < f.K / 8; i += LFN_THREADS)
      reinterpret_cast<uint4*>(f.e_fb + (int64_t)slot * f.K)[i] = reinterpret_cast<const uint4*>(f.e + r * f.K)[i];
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
static inline uint64_t up256(uint64_t x) { return (x + 255) & ~uint64_t(255); }

struct LfPlan { int num_m_tiles, num_pm, S, npt, cap, ns, stride; };

// Splits of the N range: the static schedule hands item i to unit i % units; pick the smallest power-of-two S (npt = NT / S >= 2 tiles per
// item) whose makespan ceil(items / units) * npt is within 4 % of the best one.
static LfPlan lf_plan(int64_t R, int V, int k) {
  LfPlan pl{};
  pl.num_m_tiles = (int)((R + LF_BM - 1) / LF_BM);
  pl.num_pm = pl.num_m_tiles;
  const int units = num_sms();
  const int NT = V / LF_BN;
  long best = -1;
  auto span_of = [&](int s) { const long items = (long)pl.num_pm * s; return ((items + units - 1) / units) * (long)(NT / s); };
  for (int s = 1; s <= LF_MAX_SPLITS && s <= NT; s *= 2) {
    if (NT % s || (s > 1 && NT / s < 2)) break;
    const long span = span_of(s);
    if (best < 0 || span < best) best = span;
  }
  int best_s = 1;                                              // the smallest S within 4 % of the best makespan: fewer, longer list segments
  for (int s = 1; s <= LF_MAX_SPLITS && s <= NT; s *= 2) {
    if (NT % s || (s > 1 && NT / s < 2)) break;
    if (span_of(s) * 100 <= best * 104) { best_s = s; break; }
  }
  pl.S = best_s; pl.npt = NT / best_s;
  pl.stride = V > SMP_SAMPLE ? V / SMP_SAMPLE : 1;
  pl.ns = V / pl.stride;
  // list capacity per (row, split, chunk): the candidates of a row (at most SMP_CAP or the row falls back anyway) spread evenly over the 4 S
  // segments, plus 6 binomial sigmas, as whole 32-byte sectors
  const double per = (double)SMP_CAP / ((double)LF_SEGS * pl.S);
  int cap = (int)(per + 6.0 * sqrt(per) + 8.0);
  if (cap > 64 * pl.npt) cap = 64 * pl.npt;                    // a segment cannot hold more than the columns it sees (64 per tile)
  pl.cap = (cap + 3) / 4 * 4;
  (void)k;
  return pl;
}

struct LfWs { uint64_t S, thr, parts, lists, fb_count, fb_rows, e_fb, logits_fb, total; };
static LfWs lf_carve(int64_t R_max, int V, int K) {
  LfWs w{}; uint64_t o = 0;
  const int stride = V > SMP_SAMPLE ? V / SMP_SAMPLE : 1, ns = V / stride;
  uint64_t parts = 0, lists = 0;
  for (int64_t R = LF_BM; ; R += LF_BM) {                       // every row count of a step up to R_max (S shrinks as R grows)
    const int64_t Rc = R < R_max ? R : R_max;
    const LfPlan pl = lf_plan(Rc, V, 1);
    const uint64_t pb = (uint64_t)Rc * pl.S * LF_SEGS * 16, lb = (uint64_t)Rc * pl.S * LF_SEGS * pl.cap * 8;
    if (pb > parts) parts = pb;
    if (lb > lists) lists = lb;
    if (R >= R_max) break;
  }
  w.S = o;         o += up256((uint64_t)R_max * ns * 4);
  w.thr = o;       o += up256((uint64_t)R_max * 4);
  w.parts = o;     o += up256(parts);
  w.lists = o;     o += up256(lists);
  w.fb_count = o;  o += 256;
  w.fb_rows = o;   o += up256((uint64_t)LF_FB_CAP * 4);
  w.e_fb = o;      o += up256((uint64_t)LF_FB_CAP * K * 2);
  w.logits_fb = o; o += up256((uint64_t)LF_FB_CAP * V * 4);
  w.total = o;
  return w;
}

static bool lf_supported(int V, int K, int k) {
  if (V < 1024 || V % 256 || K % 64 || K < 64 || k < 1 || k > V) return false;
  if (V > SMP_SAMPLE && V % SMP_SAMPLE) return false;
  // the candidate list of a row (expected k + 4 sigma of the sample quantile, + 4 sigma of its own) must fit the finisher's shared memory
  const int stride = V > SMP_SAMPLE ? V / SMP_SAMPLE : 1, ns = V / stride;
  if (ns == V) return k + 64 <= SMP_CAP;
  const double pf = (double)k / V, mu = pf * ns, rs = mu + 4.0 * sqrt(mu * (1 - pf)) + 2.0;
  const double n_exp = rs * stride, sd = stride * sqrt(mu * (1 - pf));
  return n_exp + 4.0 * sd <= SMP_CAP;
}

template <bool XENT>
static int launch_lf(const LfParams& p, cudaStream_t st) {
  constexpr int SMEM = LfCfg<XENT>::SMEM_BYTES;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] { attr_err = cudaFuncSetAttribute(tc_logits_kernel<XENT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); });
  if (attr_err != cudaSuccess) return fail(MMG_ECUDA, "tc_logits setup: %s", cudaGetErrorString(attr_err));
  const int items = p.num_pm * p.S;
  const int units = items < num_sms() ? items : num_sms();
  MMG_CUDA(launch_pdl(tc_logits_kernel<XENT>, dim3(units), dim3(LF_THREADS), SMEM, st, p));
  MMG_LAUNCHED();
  return MMG_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------
// cross-entropy (MaskGit.forward, muse_maskgit_pytorch.py:335, 717-726): nll[r] = logsumexp_v(e_r . W_v) - e_r . W_label[r]
// ---------------------------------------------------------------------------------------------------------------------------
static bool lx_supported(int V, int K) { return V >= LF_BN && V % LF_BN == 0 && K >= 64 && K % 64 == 0; }

// the largest record array over every row count up to R_max (S shrinks as R grows)
static uint64_t lx_parts_bytes(int64_t R_max, int V) {
  uint64_t parts = 0;
  for (int64_t R = LF_BM; ; R += LF_BM) {
    const int64_t Rc = R < R_max ? R : R_max;
    const uint64_t pb = (uint64_t)Rc * lf_plan(Rc, V, 1).S * LF_SEGS * 16;
    if (pb > parts) parts = pb;
    if (R >= R_max) break;
  }
  return parts;
}

// one thread per row: the row's S x 2 segment records merged in split order (the same sums in the same order on every run)
__global__ void __launch_bounds__(256)
logits_xent_merge_kernel(const float4* __restrict__ parts, int nseg, int64_t R, float* __restrict__ nll) {
  pdl_wait(); pdl_trigger();
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float4* rec = parts + r * nseg;
  float M = -FLT_MAX;
  for (int i = 0; i < nseg; ++i) M = fmaxf(M, rec[i].x);
  float sum = 0.f, xl = __int_as_float(0x7fc00000);              // NaN unless a segment saw the label column
  for (int i = 0; i < nseg; ++i) {
    const float4 t = rec[i];
    sum += t.y * expf(t.x - M);
    if (__float_as_int(t.w)) xl = t.z;
  }
  nll[r] = M + logf(sum) - xl;
}

// materialised logits: one CTA per row, one pass of per-thread online (max, sum exp) pairs combined in a fixed tree order
constexpr int LXR_THREADS = 256;
__device__ __forceinline__ void lse_push(float& m, float& s, float x) {
  if (x > m) { s = s * expf(m - x) + 1.f; m = x; } else s += expf(x - m);
}
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  const float M = fmaxf(m, om);
  s = s * expf(m - M) + os * expf(om - M); m = M;
}
__global__ void __launch_bounds__(LXR_THREADS)
logits_xent_rows_kernel(const float* __restrict__ logits, int64_t ld, int V, const int32_t* __restrict__ labels, float* __restrict__ nll) {
  __shared__ float s_m[LXR_THREADS / 32], s_s[LXR_THREADS / 32];
  pdl_wait(); pdl_trigger();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r = blockIdx.x;
  const float* row = logits + r * ld;
  float m = -FLT_MAX, s = 0.f;
  if ((reinterpret_cast<uintptr_t>(row) & 15) == 0 && V % 4 == 0) {
    for (int i = tid; i < V / 4; i += LXR_THREADS) {
      const float4 x = __ldcs(reinterpret_cast<const float4*>(row) + i);
      lse_push(m, s, x.x); lse_push(m, s, x.y); lse_push(m, s, x.z); lse_push(m, s, x.w);
    }
  } else {
    for (int i = tid; i < V; i += LXR_THREADS) lse_push(m, s, __ldcs(row + i));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o); lse_merge(m, s, om, os); }
  if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
  __syncthreads();
  if (tid == 0) {
    m = s_m[0]; s = s_s[0];
    for (int w = 1; w < LXR_THREADS / 32; ++w) lse_merge(m, s, s_m[w], s_s[w]);
    const int lab = labels[r];
    nll[r] = (lab >= 0 && lab < V) ? m + logf(s) - row[lab] : __int_as_float(0x7fc00000);
  }
}

}  // namespace mmg

using namespace mmg;

extern "C" uint64_t mmg_logits_fused_workspace_bytes(int64_t R_max, int32_t V, int32_t K, int32_t k) {
  if (R_max <= 0 || !lf_supported(V, K, k)) return 0;
  return lf_carve(R_max, V, K).total;
}

extern "C" int mmg_logits_fused(const mmg_logits_fused_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->e && a->w && a->workspace && a->status, "mmg_logits_fused: NULL pointer");
  const mmg_logits_sample_args& s = a->s;
  MMG_CHECK_ARG(s.masked_pos && s.ids && s.scores, "mmg_logits_fused: NULL sampler pointer");
  MMG_CHECK_ARG(lf_supported(s.V, a->K, s.k), "mmg_logits_fused: unsupported V=%d K=%d k=%d (use mmg_linear + mmg_logits_sample)", s.V, a->K, s.k);
  MMG_CHECK_ARG(s.rng_mode == 0 || (s.rng_mode == 1 && s.aten_stride >= 256 && s.aten_stride % 256 == 0 && s.aten_offset % 4 == 0 && !s.u),
                "mmg_logits_fused: rng_mode=%d aten_stride=%u", s.rng_mode, s.aten_stride);
  const int64_t R = (int64_t)s.B * s.num_masked;
  if (R == 0) return MMG_OK;
  const int64_t R_cap = a->rows_capacity > 0 ? a->rows_capacity : R;
  MMG_CHECK_ARG(R <= R_cap, "mmg_logits_fused: %lld rows > rows_capacity %lld", (long long)R, (long long)R_cap);
  const LfWs ws = lf_carve(R_cap, s.V, a->K);
  MMG_CHECK_ARG(a->workspace_bytes >= ws.total, "mmg_logits_fused: workspace %llu < %llu bytes", (unsigned long long)a->workspace_bytes, (unsigned long long)ws.total);
  MMG_CHECK_ARG((reinterpret_cast<uintptr_t>(a->workspace) & 255) == 0 && (reinterpret_cast<uintptr_t>(a->e) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->w) & 15) == 0,
                "mmg_logits_fused: workspace must be 256-byte aligned, e / w 16-byte aligned");
  uint8_t* base = static_cast<uint8_t*>(a->workspace);
  float* S = reinterpret_cast<float*>(base + ws.S);
  float* thr = reinterpret_cast<float*>(base + ws.thr);
  float4* parts = reinterpret_cast<float4*>(base + ws.parts);
  uint2* lists = reinterpret_cast<uint2*>(base + ws.lists);
  int* fb_count = reinterpret_cast<int*>(base + ws.fb_count);
  int* fb_rows = reinterpret_cast<int*>(base + ws.fb_rows);
  bf16* e_fb = reinterpret_cast<bf16*>(base + ws.e_fb);
  float* logits_fb = reinterpret_cast<float*>(base + ws.logits_fb);
  const LfPlan pl = lf_plan(R, s.V, s.k);
  int rc;
  {   // 1. sample GEMM on the strided view of W (every `stride`-th vocabulary row)
    mmg_linear_args l{};
    l.a = a->e; l.w = a->w; l.M = R; l.N = pl.ns; l.K = a->K; l.lda = a->K; l.ldw = (int64_t)pl.stride * a->K; l.dtype = MMG_BF16; l.epilogue = MMG_EPI_STORE;
    l.epi.out = S; l.epi.ldo = pl.ns; l.epi.out_dtype = MMG_F32;
    if ((rc = linear_impl(&l, nullptr, stream))) return rc;
  }
  // 2. per-row candidate threshold
  if (pl.ns == s.V) MMG_CUDA(launch_pdl(logits_threshold_exact_kernel, dim3((unsigned)((R + THR_WARPS - 1) / THR_WARPS)), dim3(THR_WARPS * 32), 0, st, (const float*)S, pl.ns, s.k, thr, R, fb_count));
  else MMG_CUDA(launch_pdl(logits_threshold_kernel, dim3((unsigned)((R + THR_WARPS - 1) / THR_WARPS)), dim3(THR_WARPS * 32), 0, st, (const float*)S, pl.ns, s.V, s.k, thr, R, fb_count));
  MMG_LAUNCHED();
  {   // 3. the logits GEMM with the candidate / softmax epilogue
    LfParams p{};
    p.R = R; p.num_kb = a->K / LF_BK; p.num_m_tiles = pl.num_m_tiles; p.num_pm = pl.num_pm; p.S = pl.S; p.npt = pl.npt; p.cap = pl.cap;
    p.thr = thr; p.parts = parts; p.lists = lists;
    uint64_t da[2] = {(uint64_t)a->K, (uint64_t)R}; uint64_t sa[1] = {(uint64_t)a->K * 2}; uint32_t ba[2] = {LF_BK, LF_BM};
    if ((rc = make_tmap_bf16(&p.tma_a, a->e, 2, da, sa, ba))) return rc;
    uint64_t db[2] = {(uint64_t)a->K, (uint64_t)s.V}; uint64_t sb[1] = {(uint64_t)a->K * 2}; uint32_t bb[2] = {LF_BK, (uint32_t)LF_BN};
    if ((rc = make_tmap_bf16(&p.tma_b, a->w, 2, db, sb, bb))) return rc;
    if ((rc = launch_lf<false>(p, st))) return rc;
  }
  float t = s.temperature; if (t < 1e-10f) t = 1e-10f;      // max(temperature, 1e-10): muse_maskgit_pytorch.py:411
  {   // 4. finish
    LfFinish f{};
    f.parts = parts; f.lists = lists; f.S = pl.S; f.cap = pl.cap; f.e = reinterpret_cast<const bf16*>(a->e); f.K = a->K;
    f.fb_count = fb_count; f.fb_rows = fb_rows; f.e_fb = e_fb; f.fb_cap = LF_FB_CAP; f.status = a->status;
    static const int minb = [] { const char* e = getenv("MMG_FINISH_MINB"); return e ? atoi(e) : 4; }();
    if (s.u) MMG_CUDA(launch_pdl(logits_finish_kernel<1, 4>, dim3((unsigned)R), dim3(LFN_THREADS), 0, st, s, t, f));
    else if (s.rng_mode == 1) MMG_CUDA(launch_pdl(logits_finish_kernel<2, 4>, dim3((unsigned)R), dim3(LFN_THREADS), 0, st, s, t, f));
    else if (minb == 6) MMG_CUDA(launch_pdl(logits_finish_kernel<0, 6>, dim3((unsigned)R), dim3(LFN_THREADS), 0, st, s, t, f));
    else MMG_CUDA(launch_pdl(logits_finish_kernel<0, 4>, dim3((unsigned)R), dim3(LFN_THREADS), 0, st, s, t, f));
    MMG_LAUNCHED();
  }
  {   // 5. fallback rows: materialised logits of at most LF_FB_CAP rows (the kernel exits at once when no row was flagged)
    mmg_linear_args l{};
    l.a = e_fb; l.w = a->w; l.M = LF_FB_CAP; l.N = s.V; l.K = a->K; l.lda = a->K; l.ldw = a->K; l.dtype = MMG_BF16; l.epilogue = MMG_EPI_STORE;
    l.epi.out = logits_fb; l.epi.ldo = s.V; l.epi.out_dtype = MMG_F32;
    if ((rc = linear_impl(&l, fb_count, stream))) return rc;
  }
  {   // 6. ... sampled by the materialised-logits kernel through the row index list
    mmg_logits_sample_args fs = s;
    fs.logits = logits_fb; fs.row_index = fb_rows; fs.row_count_dev = fb_count; fs.row_index_cap = LF_FB_CAP;
    if ((rc = mmg_logits_sample(&fs, stream))) return rc;
  }
  return MMG_OK;
}

extern "C" uint64_t mmg_logits_xent_workspace_bytes(int64_t rows_capacity, int32_t V, int32_t K) {
  if (rows_capacity <= 0 || !lx_supported(V, K)) return 0;
  return up256(lx_parts_bytes(rows_capacity, V));
}

extern "C" int mmg_logits_xent(const mmg_logits_xent_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->e && a->w && a->labels && a->nll && a->workspace, "mmg_logits_xent: NULL pointer");
  MMG_CHECK_ARG(lx_supported(a->V, a->K), "mmg_logits_xent: unsupported V=%d K=%d (use mmg_linear + mmg_logits_xent_rows)", a->V, a->K);
  MMG_CHECK_ARG(a->rows >= 0, "mmg_logits_xent: rows=%lld", (long long)a->rows);
  const int64_t R = a->rows;
  if (R == 0) return MMG_OK;
  const int64_t R_cap = a->rows_capacity > 0 ? a->rows_capacity : R;
  MMG_CHECK_ARG(R <= R_cap, "mmg_logits_xent: %lld rows > rows_capacity %lld", (long long)R, (long long)R_cap);
  const uint64_t need = up256(lx_parts_bytes(R_cap, a->V));
  MMG_CHECK_ARG(a->workspace_bytes >= need, "mmg_logits_xent: workspace %llu < %llu bytes", (unsigned long long)a->workspace_bytes, (unsigned long long)need);
  MMG_CHECK_ARG((reinterpret_cast<uintptr_t>(a->workspace) & 255) == 0 && (reinterpret_cast<uintptr_t>(a->e) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->w) & 15) == 0,
                "mmg_logits_xent: workspace must be 256-byte aligned, e / w 16-byte aligned");
  float4* parts = static_cast<float4*>(a->workspace);
  const LfPlan pl = lf_plan(R, a->V, 1);
  int rc;
  {   // the logits GEMM with the cross-entropy epilogue: per (row, split, 64-column half) softmax partials and the label's logit
    LfParams p{};
    p.R = R; p.num_kb = a->K / LF_BK; p.num_m_tiles = pl.num_m_tiles; p.num_pm = pl.num_pm; p.S = pl.S; p.npt = pl.npt;
    p.parts = parts; p.labels = a->labels;
    uint64_t da[2] = {(uint64_t)a->K, (uint64_t)R}; uint64_t sa[1] = {(uint64_t)a->K * 2}; uint32_t ba[2] = {LF_BK, LF_BM};
    if ((rc = make_tmap_bf16(&p.tma_a, a->e, 2, da, sa, ba))) return rc;
    uint64_t db[2] = {(uint64_t)a->K, (uint64_t)a->V}; uint64_t sb[1] = {(uint64_t)a->K * 2}; uint32_t bb[2] = {LF_BK, (uint32_t)LF_BN};
    if ((rc = make_tmap_bf16(&p.tma_b, a->w, 2, db, sb, bb))) return rc;
    if ((rc = launch_lf<true>(p, st))) return rc;
  }
  MMG_CUDA(launch_pdl(logits_xent_merge_kernel, dim3((unsigned)((R + 255) / 256)), dim3(256), 0, st, (const float4*)parts, LF_SEGS * pl.S, R, a->nll));
  MMG_LAUNCHED();
  return MMG_OK;
}

extern "C" int mmg_logits_xent_rows(const mmg_logits_xent_rows_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->logits && a->labels && a->nll, "mmg_logits_xent_rows: NULL pointer");
  MMG_CHECK_ARG(a->V >= 1 && a->rows >= 0 && a->ld >= a->V, "mmg_logits_xent_rows: rows=%lld V=%d ld=%lld", (long long)a->rows, a->V, (long long)a->ld);
  if (a->rows == 0) return MMG_OK;
  MMG_CUDA(launch_pdl(logits_xent_rows_kernel, dim3((unsigned)a->rows), dim3(LXR_THREADS), 0, st, a->logits, a->ld, a->V, a->labels, a->nll));
  MMG_LAUNCHED();
  return MMG_OK;
}

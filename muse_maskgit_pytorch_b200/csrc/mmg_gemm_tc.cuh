// wgmma / TMA GEMM for sm_90a:  C[M,N] = A[M,K] * W[N,K]^T, bf16 (or e4m3) operands, fp32 accumulation in registers.
//
//   warp 0      : TMA producer  (one elected lane) — A tile 128x64 and W tile BNx64 per k-block, SWIZZLE_128B, STAGES-deep ring
//                 (e4m3 operands: 128 x 128 and BN x 128 — the same 128-byte rows, so the ring, boxes and descriptors are unchanged)
//   warps 4..11 : two consumer warpgroups.  Warpgroup g multiplies rows [64 g, 64 g + 64) of the tile (wgmma m64nBNk16, 4 per k-block,
//                 accumulators in registers), then runs the fused Epilogue on those rows (EPI_MODE below): from the accumulator
//                 registers into per-warp shared-memory boxes, then a TMA store / TMA reduction (tile epilogues) or one lane per row and
//                 64-column chunk (TC_EPI_REGS, TC_EPI_ACT).  setmaxnreg moves registers from warpgroup 0 (40/thread) to the consumers
//                 (232/thread).
//   persistent grid (<= #SM CTAs), static tile schedule (M- or N-fastest); the producer runs ahead into the next tile while the consumers
//   finish the epilogue of the current one.
//
// A is either a dense [M,K] matrix (2-D tensor map) or an NHWC activation addressed as an implicit-GEMM
// convolution: the k-block (tap, channel-chunk) is fetched with a 4-D tensor map at shifted (x+dx, y+dy)
// coordinates and TMA's out-of-bounds zero fill provides the padding — no im2col buffer.
#pragma once
#include "mmg_common.cuh"
#include "mmg_sm90.cuh"
#include "mmg_epilogue.cuh"

namespace mmg {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;
constexpr int TC_THREADS = 384;          // warpgroup 0: warp 0 TMA (1-3 idle); warpgroups 1-2: wgmma + epilogue
constexpr int TC_EPI_WARPS = 8;
constexpr int TC_MAX_TAPS = 16;
constexpr int TC_SMEM_LIMIT = 227 * 1024;

// How the epilogue's results leave the CTA (the EPI_MODE of tc_gemm_kernel; described above the kernel).  The launcher picks one per product.
enum TcEpiMode : int {
  TC_EPI_REGS = 0,      // every Epilogue kind: fragments -> per-warp box -> one lane per row (CONVT_RGB: a quad reduction of the fragments)
  TC_EPI_REDUCE = 2,    // in-place residual: per-warp tiles + TMA reduction
  TC_EPI_TSTORE = 3,    // plain fp32: per-warp tiles + TMA store
  TC_EPI_QKV = 4,       // QKV heads: per-warp tiles + TMA stores
  TC_EPI_GEGLU = 5,     // GEGLU, BN = 256: per-warp tiles + TMA store
  TC_EPI_ACT = 6,       // T5 feed-forward epilogues (GEGLU_TANH, STORE + ReLU), BN = 128: TC_EPI_REGS's box, one lane per row
};
// the modes whose epilogue writes whole output boxes with TMA; the other two run an Epilogue kind on one row chunk per lane
constexpr bool tc_tile_epilogue(int mode) { return mode != TC_EPI_REGS && mode != TC_EPI_ACT; }

struct alignas(64) TcGemmParams {
  CUtensorMap tma_a[4];
  CUtensorMap tma_b;
  CUtensorMap tma_out;      // REDUCE / TSTORE: the fp32 output [M, N] in boxes of 16 rows x 32 columns (128 B), SWIZZLE_128B; GEGLU: bf16 [M, N/2], 16 x 64
  CUtensorMap tma_qkv[3];   // QKV: q / k / v as [rows, 64] bf16 matrices in boxes of 16 rows x 64 columns (128 B)
  int64_t M, N;
  int num_kb, num_m_tiles, num_n_tiles;
  int mode;                 // 0 dense, 1 conv (4-D A maps)
  int n_fast;               // tile order: 0 = consecutive tiles walk M (the W tile is shared by the CTAs in flight: huge N, e.g. the logits
                            // GEMM), 1 = consecutive tiles walk N (all column tiles of an A row block run together, so A streams from HBM once:
                            // small W that stays L2 resident, e.g. the N = 512 residual GEMMs)
  int cchunks, ntaps;       // conv: k-block = tap * cchunks + channel chunk
  int8_t tap_map[TC_MAX_TAPS], tap_dy[TC_MAX_TAPS], tap_dx[TC_MAX_TAPS];
  int TW, TH, TB, tiles_x, tiles_y;   // conv: tile = TB images x TH rows x TW cols of the OUTPUT grid (Ho x Wo)
  int Ho, Wo, B;
  const int* skip_if_zero;  // optional device word written by an earlier kernel of the stream: 0 -> every CTA returns at once
  Epilogue epi;
  const float* a_scale;     // e4m3 operands: the product of row r, column c is acc * a_scale[r] * w_scale[c] ([M], [N])
  const float* w_scale;
};

// Shared memory: [<= 1 KB to align][operand ring][barriers, 1 KB][per-warp output boxes, 32 KB]: 4 operand stages at BN = 256 and 6 at
// BN <= 128; the 512 B static s_scale fits in what the 227 KB limit leaves over.
template <int BN> struct TcCfg {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int TILE_BYTES = TC_EPI_WARPS * 4096;
  static constexpr int FIT = (TC_SMEM_LIMIT - 1024 - 1024 - TILE_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT < 6 ? FIT : 6;
  static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 1024 + TILE_BYTES;
  static_assert(STAGES >= 2, "operand ring too shallow");
  static_assert(SMEM_BYTES + 512 <= TC_SMEM_LIMIT, "dynamic + static shared memory over the opt-in limit");
};

// The Epilogue kinds (mmg_epilogue.cuh) are written for one thread that owns a 64-column chunk of a row.  The tile epilogues need no
// such thing: each of their terms is elementwise, or (GEGLU) pairs column i with column 32 + i, which the wgmma fragment keeps in the
// same thread.  They go from the accumulator registers straight into the warp's output boxes, and the TMA engine writes the boxes out.
// Thread t of a warpgroup (warp w, lane l) holds rows 16 w + l / 4 and + 8 at columns 8 j + 2 (l % 4) and + 1, so a warp owns 16 whole
// rows; a box is 16 rows x 128 bytes (TMA 128-byte swizzle), and the warp's 4 KB tile double-buffers two.  The launcher takes a tile
// epilogue only at a tile width BN that divides N, so every box lies inside the N columns.
// TC_EPI_REGS and TC_EPI_ACT use the same 4 KB per warp as one fp32 box of its 16 rows x 64 columns: each 64-column chunk of the fragments
// goes into it, and lane r < 16 reads row r back and runs the Epilogue kind on it (TC_EPI_ACT: apply_act), so every kind computes what it
// computes elsewhere, element for element.  CONVT_RGB never forms a row: each thread projects its own fragment columns onto the (<= 4)
// RGB weights and two shuffles finish the sum over the lane quad that shares a row.
// TC_EPI_REDUCE: in-place residual epilogues (out == resid, fp32) push the term they add with a TMA reduction
// (cp.reduce.async.bulk.tensor .add), 32 columns per box: the residual is never read and the adds happen in L2.
// TC_EPI_TSTORE: plain fp32 outputs (no bias / activation; the logits GEMM) leave through the same boxes with a TMA store.
// TC_EPI_QKV: the QKV epilogue (bf16; tokens % 32 == 0 and M % 128 == 0, so a warp's 16 rows are 16 consecutive tokens of one
// sequence and land on 16 consecutive rows of one head of q / k / v): one box and one TMA store per warp and head chunk.
// TC_EPI_GEGLU: the GEGLU epilogue (bf16 out, BN == 256): two 64-column chunks make 64 outputs = one box per warp.
// e4m3 operands (TA = __nv_fp8_e4m3; the dense QKV and GEGLU tile epilogues, and the register epilogues of the convolutions): a k-block
// is 128 elements, four m64nBNk32 wgmma, and the epilogue starts by dequantising the fragment with dequant_acc (per-row A scales) or
// dequant_acc_images (per-image A scales, conv mode); everything after it is the bf16 code.
template <int BN>
__device__ __forceinline__ void dequant_acc(float (&acc)[BN / 2], const float* __restrict__ a_scale, const float* __restrict__ w_scale,
                                            int64_t brow, int64_t M, int col0, int lane) {
  const int q = lane & 3, fr = lane >> 2;
  const float sa0 = brow + fr < M ? __ldg(a_scale + brow + fr) : 0.f;         // rows past M hold zero accumulators
  const float sa1 = brow + fr + 8 < M ? __ldg(a_scale + brow + fr + 8) : 0.f;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const float2 ws = __ldg(reinterpret_cast<const float2*>(w_scale + col0 + 8 * j + 2 * q));
    acc[4 * j] *= sa0 * ws.x; acc[4 * j + 1] *= sa0 * ws.y;
    acc[4 * j + 2] *= sa1 * ws.x; acc[4 * j + 3] *= sa1 * ws.y;
  }
}

// e4m3 convolutions (mode 1, register epilogues): A holds one scale per IMAGE (mmg_quantize_e4m3_images), which factors out of the sum
// over taps and channels because an output pixel reads only pixels of its own image.  The warp's fragment rows r0 + l / 4 and + 8 of
// the tile belong to image bt * TB + row / (TW * TH); rows of images past B hold zero accumulators and are never stored.
template <int BN>
__device__ __forceinline__ void dequant_acc_images(float (&acc)[BN / 2], const TcGemmParams& p, int m_blk, int r0, int col0, int lane) {
  const int q = lane & 3, fr = lane >> 2;
  const int per = p.TW * p.TH, bbase = (m_blk / (p.tiles_x * p.tiles_y)) * p.TB;
  const int b0 = bbase + (r0 + fr) / per, b1 = bbase + (r0 + fr + 8) / per;
  const float sa0 = b0 < p.B ? __ldg(p.a_scale + b0) : 0.f;
  const float sa1 = b1 < p.B ? __ldg(p.a_scale + b1) : 0.f;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const float2 ws = __ldg(reinterpret_cast<const float2*>(p.w_scale + col0 + 8 * j + 2 * q));
    acc[4 * j] *= sa0 * ws.x; acc[4 * j + 1] *= sa0 * ws.y;
    acc[4 * j + 2] *= sa1 * ws.x; acc[4 * j + 3] *= sa1 * ws.y;
  }
}

template <int BN, int EPI_MODE, typename TA = bf16>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ TcGemmParams p) {
  using namespace sm90;
  using Cfg = TcCfg<BN>;
  constexpr bool FP8 = sizeof(TA) == 1;
  constexpr int BK = 128 / (int)sizeof(TA);           // elements per k-block: one 128-byte row
  static_assert(!FP8 || EPI_MODE == TC_EPI_QKV || EPI_MODE == TC_EPI_GEGLU || EPI_MODE == TC_EPI_REGS,
                "e4m3 operands are dequantised by the QKV / GEGLU tile epilogues (dense) or the register epilogues (convolutions) only");
  // e4m3 convolutions: a k-block is one tap x 128 channels.  The dense e4m3 instantiations never run mode 1 and keep the bf16 channel step.
  constexpr bool FP8_CONV = FP8 && EPI_MODE == TC_EPI_REGS;
  constexpr int CBK = FP8_CONV ? BK : TC_BK;
  constexpr bool RED = EPI_MODE == TC_EPI_REDUCE || EPI_MODE == TC_EPI_TSTORE, RED_ADD = EPI_MODE == TC_EPI_REDUCE;   // TSTORE: same tiles, plain TMA store
  constexpr bool QKVT = EPI_MODE == TC_EPI_QKV;
  constexpr bool GEGLUT = EPI_MODE == TC_EPI_GEGLU;
  constexpr bool ACTT = EPI_MODE == TC_EPI_ACT;
  constexpr bool TILES = tc_tile_epilogue(EPI_MODE);
  static_assert(!GEGLUT || BN == 256, "the GEGLU tile epilogue pairs adjacent 64-column chunks of a 256-column tile");
  constexpr int STAGES = Cfg::STAGES;
  constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;

  if (p.skip_if_zero) { pdl_wait(); if (*p.skip_if_zero == 0) return; }       // uniform over the grid: nothing has been set up yet

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint8_t* tiles = smem + STAGES * STAGE_BYTES + 1024;      // per-warp output boxes, 4 KB each

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int tile0 = (int)blockIdx.x, tile_step = (int)gridDim.x;
  __shared__ float s_scale[128];               // QKV epilogue: q_scale | k_scale staged once per CTA
  if (p.epi.kind == MMG_EPI_QKV && threadIdx.x < 128) {
    const float* src = threadIdx.x < 64 ? p.epi.p.q_scale : p.epi.p.k_scale;
    s_scale[threadIdx.x] = src ? src[threadIdx.x & 63] : 1.f;
  }

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&p.tma_b);
    prefetch_tmap(&p.tma_a[0]);
    for (int i = 0; i < STAGES; ++i) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, TC_EPI_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                                   // everything above overlapped the previous kernel's tail
  pdl_trigger();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && elect_one()) {
      // ===================== TMA producer =====================
      int stage = 0; uint32_t phase = 0;
      for (int tile = tile0; tile < num_tiles; tile += tile_step) {
        const int m_blk = p.n_fast ? tile / p.num_n_tiles : tile % p.num_m_tiles, n_blk = p.n_fast ? tile % p.num_n_tiles : tile / p.num_m_tiles;
        int x0 = 0, y0 = 0, b0 = 0;
        if (p.mode == 1) {
          const int xt = m_blk % p.tiles_x, yt = (m_blk / p.tiles_x) % p.tiles_y, bt = m_blk / (p.tiles_x * p.tiles_y);
          x0 = xt * p.TW; y0 = yt * p.TH; b0 = bt * p.TB;
        }
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(empty_bar + stage, phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          mbar_expect_tx(full_bar + stage, STAGE_BYTES);
          if (p.mode == 0) {
            tma_load_2d(sa, &p.tma_a[0], full_bar + stage, kb * BK, m_blk * TC_BM);
          } else {
            const int tap = kb / p.cchunks, cc = kb - tap * p.cchunks;
            tma_load_4d(sa, &p.tma_a[p.tap_map[tap]], full_bar + stage, cc * CBK, x0 + p.tap_dx[tap], y0 + p.tap_dy[tap], b0);
          }
          tma_load_2d(sb, &p.tma_b, full_bar + stage, kb * BK, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===================== consumer warpgroups: wgmma main loop, then the epilogue of their 64 rows =====================
    const int wg = (warp - 4) >> 2, wq = warp & 3;
    Epilogue epi = p.epi;
    if (epi.kind == MMG_EPI_QKV) { epi.p.q_scale = s_scale; epi.p.k_scale = s_scale + 64; }
    const bool prefetch_resid = epi.can_prefetch_resid();
    const uint32_t wtile = smem_u32(tiles) + (uint32_t)(warp - 4) * 4096u;   // tile epilogues: this warp's two 2 KB output boxes
    uint32_t nbox = 0;                                                         // boxes this warp has filled so far
    int stage = 0; uint32_t phase = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
      const int m_blk = p.n_fast ? tile / p.num_n_tiles : tile % p.num_m_tiles, n_blk = p.n_fast ? tile % p.num_n_tiles : tile / p.num_m_tiles;
      // tile epilogues: the warp's 16 fragment rows start at brow; LNFOLD statistics of row brow + l / 4 + 8 (l % 4) in lanes l % 4 < 2
      const int64_t brow = (int64_t)m_blk * TC_BM + wg * 64 + 16 * wq;
      float ln_a = 0.f, ln_b = 0.f;
      if (RED_ADD && epi.kind == MMG_EPI_LNFOLD_RESIDUAL && (lane & 3) < 2 && brow + (lane >> 2) + 8 * (lane & 3) < p.M)
        epi.ln_row_stats(brow + (lane >> 2) + 8 * (lane & 3), ln_a, ln_b);

      // ---- main loop: 4 wgmma (K = 16, e4m3: 32) per k-block; a ring slot goes back to the producer once the wgmma group after it was issued ----
      // e4m3 convolutions promote instead: the fp8 tensor core adds each k32 step into its accumulator with fewer bits than fp32, so every
      // k-block starts a fresh accumulator, waits for its own group, and is added into the fp32 sum `tot` (one promotion per 128 elements
      // of K, BN / 2 more registers per thread).  The dense e4m3 products (K = 512: four k-blocks) accumulate in place.
      float tot[FP8_CONV ? BN / 2 : 1];
      if constexpr (FP8_CONV) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) tot[i] = 0.f;
      }
      int prev_stage = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(full_bar + stage, phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        const uint64_t adesc = smem_desc_kmajor_sw128(sa + (uint32_t)wg * 8192u);
        const uint64_t bdesc = smem_desc_kmajor_sw128(sa + Cfg::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if constexpr (FP8_CONV) WgmmaE4m3<BN>::mma(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), k ? 1u : 0u);
          else if constexpr (FP8) WgmmaE4m3<BN>::mma(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
          else Wgmma<BN>::template mma<0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
        }
        wgmma_commit();
        if constexpr (FP8_CONV) {
          wgmma_wait<0>();
          reg_fence(acc);
          __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + stage);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) tot[i] += acc[i];
        } else {
          wgmma_wait<1>();
          if (prev_stage >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + prev_stage); }
          prev_stage = stage;
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (prev_stage >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + prev_stage); }
      if constexpr (FP8_CONV) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = tot[i];
      }

      if constexpr (TILES) {
        // ---- tile epilogues, from the accumulator fragments (layout above the kernel) ----
        // acc[4 j + e] / acc[4 j + 2 + e] = rows fr / fr + 8 of the warp's 16 at column 8 j + 2 q + e of the tile; the boxes' rows are
        // 128 bytes whose 16-byte chunk k sits at k ^ (row & 7), and (fr + 8) & 7 == fr
        if constexpr (FP8) dequant_acc<BN>(acc, p.a_scale, p.w_scale, brow, p.M, n_blk * BN, lane);
        const int q = lane & 3, fr = lane >> 2;
        const uint32_t rowa = (uint32_t)fr * 128u, rowb = rowa + 1024u;
        // the next free 2 KB box of the warp's tile: the store two boxes back has read it
        auto box_begin = [&]() {
          if (lane == 0) bulk_wait_read1();
          __syncwarp();
          const uint32_t b = wtile + (nbox & 1u) * 2048u;
          ++nbox;
          return b;
        };
        // generic-proxy writes -> visible to the TMA (async-proxy) read
        auto box_ready = [&]() { fence_proxy_async(); __syncwarp(); };
        if constexpr (RED) {
          // rows past M are zero accumulators and are clipped by the tensor map
          float a0 = 0.f, b0 = 0.f, a1 = 0.f, b1 = 0.f;
          if (RED_ADD && epi.kind == MMG_EPI_LNFOLD_RESIDUAL) {
            a0 = __shfl_sync(0xffffffffu, ln_a, lane & ~3); b0 = __shfl_sync(0xffffffffu, ln_b, lane & ~3);
            a1 = __shfl_sync(0xffffffffu, ln_a, (lane & ~3) | 1); b1 = __shfl_sync(0xffffffffu, ln_b, (lane & ~3) | 1);
          }
#pragma unroll
          for (int g = 0; g < BN / 32; ++g) {                 // one box = 32 fp32 columns
            const int col = n_blk * BN + 32 * g;
            const uint32_t box = box_begin();
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * g + jj, c = col + 8 * jj + 2 * q;
              float x0 = acc[4 * j], x1 = acc[4 * j + 1], y0 = acc[4 * j + 2], y1 = acc[4 * j + 3];
              if (RED_ADD) {
                x0 = epi.resid_term(x0, c, a0, b0); x1 = epi.resid_term(x1, c + 1, a0, b0);
                y0 = epi.resid_term(y0, c, a1, b1); y1 = epi.resid_term(y1, c + 1, a1, b1);
              }
              const uint32_t off = (uint32_t)(((2 * jj + (q >> 1)) ^ fr) * 16 + 8 * (q & 1));
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" :: "r"(box + rowa + off), "f"(x0), "f"(x1) : "memory");
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" :: "r"(box + rowb + off), "f"(y0), "f"(y1) : "memory");
            }
            box_ready();
            if (lane == 0) {
              if (RED_ADD) tma_reduce_add_2d(&p.tma_out, box, col, (int)brow);
              else tma_store_2d(&p.tma_out, box, col, (int)brow);
              bulk_commit();
            }
          }
        } else if constexpr (GEGLUT) {
          // rows past M are zero accumulators and are clipped by the tensor map
#pragma unroll
          for (int bx = 0; bx < 2; ++bx) {                    // one box = chunks 2 bx, 2 bx + 1 = 64 bf16 outputs
            const int col0 = n_blk * BN + 128 * bx;
            const uint32_t box = box_begin();
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {                // output columns 32 cc + 8 jj + 2 q + e = x column 8 jx + ..., gate column 8 jg + ...
                const int jx = 8 * (2 * bx + cc) + jj, jg = jx + 4;
                const uint32_t off = (uint32_t)(((4 * cc + jj) ^ fr) * 16 + 4 * q);
                asm volatile("st.shared.b32 [%0], %1;" :: "r"(box + rowa + off),
                             "r"(pack_bf16(acc[4 * jg] * gelu_fast(acc[4 * jx]), acc[4 * jg + 1] * gelu_fast(acc[4 * jx + 1]))) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" :: "r"(box + rowb + off),
                             "r"(pack_bf16(acc[4 * jg + 2] * gelu_fast(acc[4 * jx + 2]), acc[4 * jg + 3] * gelu_fast(acc[4 * jx + 3]))) : "memory");
              }
            }
            box_ready();
            if (lane == 0) { tma_store_2d(&p.tma_out, box, col0 >> 1, (int)brow); bulk_commit(); }
            if (epi.p.row_stats) {
              // each chunk's (sum, sumsq) of its bf16 outputs in ascending column order (geglu_chunk's), read back from the box:
              // lane l sums row l % 16 of chunk 2 bx + l / 16
              const int rr = lane & 15, cc = lane >> 4, cs = col0 + 64 * cc;
              if (brow + rr < p.M) {
                float sx = 0.f, sq = 0.f;
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                  uint32_t w[4];
                  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
                               : "r"(box + (uint32_t)rr * 128u + (uint32_t)(((4 * cc + jj) ^ (rr & 7)) * 16)) : "memory");
#pragma unroll
                  for (int k = 0; k < 8; ++k) {
                    const float t = __uint_as_float((k & 1) ? (w[k >> 1] & 0xffff0000u) : (w[k >> 1] << 16));
                    sx += t; sq = fmaf(t, t, sq);
                  }
                }
                reinterpret_cast<float2*>(epi.p.row_stats)[(brow + rr) * (int64_t)epi.p.stats_slots + (cs >> 6)] = make_float2(sx, sq);
              }
            }
          }
        } else if constexpr (QKVT) {
          const uint32_t rw = (uint32_t)brow, tok = (uint32_t)epi.p.tokens;
          const uint32_t bq = rw / tok, t0 = rw - bq * tok;   // warp-uniform: the 16 rows are tokens t0 .. t0+15 of sequence bq
#pragma unroll
          for (int c = 0; c < BN / 64; ++c) {                 // one box = one head chunk
            const int col0 = n_blk * BN + 64 * c;
            int h;
            const int which = epi.qkv_head(col0, h);
            const float* sc = which == 0 ? epi.p.q_scale : (which == 1 ? epi.p.k_scale : nullptr);
            float t[32];                                      // t[2 jj + e]: row fr, t[16 + 2 jj + e]: row fr + 8, at head column 8 jj + 2 q + e
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int e = 0; e < 2; ++e) { t[2 * jj + e] = acc[4 * (8 * c + jj) + e]; t[16 + 2 * jj + e] = acc[4 * (8 * c + jj) + 2 + e]; }
            if (sc) {
              // qkv_chunk's sum of squares, bit for bit: chain k = i & 3 over ascending columns i, then (s0 + s1) + (s2 + s3).  Chain
              // 2 (q & 1) + e of a row is columns 8 jj + 2 (q & 1) + e (lane q & 1) and + 4 (lane q | 2), jj ascending: lanes q < 2 run
              // it for row fr, lanes q >= 2 for row fr + 8, each after fetching the other half from lane q ^ 2
              const bool up = (q & 2) != 0;
              float s[2] = {0.f, 0.f};
#pragma unroll
              for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float mine = up ? t[16 + 2 * jj + e] : t[2 * jj + e], give = up ? t[2 * jj + e] : t[16 + 2 * jj + e];
                  const float got = __shfl_xor_sync(0xffffffffu, give, 2);
                  const float lo = up ? got : mine, hi = up ? mine : got;
                  s[e] = fmaf(lo, lo, s[e]);
                  s[e] = fmaf(hi, hi, s[e]);
                }
              const float pair = s[0] + s[1];
              const float ss = pair + __shfl_xor_sync(0xffffffffu, pair, 1);
              const float inv = rsqrtf(fmaxf(ss, 1e-24f)), inv_x = __shfl_xor_sync(0xffffffffu, inv, 2);
              const float i0 = up ? inv_x : inv, i1 = up ? inv : inv_x;
#pragma unroll
              for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float sv = sc[8 * jj + 2 * q + e];
                  t[2 * jj + e] = t[2 * jj + e] * i0 * sv;
                  t[16 + 2 * jj + e] = t[16 + 2 * jj + e] * i1 * sv;
                }
            }
            const uint32_t box = box_begin();
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const uint32_t off = (uint32_t)((jj ^ fr) * 16 + 4 * q);
              asm volatile("st.shared.b32 [%0], %1;" :: "r"(box + rowa + off), "r"(pack_bf16(t[2 * jj], t[2 * jj + 1])) : "memory");
              asm volatile("st.shared.b32 [%0], %1;" :: "r"(box + rowb + off), "r"(pack_bf16(t[16 + 2 * jj], t[16 + 2 * jj + 1])) : "memory");
            }
            box_ready();
            if (lane == 0) {
              const int64_t drow = which == 0 ? ((int64_t)bq * epi.p.heads + h) * epi.p.q_rows + t0
                                              : ((int64_t)bq * epi.p.heads + h) * epi.p.kv_rows + epi.p.key_off + t0;
              tma_store_2d(&p.tma_qkv[which], box, 0, (int)drow);
              bulk_commit();
              if (which != 0 && t0 == 0) epi.qkv_null_row(which, bq, h);
            }
          }
        }
      } else {
        // ---- TC_EPI_REGS and TC_EPI_ACT, from the accumulator fragments (layout above the kernel) ----
        const int r0 = wg * 64 + 16 * wq;                          // the warp's 16 rows of the tile
        if constexpr (FP8_CONV) dequant_acc_images<BN>(acc, p, m_blk, r0, n_blk * BN, lane);
        const int q = lane & 3, fr = lane >> 2;
        // global output row of tile row r; false for rows past M (dense) or of images past B (conv), which are never stored
        auto out_row = [&](int r, int64_t& orow) {
          if (p.mode == 0) { orow = (int64_t)m_blk * TC_BM + r; return orow < p.M; }
          const int xt = m_blk % p.tiles_x, yt = (m_blk / p.tiles_x) % p.tiles_y, bt = m_blk / (p.tiles_x * p.tiles_y);
          const int tx = r % p.TW, ty = (r / p.TW) % p.TH, b = bt * p.TB + r / (p.TW * p.TH);
          orow = ((int64_t)b * p.Ho + (yt * p.TH + ty)) * p.Wo + xt * p.TW + tx;
          return b < p.B;
        };
        if (!ACTT && epi.kind == MMG_EPI_CONVT_RGB) {
          // bias + LeakyReLU per element, then the <= 4 channel dot products over this thread's BN / 4 columns of rows fr and fr + 8, and
          // over the lane quad (shfl.xor 1, 2).  The launcher gives CONVT_RGB one tile of BN = N columns, so n_blk == 0 and every column
          // is valid.  Lane q = 0 writes row fr's pixel, lane q = 1 row fr + 8's (NCHW fp32).
          const mmg_epilogue_args& e = epi.p;
          float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + 2 * q;
            const float b0 = e.bias ? __ldg(e.bias + c) : 0.f, b1 = e.bias ? __ldg(e.bias + c + 1) : 0.f;
            const float x0 = leaky01(acc[4 * j] + b0), x1 = leaky01(acc[4 * j + 1] + b1);
            const float y0 = leaky01(acc[4 * j + 2] + b0), y1 = leaky01(acc[4 * j + 3] + b1);
#pragma unroll
            for (int ch = 0; ch < 4; ++ch) {
              if (ch < e.rgb_channels) {
                const float* w = e.rgb_w + (int64_t)ch * BN + c;
                const float w0 = __ldg(w), w1 = __ldg(w + 1);
                s0[ch] = fmaf(x1, w1, fmaf(x0, w0, s0[ch]));
                s1[ch] = fmaf(y1, w1, fmaf(y0, w0, s1[ch]));
              }
            }
          }
#pragma unroll
          for (int ch = 0; ch < 4; ++ch) {
            s0[ch] += __shfl_xor_sync(0xffffffffu, s0[ch], 1); s0[ch] += __shfl_xor_sync(0xffffffffu, s0[ch], 2);
            s1[ch] += __shfl_xor_sync(0xffffffffu, s1[ch], 1); s1[ch] += __shfl_xor_sync(0xffffffffu, s1[ch], 2);
          }
          int64_t orow;
          if (q < 2 && out_row(r0 + fr + 8 * q, orow)) {
            const uint32_t hw = (uint32_t)(e.H * e.W), rr = (uint32_t)orow;
            const int64_t b = rr / hw;
            const int rem = (int)(rr - (uint32_t)b * hw), y = rem / e.W, x = rem - y * e.W;
            const int64_t plane = (int64_t)(2 * e.H) * (2 * e.W), pix = (int64_t)(2 * y + e.py) * (2 * e.W) + 2 * x + e.px;
            float* o = reinterpret_cast<float*>(e.out) + b * e.rgb_channels * plane + pix;
#pragma unroll
            for (int ch = 0; ch < 4; ++ch)
              if (ch < e.rgb_channels) o[ch * plane] = e.rgb_b[ch] + (q ? s1[ch] : s0[ch]);
          }
        } else if constexpr (BN <= 128) {
          // every other kind, 64 columns at a time: the fragments of chunk c -> the warp's box (16 rows of 256 B; 16-byte slot k of row r
          // at k ^ (r & 7), conflict-free for both the fragment writes and the row reads) -> lane r < 16 runs row r0 + r.  The launchers
          // give these kinds BN <= 128 only: at BN = 256 the 128 accumulators and a 64-column row would not fit the registers.
          const uint32_t box = smem_u32(tiles) + (uint32_t)(warp - 4) * 4096u;
          int64_t orow = 0;
          const bool own = lane < 16 && out_row(r0 + lane, orow);
          if (own) epi.begin_row(orow);
#pragma unroll
          for (int c = 0; c < BN / 64; ++c) {
            const int col0 = n_blk * BN + 64 * c;
            if (col0 >= p.N) break;
            __syncwarp();                                        // the lanes are done reading the previous chunk
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * c + jj;
              const uint32_t off = (uint32_t)(((2 * jj + (q >> 1)) ^ fr) * 16 + 8 * (q & 1));
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" :: "r"(box + (uint32_t)fr * 256u + off), "f"(acc[4 * j]), "f"(acc[4 * j + 1]) : "memory");
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" :: "r"(box + (uint32_t)(fr + 8) * 256u + off), "f"(acc[4 * j + 2]), "f"(acc[4 * j + 3]) : "memory");
            }
            __syncwarp();
            if (own) {
              float v[64];
#pragma unroll
              for (int k = 0; k < 16; ++k)
                asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[4 * k]), "=f"(v[4 * k + 1]), "=f"(v[4 * k + 2]), "=f"(v[4 * k + 3])
                             : "r"(box + (uint32_t)lane * 256u + (uint32_t)((k ^ (lane & 7)) * 16)) : "memory");
              if constexpr (ACTT) {
                epi.apply_act(orow, col0, v, 64);
              } else if (prefetch_resid) {
                float r[64];
                epi.load_resid(orow, col0, r);
                epi.fuse_resid(col0, v, r);
                epi.store_f32(orow, col0, v);
              } else {
                epi.template apply<true>(orow, col0, v, 64);
              }
            }
          }
        }
      }
    }
  }

  if (TILES && warp >= 4 && lane == 0) bulk_wait0();   // every pushed tile has landed before the CTA (and its shared memory) goes away
  __syncthreads();
}

}  // namespace mmg

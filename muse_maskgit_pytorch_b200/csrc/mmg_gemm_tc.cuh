// wgmma / TMA GEMM for sm_90a:  C[M,N] = A[M,K] * W[N,K]^T, bf16 operands, fp32 accumulation in registers.
//
//   warp 0      : TMA producer  (one elected lane) — A tile 128x64 and W tile BNx64 per k-block, SWIZZLE_128B, STAGES-deep ring
//   warps 4..11 : two consumer warpgroups.  Warpgroup g multiplies rows [64 g, 64 g + 64) of the tile (wgmma m64nBNk16, 4 per k-block,
//                 accumulators in registers), then runs the fused Epilogue on those rows: the accumulators go through a shared-memory
//                 staging buffer (128 columns at a time) so that one thread owns one output row, 64 columns per chunk; two warps share a
//                 32-row quarter and take alternate 64-column chunks.  Results leave directly, or through a per-warp shared-memory tile and
//                 a TMA store / TMA reduction (EPI_MODE below).  setmaxnreg moves registers from warpgroup 0 (40/thread) to the consumers
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
constexpr int TC_STG_LD = 132;           // staging row stride (floats): 128 columns + 4, conflict-free 16-byte row reads
constexpr int TC_SMEM_LIMIT = 227 * 1024;

// How the epilogue's results leave the CTA (the EPI_MODE of tc_gemm_kernel; described above the kernel).  The launcher picks one per product.
enum TcEpiMode : int {
  TC_EPI_REGS = 0,      // from registers, one thread per row
  TC_EPI_REDUCE = 2,    // in-place residual: per-warp tiles + TMA reduction
  TC_EPI_TSTORE = 3,    // plain fp32: per-warp tiles + TMA store
  TC_EPI_QKV = 4,       // QKV heads: per-warp tiles + TMA stores
  TC_EPI_GEGLU = 5,     // GEGLU, BN = 256: per-warp tiles + TMA store
};

struct alignas(64) TcGemmParams {
  CUtensorMap tma_a[4];
  CUtensorMap tma_b;
  CUtensorMap tma_out;      // REDUCE / TSTORE: the fp32 output [M, N] in boxes of 32 rows x 32 columns (128 B), SWIZZLE_128B; GEGLU: bf16 [M, N/2], 32 x 64
  CUtensorMap tma_qkv[3];   // QKV: q / k / v as [rows, 64] bf16 matrices in boxes of 32 rows x 64 columns (128 B)
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
};

// Shared memory: [<= 1 KB to align][operand ring][barriers, 1 KB][per-warp output tiles, 32 KB (tile epilogues only)][staging, 2 x 64 x 132 fp32]
template <int BN> struct TcCfg {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STG_BYTES = 2 * 64 * TC_STG_LD * 4;
  static constexpr int TILE_BYTES = TC_EPI_WARPS * 4096;
  static constexpr int stages(int extra) {
    return (TC_SMEM_LIMIT - 1024 - 1024 - STG_BYTES - extra) / STAGE_BYTES < 6 ? (TC_SMEM_LIMIT - 1024 - 1024 - STG_BYTES - extra) / STAGE_BYTES : 6;
  }
  static constexpr int STAGES = stages(0);
  static constexpr int STAGES_RED = stages(TILE_BYTES);
  static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 1024 + STG_BYTES;
  static constexpr int SMEM_BYTES_RED = 1024 + STAGES_RED * STAGE_BYTES + 1024 + TILE_BYTES + STG_BYTES;
  static_assert(STAGES >= 2 && STAGES_RED >= 2, "operand ring too shallow");
};

// One thread owns one output ROW, so a direct 32-byte store / load touches 32 different 128-byte lines per instruction, and the L1
// retires such row-strided accesses slowly.  The fp32 epilogues therefore leave through shared memory and the TMA engine instead:
// TC_EPI_REDUCE: in-place residual epilogues (out == resid, fp32) write the term they add into a per-warp
// 32 x 32 tile and push it with ONE TMA reduction (cp.reduce.async.bulk.tensor .add): the residual is never read, the adds happen
// in L2, and the L1 sees 8 conflict-free shared-memory stores per thread instead of 16 row-strided global accesses.
// TC_EPI_TSTORE: plain fp32 outputs (no bias / activation; the logits GEMM) leave through the same tiles with a TMA store.
// TC_EPI_QKV: the QKV epilogue (bf16; tokens % 32 == 0 and M % 128 == 0, so a warp's 32 rows are 32 consecutive tokens of one
// sequence and land on 32 consecutive rows of one head of q / k / v): head chunk -> tile -> one TMA store per warp and chunk.
// TC_EPI_GEGLU: the GEGLU epilogue (bf16 out, BN == 256): the two warps of a lane quarter take ADJACENT chunk pairs (0,1 | 2,3), so a
// warp's 2 x 32 outputs per row are 128 contiguous bytes -> one 32-row x 128-byte tile -> one TMA store per warp and tile.
template <int BN, int EPI_MODE>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ TcGemmParams p) {
  using namespace sm90;
  using Cfg = TcCfg<BN>;
  constexpr bool RED = EPI_MODE == TC_EPI_REDUCE || EPI_MODE == TC_EPI_TSTORE, RED_ADD = EPI_MODE == TC_EPI_REDUCE;   // TSTORE: same tiles, plain TMA store
  constexpr bool QKVT = EPI_MODE == TC_EPI_QKV;
  constexpr bool GEGLUT = EPI_MODE == TC_EPI_GEGLU;
  constexpr bool TILES = EPI_MODE != TC_EPI_REGS;
  static_assert(!GEGLUT || BN == 256, "the GEGLU tile epilogue pairs adjacent 64-column chunks of a 256-column tile");
  constexpr int STAGES = TILES ? Cfg::STAGES_RED : Cfg::STAGES;
  constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;
  constexpr int ROUNDS = (BN + 127) / 128;
  // residual rows are fetched one chunk ahead (the first one during the main loop) only at BN <= 128: at BN = 256 the 128 accumulator
  // registers leave no room for a 64-register residual buffer next to them, so each chunk loads its residual when it needs it
  constexpr bool EARLY_RESID = BN <= 128;

  if (p.skip_if_zero) { pdl_wait(); if (*p.skip_if_zero == 0) return; }       // uniform over the grid: nothing has been set up yet

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint8_t* tiles = smem + STAGES * STAGE_BYTES + 1024;
  float* staging = reinterpret_cast<float*>(tiles + (TILES ? Cfg::TILE_BYTES : 0));

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
            tma_load_2d(sa, &p.tma_a[0], full_bar + stage, kb * TC_BK, m_blk * TC_BM);
          } else {
            const int tap = kb / p.cchunks, cc = kb - tap * p.cchunks;
            tma_load_4d(sa, &p.tma_a[p.tap_map[tap]], full_bar + stage, cc * TC_BK, x0 + p.tap_dx[tap], y0 + p.tap_dy[tap], b0);
          }
          tma_load_2d(sb, &p.tma_b, full_bar + stage, kb * TC_BK, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===================== consumer warpgroups: wgmma main loop, then the epilogue of their 64 rows =====================
    const int wg = (warp - 4) >> 2, wq = warp & 3;
    const int quarter = 2 * wg + (wq & 1);        // this warp's 32 rows of the tile, inside its warpgroup's 64
    const int half = wq >> 1;                     // 0: even 64-column chunks, 1: odd chunks
    const int r_in_tile = quarter * 32 + lane;
    float* stg = staging + wg * 64 * TC_STG_LD;
    const float* my_row = stg + ((wq & 1) * 32 + lane) * TC_STG_LD;
    Epilogue epi = p.epi;
    if (epi.kind == MMG_EPI_QKV) { epi.p.q_scale = s_scale; epi.p.k_scale = s_scale + 64; }
    const bool whole_row = (epi.kind == MMG_EPI_CONVT_RGB);      // needs every chunk of a row in one thread
    const bool prefetch_resid = epi.can_prefetch_resid();
    int stage = 0; uint32_t phase = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
      const int m_blk = p.n_fast ? tile / p.num_n_tiles : tile % p.num_m_tiles, n_blk = p.n_fast ? tile % p.num_n_tiles : tile / p.num_m_tiles;
      int64_t row; bool valid;
      if (p.mode == 0) {
        row = (int64_t)m_blk * TC_BM + r_in_tile; valid = row < p.M;
      } else {
        const int xt = m_blk % p.tiles_x, yt = (m_blk / p.tiles_x) % p.tiles_y, bt = m_blk / (p.tiles_x * p.tiles_y);
        const int tx = r_in_tile % p.TW, ty = (r_in_tile / p.TW) % p.TH, tb = r_in_tile / (p.TW * p.TH);
        const int b = bt * p.TB + tb;
        valid = b < p.B;
        row = ((int64_t)b * p.Ho + (yt * p.TH + ty)) * p.Wo + xt * p.TW + tx;
      }
      const bool mine = !whole_row || half == 0;
      const int c_first = GEGLUT ? 2 * half : whole_row ? 0 : half, c_step = (GEGLUT || whole_row) ? 1 : 2;
      const int c_end = GEGLUT ? c_first + 2 : BN / 64;
      const bool pre = EARLY_RESID && !RED && prefetch_resid && valid && mine && (n_blk * BN + c_first * 64 < p.N) && c_first < BN / 64;
      float rbuf[64];
      if (pre) epi.load_resid(row, n_blk * BN + c_first * 64, rbuf);      // in flight during the main loop
      if (valid && mine) epi.begin_row(row);                               // row geometry / folded-LayerNorm statistics: independent of the accumulator

      // ---- main loop: 4 wgmma (K = 16) per k-block; a ring slot goes back to the producer once the wgmma group after it was issued ----
      int prev_stage = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(full_bar + stage, phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        const uint64_t adesc = smem_desc_kmajor_sw128(sa + (uint32_t)wg * 8192u);
        const uint64_t bdesc = smem_desc_kmajor_sw128(sa + Cfg::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k)
          Wgmma<BN>::template mma<0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev_stage >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + prev_stage); }
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (prev_stage >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + prev_stage); }

      // the epilogue of one 64-column accumulator chunk held in v
      auto chunk = [&](const int c, float (&v)[64]) {
        const int col0 = n_blk * BN + c * 64;
        if (GEGLUT) {
          // columns past N are zero accumulators (TMA zero-fills the missing W rows) and are clipped by the tensor map, rows past M too
          float o[32];
          epi.template geglu_chunk<true>(v, o, row, col0, valid && col0 < p.N);
          const uint32_t wtile = smem_u32(tiles) + (uint32_t)(warp - 4) * 4096u;
          const int cc = c - c_first;                       // 0 / 1: left / right 64 bytes of the warp's 128-byte rows
          if (cc == 0) { if (lane == 0) bulk_wait_read0(); __syncwarp(); }     // this warp's previous store has left the tile
#pragma unroll
          for (int j = 0; j < 4; ++j)
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" :: "r"(wtile + (uint32_t)lane * 128u + (uint32_t)(((cc * 4 + j) ^ (lane & 7)) * 16)),
                         "r"(pack_bf16(o[8 * j], o[8 * j + 1])), "r"(pack_bf16(o[8 * j + 2], o[8 * j + 3])),
                         "r"(pack_bf16(o[8 * j + 4], o[8 * j + 5])), "r"(pack_bf16(o[8 * j + 6], o[8 * j + 7])) : "memory");
          if (cc == 1) {
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) { tma_store_2d(&p.tma_out, wtile, (n_blk * BN + c_first * 64) >> 1, m_blk * TC_BM + quarter * 32); bulk_commit(); }
          }
        } else if (QKVT && col0 < p.N) {
          int h;
          const int which = epi.template qkv_chunk<true>(col0, v, h);
          const uint32_t wtile = smem_u32(tiles) + (uint32_t)(warp - 4) * 4096u;
          const uint32_t rw = (uint32_t)(m_blk * TC_BM + quarter * 32), tok = (uint32_t)epi.p.tokens;
          const uint32_t bq = rw / tok, t0 = rw - bq * tok;                       // warp-uniform: the 32 rows are tokens t0 .. t0+31 of sequence bq
          const int64_t drow = which == 0 ? ((int64_t)bq * epi.p.heads + h) * epi.p.q_rows + t0
                                          : ((int64_t)bq * epi.p.heads + h) * epi.p.kv_rows + epi.p.key_off + t0;
          if (lane == 0) bulk_wait_read0();          // the store that last used this tile has read it
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 8; ++j)
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" :: "r"(wtile + (uint32_t)lane * 128u + (uint32_t)((j ^ (lane & 7)) * 16)),
                         "r"(pack_bf16(v[8 * j], v[8 * j + 1])), "r"(pack_bf16(v[8 * j + 2], v[8 * j + 3])),
                         "r"(pack_bf16(v[8 * j + 4], v[8 * j + 5])), "r"(pack_bf16(v[8 * j + 6], v[8 * j + 7])) : "memory");
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) { tma_store_2d(&p.tma_qkv[which], wtile, 0, (int)drow); bulk_commit(); }
          if (which != 0 && t0 == 0 && lane == 0) epi.qkv_null_row(which, bq, h);
        } else if (RED && col0 < p.N) {
          // rows past M hold garbage here and are clipped by the tensor map; the tile layout is the TMA 128-byte swizzle
          if (RED_ADD) epi.resid_term(col0, v);
          const uint32_t wtile = smem_u32(tiles) + (uint32_t)(warp - 4) * 4096u;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (lane == 0) bulk_wait_read0();             // this warp's previous push has left the tile
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 8; ++j)
              asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" :: "r"(wtile + (uint32_t)lane * 128u + (uint32_t)((j ^ (lane & 7)) * 16)),
                           "f"(v[32 * h + 4 * j]), "f"(v[32 * h + 4 * j + 1]), "f"(v[32 * h + 4 * j + 2]), "f"(v[32 * h + 4 * j + 3]) : "memory");
            fence_proxy_async();                          // generic-proxy writes -> visible to the TMA (async-proxy) read
            __syncwarp();
            if (lane == 0) {
              if (RED_ADD) tma_reduce_add_2d(&p.tma_out, wtile, col0 + 32 * h, m_blk * TC_BM + quarter * 32);
              else tma_store_2d(&p.tma_out, wtile, col0 + 32 * h, m_blk * TC_BM + quarter * 32);
              bulk_commit();
            }
          }
        } else if (valid && col0 < p.N) {
          if (prefetch_resid) {
            if (!EARLY_RESID) epi.load_resid(row, col0, rbuf);
            epi.fuse_resid(col0, v, rbuf);
            const int cn = col0 + c_step * 64;
            if (EARLY_RESID && c + c_step < BN / 64 && cn < p.N) epi.load_resid(row, cn, rbuf);   // next chunk's residual overlaps the stores
            epi.store_f32(row, col0, v);
          } else {
            epi.template apply<true>(row, col0, v, 64);
          }
        }
      };
#pragma unroll
      for (int rd = 0; rd < ROUNDS; ++rd) {
        // columns [128 rd, 128 rd + 128) of the warpgroup's 64 rows -> staging -> one row per thread
        named_sync(1 + wg, 128);                   // the previous round's (tile's) readers are done with the staging buffer
        stage_acc<BN / 2, TC_STG_LD>(acc, stg, 128 * rd, BN - 128 * rd < 128 ? BN - 128 * rd : 128);
        named_sync(1 + wg, 128);
#pragma unroll 1
        for (int c = c_first; c < c_end; c += c_step) {
          if (!mine) break;
          if ((c >> 1) != rd) continue;
          float v[64];
          stage_ld32(my_row + (c & 1) * 64, v);
          stage_ld32(my_row + (c & 1) * 64 + 32, v + 32);
          chunk(c, v);
        }
      }
      if (valid && mine) epi.end_row(row);
    }
  }

  if (TILES && warp >= 4 && lane == 0) bulk_wait0();   // every pushed tile has landed before the CTA (and its shared memory) goes away
  __syncthreads();
}

}  // namespace mmg

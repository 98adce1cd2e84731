// mmg_linear / mmg_conv2d / mmg_conv_transpose2d and their e4m3 forms: launchers for the wgmma GEMM (bf16 / e4m3) and the fp32
// CUDA-core GEMM.
#include "mmg_gemm_tc.cuh"
#include "mmg_tmap.cuh"
#include <mutex>

namespace mmg {

int linear_impl(const mmg_linear_args* a, const int* skip_if_zero, void* stream);

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

// persistent grid of min(tiles, #SM) CTAs
template <int BN, int EPI_MODE, typename TA = bf16>
static int launch_tc(const TcGemmParams& p, cudaStream_t st) {
  constexpr int smem = TcCfg<BN>::SMEM_BYTES;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] { attr_err = cudaFuncSetAttribute(tc_gemm_kernel<BN, EPI_MODE, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
  if (attr_err != cudaSuccess) return fail(MMG_ECUDA, "cudaFuncSetAttribute(tc_gemm<%d, %d>): %s", BN, EPI_MODE, cudaGetErrorString(attr_err));
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  MMG_CUDA(launch_pdl(tc_gemm_kernel<BN, EPI_MODE, TA>, dim3(grid), dim3(TC_THREADS), smem, st, p));
  MMG_LAUNCHED();
  return MMG_OK;
}

// every instantiation of tc_gemm_kernel: 17 with bf16 operands, 8 with e4m3 ones
static constexpr int tc_key(bool fp8, int bn, int mode) { return (fp8 ? 1 << 16 : 0) | bn << 4 | mode; }

static int launch_instantiation(bool fp8, int bn, int mode, const TcGemmParams& p, cudaStream_t st) {
  if (bn != 64 && bn != 128 && bn != 256) return fail(MMG_EINVAL, "unsupported tile width %d", bn);
  switch (tc_key(fp8, bn, mode)) {
    case tc_key(false, 64, TC_EPI_REGS): return launch_tc<64, TC_EPI_REGS>(p, st);
    case tc_key(false, 128, TC_EPI_REGS): return launch_tc<128, TC_EPI_REGS>(p, st);
    case tc_key(false, 256, TC_EPI_REGS): return launch_tc<256, TC_EPI_REGS>(p, st);          // CONVT_RGB only
    case tc_key(false, 64, TC_EPI_REDUCE): return launch_tc<64, TC_EPI_REDUCE>(p, st);
    case tc_key(false, 128, TC_EPI_REDUCE): return launch_tc<128, TC_EPI_REDUCE>(p, st);
    case tc_key(false, 256, TC_EPI_REDUCE): return launch_tc<256, TC_EPI_REDUCE>(p, st);
    case tc_key(false, 128, TC_EPI_TSTORE): return launch_tc<128, TC_EPI_TSTORE>(p, st);      // the sample GEMM of the fused tail at small batch
    case tc_key(false, 256, TC_EPI_TSTORE): return launch_tc<256, TC_EPI_TSTORE>(p, st);
    case tc_key(false, 128, TC_EPI_QKV): return launch_tc<128, TC_EPI_QKV>(p, st);
    case tc_key(false, 256, TC_EPI_QKV): return launch_tc<256, TC_EPI_QKV>(p, st);
    case tc_key(false, 256, TC_EPI_GEGLU): return launch_tc<256, TC_EPI_GEGLU>(p, st);
    case tc_key(false, 128, TC_EPI_ACT): return launch_tc<128, TC_EPI_ACT>(p, st);
    case tc_key(false, 128, TC_EPI_QKV128): return launch_tc<128, TC_EPI_QKV128>(p, st);
    case tc_key(false, 256, TC_EPI_QKV128): return launch_tc<256, TC_EPI_QKV128>(p, st);
    case tc_key(false, 128, TC_EPI_QKV128_REGS): return launch_tc<128, TC_EPI_QKV128_REGS>(p, st);
    case tc_key(false, 256, TC_EPI_GLU): return launch_tc<256, TC_EPI_GLU>(p, st);
    case tc_key(false, 256, TC_EPI_CONVT): return launch_tc<256, TC_EPI_CONVT>(p, st);
    case tc_key(true, 64, TC_EPI_REGS): return launch_tc<64, TC_EPI_REGS, fp8e4>(p, st);
    case tc_key(true, 128, TC_EPI_REGS): return launch_tc<128, TC_EPI_REGS, fp8e4>(p, st);
    case tc_key(true, 256, TC_EPI_REGS): return launch_tc<256, TC_EPI_REGS, fp8e4>(p, st);  // CONVT_RGB only
    case tc_key(true, 128, TC_EPI_QKV): return launch_tc<128, TC_EPI_QKV, fp8e4>(p, st);
    case tc_key(true, 256, TC_EPI_QKV): return launch_tc<256, TC_EPI_QKV, fp8e4>(p, st);
    case tc_key(true, 256, TC_EPI_GEGLU): return launch_tc<256, TC_EPI_GEGLU, fp8e4>(p, st);
    case tc_key(true, 128, TC_EPI_QKV128): return launch_tc<128, TC_EPI_QKV128, fp8e4>(p, st);
    case tc_key(true, 256, TC_EPI_QKV128): return launch_tc<256, TC_EPI_QKV128, fp8e4>(p, st);
  }
  return fail(MMG_EINVAL, "no tc_gemm_kernel<%d, %d> instantiation for %s operands", bn, mode, fp8 ? "e4m3" : "bf16");
}

static int pick_bn(int64_t M_tiles, int64_t N, int epilogue) {
  if (epilogue == MMG_EPI_CONVT_RGB) return (int)N;             // whole row in one tile
  if (N % 256 == 0 && M_tiles * (N / 256) >= 2 * num_sms()) return 256;
  if (N % 128 == 0 && M_tiles * (N / 128) >= num_sms()) return 128;
  if (N % 128 == 0 && N >= 1024) return 128;
  return (N % 64 == 0 && N % 128 != 0) ? 64 : ((M_tiles * ((N + 127) / 128) >= 96) ? 128 : 64);
}

// The tile plan of every wgmma GEMM launch: (BN, EPI_MODE) from the operand type and p's geometry (mode, M, num_m_tiles) and epilogue.
static int plan_tc(const TcGemmParams& p, bool fp8, int* bn_out, int* mode_out) {
  const mmg_epilogue_args& e = p.epi.p;
  const int kind = p.epi.kind;
  MMG_CHECK_ARG(kind != MMG_EPI_QKV128 || p.mode == 0, "QKV128: dense products only");
  int bn = pick_bn(p.num_m_tiles, p.N, kind), mode;
  const bool in_place = (kind == MMG_EPI_LNFOLD_RESIDUAL || (kind == MMG_EPI_RESIDUAL && e.act == 0)) && e.out_dtype == MMG_F32 &&
                        e.out == e.resid && e.ldo == e.ldr && (e.ldo % 4) == 0 && aligned16(e.out) && p.mode == 0;
  const bool plain_f32 = kind == MMG_EPI_STORE && e.out_dtype == MMG_F32 && p.mode == 0 && !e.bias && e.act == 0 && (e.ldo % 4) == 0 && aligned16(e.out);
  // QKV / QKV128 tile epilogue: bf16 heads, whole 16-token boxes of one sequence
  const bool qkv_tiles = (kind == MMG_EPI_QKV || kind == MMG_EPI_QKV128) && e.out_dtype == MMG_BF16 && p.mode == 0 && e.tokens % 32 == 0 &&
                         p.M % 128 == 0 && e.nk_heads == e.nv_heads && (!e.nq_heads || aligned16(e.q_out)) &&
                         (!e.nk_heads || (aligned16(e.k_out) && aligned16(e.v_out)));
  const bool geglu_tiles = kind == MMG_EPI_GEGLU && e.out_dtype == MMG_BF16 && p.mode == 0 && (e.ldo % 8) == 0 && aligned16(e.out);
  // GLU / CONVT tile epilogues (the VAE decoder's long-K products): bf16 operands and output, conv mode, whole 256-column tiles.  CONVT
  // also needs the launch's geometry in its epilogue (H, W) to be the grid's, W % 16 == 0 (a warp's 16 rows in one input row) and its
  // output rows (b H + y) 2 W + x inside int32
  const bool conv_tiles = !fp8 && p.mode == 1 && e.out_dtype == MMG_BF16 && (e.ldo % 8) == 0 && aligned16(e.out) && p.N % 256 == 0;
  const bool glu_tiles = conv_tiles && kind == MMG_EPI_GLU;
  const bool convt_tiles = conv_tiles && kind == MMG_EPI_CONVT && e.H == p.Ho && e.W == p.Wo && p.Wo % 16 == 0 && 2 * p.M < INT32_MAX;
  // A dense e4m3 product has no register-epilogue instantiation: its argument checks leave it only the shapes its tile epilogue takes, and
  // it runs that epilogue at every M: QKV at 128 where pick_bn gives 64 (where the bf16 product takes <64, REGS>), GEGLU at 256 whatever
  // pick_bn gives.  QKV128 (whole 128-column heads) runs its tile epilogue at 128 or 256 for either operand type.
  const bool tile_at_any_bn = fp8 && p.mode == 0;
  if (p.epi.is_act()) {
    mode = TC_EPI_ACT; bn = 128;              // the T5 feed-forward epilogues: an instantiation of their own, kept out of the VAE's
  } else if (in_place) {
    mode = TC_EPI_REDUCE;
  } else if (plain_f32 && bn >= 128) {
    mode = TC_EPI_TSTORE;
  } else if (qkv_tiles && (bn != 64 || tile_at_any_bn || kind == MMG_EPI_QKV128)) {
    mode = kind == MMG_EPI_QKV ? TC_EPI_QKV : TC_EPI_QKV128; bn = bn == 256 ? 256 : 128;
  } else if (kind == MMG_EPI_QKV128) {
    mode = TC_EPI_QKV128_REGS; bn = 128;      // 64 accumulators per thread, stored from the fragments
  } else if (geglu_tiles && (bn == 256 || tile_at_any_bn)) {
    mode = TC_EPI_GEGLU; bn = 256;
  } else if ((glu_tiles || convt_tiles) && bn == 256) {
    mode = glu_tiles ? TC_EPI_GLU : TC_EPI_CONVT;
  } else {
    // 128 accumulator registers per thread at BN = 256 next to a 64-column row chunk would spill, so <256, TC_EPI_REGS> compiles only
    // the fused RGB epilogue, which reduces the fragments in place; every other register-epilogue kind runs at BN <= 128 (GLU and
    // CONVT where pick_bn gives 256 and the conditions above hold take their tile epilogues instead)
    mode = TC_EPI_REGS;
    if (bn == 256 && kind != MMG_EPI_CONVT_RGB) bn = 128;
  }
  // the tile epilogues write whole 32- / 64-column boxes: pick_bn's widths divide N (N % 64 == 0 on this path)
  MMG_CHECK_ARG(!tc_tile_epilogue(mode) || p.N % bn == 0, "tile epilogue: tile width %d does not divide N = %lld", bn, (long long)p.N);
  *bn_out = bn; *mode_out = mode;
  return MMG_OK;
}

// the output tensor maps of the tile epilogues: q / k / v heads (QKV, QKV128), bf16 [M, N / 2] (GEGLU, GLU), fp32 [M, N] (REDUCE,
// TSTORE), bf16 pixels of one conv-transpose parity (CONVT)
static int tile_out_maps(TcGemmParams& p, int mode) {
  const mmg_epilogue_args& e = p.epi.p;
  int rc = MMG_OK;
  if (mode == TC_EPI_CONVT) {
    // out is [B, 2H, 2W, ldo]: pixel (b, 2 y + py, 2 x + px) sits (b H + y) 4 W ldo + 2 x ldo elements past pixel (0, py, px), so from
    // there the parity's pixels are rows (b H + y) 2 W + x of 2 ldo elements; the last one is row (B H - 1) 2 W + W - 1
    const uint64_t W = (uint64_t)p.Wo, BH = (uint64_t)(p.M / p.Wo);
    const bf16* base = reinterpret_cast<const bf16*>(e.out) + (uint64_t)(e.py * 2 * W + e.px) * e.ldo;
    uint64_t od[2] = {(uint64_t)p.N, BH * 2 * W - W}; uint64_t os[1] = {(uint64_t)e.ldo * 4}; uint32_t ob[2] = {64, 16};
    return make_tmap_bf16(&p.tma_out, base, 2, od, os, ob);
  }
  if (mode == TC_EPI_QKV || mode == TC_EPI_QKV128) {
    const uint64_t seqs = (uint64_t)(p.M / e.tokens) * (uint64_t)e.heads, hd = mode == TC_EPI_QKV ? 64 : 128;
    uint64_t str[1] = {hd * 2}; uint32_t box[2] = {64, 16};
    if (e.nq_heads) { uint64_t d[2] = {hd, seqs * (uint64_t)e.q_rows}; rc = make_tmap_bf16(&p.tma_qkv[0], e.q_out, 2, d, str, box); if (rc) return rc; }
    if (e.nk_heads) {
      uint64_t d[2] = {hd, seqs * (uint64_t)e.kv_rows};
      rc = make_tmap_bf16(&p.tma_qkv[1], e.k_out, 2, d, str, box); if (rc) return rc;
      rc = make_tmap_bf16(&p.tma_qkv[2], e.v_out, 2, d, str, box); if (rc) return rc;
    }
  } else if (mode == TC_EPI_GEGLU || mode == TC_EPI_GLU) {
    uint64_t od[2] = {(uint64_t)(p.N / 2), (uint64_t)p.M}; uint64_t os[1] = {(uint64_t)e.ldo * 2}; uint32_t ob[2] = {64, 16};
    rc = make_tmap_bf16(&p.tma_out, e.out, 2, od, os, ob);
  } else if (mode == TC_EPI_REDUCE || mode == TC_EPI_TSTORE) {
    uint64_t od[2] = {(uint64_t)p.N, (uint64_t)p.M}; uint64_t os[1] = {(uint64_t)e.ldo * 4}; uint32_t ob[2] = {32, 16};
    rc = make_tmap_f32(&p.tma_out, e.out, 2, od, os, ob);
  }
  return rc;
}

// an operand tensor map of the wgmma GEMM: bf16, or e4m3 moved as bytes
static int operand_map(CUtensorMap* m, bool fp8, const void* base, int rank, const uint64_t* dims, const uint64_t* strides, const uint32_t* box) {
  return fp8 ? make_tmap_u8(m, base, rank, dims, strides, box) : make_tmap_bf16(m, base, rank, dims, strides, box);
}

// Plans and launches one wgmma GEMM whose A operand map(s), geometry and epilogue p already holds.  w: the [N, K] weights, rows ldw
// elements apart; a k-block is 128 bytes of them.
static int dispatch_tc(TcGemmParams& p, bool fp8, const void* w, int64_t K, int64_t ldw, cudaStream_t st) {
  int bn, mode;
  int rc = plan_tc(p, fp8, &bn, &mode); if (rc) return rc;
  const uint64_t esz = fp8 ? 1 : 2;
  p.num_n_tiles = (int)((p.N + bn - 1) / bn);
  // N-fastest while the weights (counted at 2 bytes an element for either operand type) fit 8 MiB in 2..16 column tiles
  p.n_fast = ((int64_t)p.N * K * 2 <= (8 << 20) && p.num_n_tiles > 1 && p.num_n_tiles <= 16) ? 1 : 0;
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)p.N}; uint64_t str[1] = {(uint64_t)ldw * esz}; uint32_t box[2] = {(uint32_t)(128 / esz), (uint32_t)bn};
  rc = operand_map(&p.tma_b, fp8, w, 2, dims, str, box); if (rc) return rc;
  rc = tile_out_maps(p, mode); if (rc) return rc;
  return launch_instantiation(fp8, bn, mode, p, st);
}

// ------------------------------------------------------------------------------------------------------------------
// fp32-accumulate CUDA-core GEMM (parity precision, and shapes the TMA path does not take).  64x64x16 tiles,
// 256 threads, 4x4 micro-tile per thread; A is addressed through a loader (dense or implicit conv).
// ------------------------------------------------------------------------------------------------------------------
struct ConvGeom {
  int B, H, W, Cin, Ho, Wo, stride, ntaps;
  int8_t tdy[25], tdx[25];
};

template <typename T, bool CONV, bool ACT>
__global__ void __launch_bounds__(256)
simt_gemm_kernel(const T* __restrict__ A, const T* __restrict__ Wt, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldw,
                 ConvGeom g, Epilogue epi) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  __shared__ float Cs[64][64 + 1];
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * 64;
  const int n0 = blockIdx.y * 64;
  const int tx = tid & 15, ty = tid >> 4;
  float acc[4][4] = {};
  // loader mapping: each thread loads 4 elements of A and of W per k-step: row = tid/4 (0..63), k = (tid%4)*4 .. +3
  const int lr = tid >> 2, lk = (tid & 3) * 4;
  const int64_t am = m0 + lr;
  int ab = 0, ay = 0, ax = 0;
  if (CONV && am < M) { ab = (int)(am / ((int64_t)g.Ho * g.Wo)); int rem = (int)(am - (int64_t)ab * g.Ho * g.Wo); ay = rem / g.Wo; ax = rem - ay * g.Wo; }
  for (int64_t k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t k = k0 + lk + j;
      float av = 0.f, bv = 0.f;
      if (am < M && k < K) {
        if (!CONV) av = to_f(A[am * lda + k]);
        else {
          const int tap = (int)(k / g.Cin), c = (int)(k - (int64_t)tap * g.Cin);
          const int iy = ay * g.stride + g.tdy[tap], ix = ax * g.stride + g.tdx[tap];
          if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) av = to_f(A[(((int64_t)ab * g.H + iy) * g.W + ix) * g.Cin + c]);
        }
      }
      if (n0 + lr < N && k < K) bv = to_f(Wt[(int64_t)(n0 + lr) * ldw + k]);
      As[lk + j][lr] = av; Bs[lk + j][lr] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) Cs[ty * 4 + i][tx * 4 + j] = acc[i][j];
  __syncthreads();
  if (tid < 64) {
    const int64_t row = m0 + tid;
    if (row < M) {
      float v[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) v[i] = Cs[tid][i];
      int nvalid = (int)(N - n0); if (nvalid > 64) nvalid = 64;
      // CONVT_RGB needs the whole row in one pass and is not offered on this path (validated by the launcher)
      if (ACT) {                                  // the T5 feed-forward epilogues (GEGLU_TANH, STORE + ReLU): an instantiation of their own
        epi.apply_act(row, n0, v, nvalid);
      } else {
        epi.begin_row(row);
        epi.template apply<false>(row, n0, v, nvalid);
      }
    }
  }
}

template <bool CONV>
static int launch_simt(int dtype, const void* a, const void* w, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldw,
                       const ConvGeom& g, const Epilogue& epi, cudaStream_t st) {
  MMG_CHECK_ARG(epi.kind != MMG_EPI_CONVT_RGB, "CONVT_RGB epilogue requires the bf16 tensor-core path");
  MMG_CHECK_ARG(epi.kind != MMG_EPI_QKV128, "QKV128 epilogue requires the wgmma path of mmg_linear");
  MMG_CHECK_ARG(M > 0 && N > 0 && K > 0, "empty GEMM");
  dim3 grid((unsigned)((M + 63) / 64), (unsigned)((N + 63) / 64));
  MMG_CHECK_ARG(grid.y < 65536, "N too large for the fp32 path");
  if (!CONV && epi.is_act()) {
    if (dtype == MMG_F32) simt_gemm_kernel<float, false, true><<<grid, 256, 0, st>>>((const float*)a, (const float*)w, M, N, K, lda, ldw, g, epi);
    else simt_gemm_kernel<bf16, false, true><<<grid, 256, 0, st>>>((const bf16*)a, (const bf16*)w, M, N, K, lda, ldw, g, epi);
  } else if (dtype == MMG_F32) simt_gemm_kernel<float, CONV, false><<<grid, 256, 0, st>>>((const float*)a, (const float*)w, M, N, K, lda, ldw, g, epi);
  else simt_gemm_kernel<bf16, CONV, false><<<grid, 256, 0, st>>>((const bf16*)a, (const bf16*)w, M, N, K, lda, ldw, g, epi);
  simt_launch_counter()++;
  MMG_LAUNCHED();
  return MMG_OK;
}


// conv tap tables.  kind 0: 1x1; 1: 3x3 s1 p1; 2: 4x4 s2 p1; 3: 5x5 s1 p2.  Tap index t = r*kw + s (weights packed tap-major).
// CONVT_PARITY + py * 2 + px: conv-transpose (k4 s2 p1) parity class (py, px) over the input grid: 2x2 taps, tap t = a*2+b at input
// offset (CT_D[py][a], CT_D[px][b]).
constexpr int CONVT_PARITY = 4;
static const int CT_D[2][2] = {{0, -1}, {1, 0}};

static void conv_geom(int kind, int B, int H, int W, int Cin, ConvGeom* g) {
  g->B = B; g->H = H; g->W = W; g->Cin = Cin;
  if (kind >= CONVT_PARITY) {
    const int py = (kind - CONVT_PARITY) >> 1, px = (kind - CONVT_PARITY) & 1;
    g->stride = 1; g->Ho = H; g->Wo = W; g->ntaps = 4;
    for (int t = 0; t < 4; ++t) { g->tdy[t] = (int8_t)CT_D[py][t >> 1]; g->tdx[t] = (int8_t)CT_D[px][t & 1]; }
    return;
  }
  const int k = kind == 0 ? 1 : kind == 1 ? 3 : kind == 2 ? 4 : 5;
  const int pad = kind == 0 ? 0 : kind == 1 ? 1 : kind == 2 ? 1 : 2;
  g->stride = (kind == 2) ? 2 : 1;
  g->Ho = H / g->stride; g->Wo = W / g->stride; g->ntaps = k * k;
  for (int r = 0; r < k; ++r) for (int s = 0; s < k; ++s) { g->tdy[r * k + s] = (int8_t)(r - pad); g->tdx[r * k + s] = (int8_t)(s - pad); }
}

static int tile_geometry(int Ho, int Wo, TcGemmParams* p) {
  int TW = Wo < 128 ? Wo : 128;
  if (128 % TW != 0 || Wo % TW != 0) return -1;
  int TH = 128 / TW; if (TH > Ho) TH = Ho;
  if (Ho % TH != 0 || 128 % (TW * TH) != 0) return -1;
  p->TW = TW; p->TH = TH; p->TB = 128 / (TW * TH);
  p->tiles_x = Wo / TW; p->tiles_y = Ho / TH;
  return 0;
}

// the tap table of tc_gemm_kernel's conv mode: tap t reads A map tap_map[t] at the output pixel + (tap_dy[t], tap_dx[t]).  Stride 2:
// input row 2y + dy = 2(y + (dy - py) / 2) + py, so the tap reads the map of input parity (py, px) at the half-resolution offset.
static void conv_taps(TcGemmParams& p, const ConvGeom& g) {
  for (int t = 0; t < g.ntaps; ++t) {
    if (g.stride == 1) { p.tap_map[t] = 0; p.tap_dy[t] = g.tdy[t]; p.tap_dx[t] = g.tdx[t]; continue; }
    const int oy = g.tdy[t], ox = g.tdx[t];
    const int py = ((oy % 2) + 2) % 2, px = ((ox % 2) + 2) % 2;
    p.tap_map[t] = (int8_t)(py * 2 + px); p.tap_dy[t] = (int8_t)((oy - py) / 2); p.tap_dx[t] = (int8_t)((ox - px) / 2);
  }
}

// The implicit-GEMM operand of tc_gemm_kernel's conv mode over the NHWC image x (bf16, or e4m3 bytes) of geometry g: the problem shape,
// the tap table and the A tensor map(s), one 4-D map or, at stride 2, one per input parity (py, px) over the (H/2, W/2) grid.  A k-block
// is one tap x 128 bytes of channels.  tile_geometry() has filled p's tile fields.
static int conv_operand(TcGemmParams& p, const ConvGeom& g, const void* x, bool fp8, int64_t N) {
  const uint64_t esz = fp8 ? 1 : 2, C = g.Cin, W = g.W, H = g.H;
  p.M = (int64_t)g.B * g.Ho * g.Wo; p.N = N; p.mode = 1; p.cchunks = (int)(C * esz / 128); p.ntaps = g.ntaps; p.num_kb = p.ntaps * p.cchunks;
  p.Ho = g.Ho; p.Wo = g.Wo; p.B = g.B;
  p.num_m_tiles = p.tiles_x * p.tiles_y * ((g.B + p.TB - 1) / p.TB);
  conv_taps(p, g);
  uint32_t box[4] = {(uint32_t)(128 / esz), (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TB};
  if (g.stride == 1) {
    uint64_t dims[4] = {C, W, H, (uint64_t)g.B}; uint64_t str[3] = {C * esz, W * C * esz, H * W * C * esz};
    return operand_map(&p.tma_a[0], fp8, x, 4, dims, str, box);
  }
  for (int py = 0; py < 2; ++py) for (int px = 0; px < 2; ++px) {
    const uint8_t* base = reinterpret_cast<const uint8_t*>(x) + ((uint64_t)py * W + px) * C * esz;
    uint64_t dims[4] = {C, W / 2, H / 2, (uint64_t)g.B}; uint64_t str[3] = {2 * C * esz, 2 * W * C * esz, H * W * C * esz};
    const int rc = operand_map(&p.tma_a[py * 2 + px], fp8, base, 4, dims, str, box); if (rc) return rc;
  }
  return MMG_OK;
}

}  // namespace mmg

using namespace mmg;

extern "C" int mmg_linear(const mmg_linear_args* a, void* stream) { return mmg::linear_impl(a, nullptr, stream); }

// skip_if_zero: optional device word; the tensor-core kernel returns at once when it reads 0 there (the fallback leg of mmg_logits_fused)
int mmg::linear_impl(const mmg_linear_args* a, const int* skip_if_zero, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->a && a->w, "mmg_linear: NULL operand");
  MMG_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0, "mmg_linear: bad shape M=%lld N=%lld K=%lld", (long long)a->M, (long long)a->N, (long long)a->K);
  int rc = validate_epilogue(a->epilogue, a->epi, a->N); if (rc) return rc;
  Epilogue epi; epi.p = a->epi; epi.kind = a->epilogue;
  const bool tc_ok = a->dtype == MMG_BF16 && (a->K % 64 == 0) && (a->N % 64 == 0) && (a->lda % 8 == 0) && (a->ldw % 8 == 0) &&
                     aligned16(a->a) && aligned16(a->w) && (a->epi.ldo % 8 == 0 || a->epilogue == MMG_EPI_QKV || a->epilogue == MMG_EPI_QKV128 ||
                                                             a->epilogue == MMG_EPI_CONVT_RGB || a->epilogue == MMG_EPI_LFQ_IDS || a->epilogue == MMG_EPI_ARGMIN);
  // QKV128 has no CUDA-core epilogue: bf16 operands with K % 64 == 0, 8-element rows and 16-byte aligned a / w, or nothing
  MMG_CHECK_ARG(tc_ok || a->epilogue != MMG_EPI_QKV128, "mmg_linear: QKV128 needs the wgmma path (bf16, K %% 64 == 0, lda / ldw %% 8 == 0, aligned a / w)");
  if (!tc_ok) {
    MMG_CHECK_ARG(!skip_if_zero, "skippable GEMM requires the bf16 tensor-core path");
    if (a->dtype == MMG_BF16) note_simt_fallback("mmg_linear", a->M, a->N, a->K);
    ConvGeom g{};
    return launch_simt<false>(a->dtype, a->a, a->w, a->M, a->N, a->K, a->lda, a->ldw, g, epi, st);
  }
  TcGemmParams p{};
  p.skip_if_zero = skip_if_zero;
  p.M = a->M; p.N = a->N; p.num_kb = (int)(a->K / TC_BK); p.mode = 0;
  p.num_m_tiles = (int)((a->M + TC_BM - 1) / TC_BM);
  p.epi = epi;
  uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M}; uint64_t str[1] = {(uint64_t)a->lda * 2}; uint32_t box[2] = {TC_BK, TC_BM};
  rc = make_tmap_bf16(&p.tma_a[0], a->a, 2, dims, str, box); if (rc) return rc;
  // CONVT_RGB takes the whole row in one tile
  MMG_CHECK_ARG(a->epilogue != MMG_EPI_CONVT_RGB || a->N == 64 || a->N == 128 || a->N == 256, "mmg_linear: unsupported N=%lld for this epilogue", (long long)a->N);
  return dispatch_tc(p, false, a->w, a->K, a->ldw, st);
}

// e4m3 operands: the QKV and GEGLU tile epilogues only (plan_tc states the tile widths), in the tile order the bf16 product of the same
// shape takes
extern "C" int mmg_linear_fp8(const mmg_linear_fp8_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->a && a->w && a->a_scale && a->w_scale, "mmg_linear_fp8: NULL operand or scale");
  MMG_CHECK_ARG(a->dtype == MMG_E4M3, "mmg_linear_fp8: dtype %d is not MMG_E4M3", a->dtype);
  MMG_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0 && a->K % 128 == 0, "mmg_linear_fp8: bad shape M=%lld N=%lld K=%lld (K %% 128 == 0)",
                (long long)a->M, (long long)a->N, (long long)a->K);
  MMG_CHECK_ARG(a->lda >= a->K && a->ldw >= a->K && a->lda % 16 == 0 && a->ldw % 16 == 0 && aligned16(a->a) && aligned16(a->w) &&
                aligned8(a->w_scale), "mmg_linear_fp8: operands need 16-byte rows, w_scale 8-byte alignment");
  MMG_CHECK_ARG(a->epilogue == MMG_EPI_QKV || a->epilogue == MMG_EPI_QKV128 || a->epilogue == MMG_EPI_GEGLU, "mmg_linear_fp8: epilogue %d (QKV or GEGLU only, or QKV128)", a->epilogue);
  int rc = validate_epilogue(a->epilogue, a->epi, a->N); if (rc) return rc;
  const mmg_epilogue_args& e = a->epi;
  if (a->epilogue == MMG_EPI_QKV || a->epilogue == MMG_EPI_QKV128) {
    MMG_CHECK_ARG(e.out_dtype == MMG_BF16 && e.tokens > 0 && e.tokens % 32 == 0 && a->M % 128 == 0 && a->N % 128 == 0 && e.nk_heads == e.nv_heads &&
                  (!e.nq_heads || aligned16(e.q_out)) && (!e.nk_heads || (aligned16(e.k_out) && aligned16(e.v_out))),
                  "mmg_linear_fp8: QKV needs bf16 outputs, tokens %% 32 == 0, M %% 128 == 0, N %% 128 == 0 (M=%lld N=%lld tokens=%d)",
                  (long long)a->M, (long long)a->N, e.tokens);
  } else {
    MMG_CHECK_ARG(e.out_dtype == MMG_BF16 && a->N % 256 == 0 && e.ldo % 8 == 0 && aligned16(e.out),
                  "mmg_linear_fp8: GEGLU needs bf16 out, N %% 256 == 0, ldo %% 8 == 0 (N=%lld)", (long long)a->N);
  }
  TcGemmParams p{};
  p.M = a->M; p.N = a->N; p.num_kb = (int)(a->K / 128); p.mode = 0;
  p.num_m_tiles = (int)((a->M + TC_BM - 1) / TC_BM);
  p.epi.p = a->epi; p.epi.kind = a->epilogue;
  p.a_scale = a->a_scale; p.w_scale = a->w_scale;
  uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M}; uint64_t str[1] = {(uint64_t)a->lda}; uint32_t box[2] = {128, TC_BM};
  rc = make_tmap_u8(&p.tma_a[0], a->a, 2, dims, str, box); if (rc) return rc;
  return dispatch_tc(p, true, a->w, a->K, a->ldw, st);
}

extern "C" int mmg_conv2d(const mmg_conv2d_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->w, "mmg_conv2d: NULL operand");
  MMG_CHECK_ARG(a->kind >= 0 && a->kind <= 3, "mmg_conv2d: kind %d", a->kind);
  MMG_CHECK_ARG(a->B > 0 && a->H > 0 && a->W > 0 && a->Cin > 0 && a->Cout > 0, "mmg_conv2d: bad geometry");
  MMG_CHECK_ARG(a->kind != 2 || (a->H % 2 == 0 && a->W % 2 == 0), "mmg_conv2d: stride-2 conv needs even H, W");
  ConvGeom g; conv_geom(a->kind, a->B, a->H, a->W, a->Cin, &g);
  const int64_t M = (int64_t)a->B * g.Ho * g.Wo, N = a->Cout, K = (int64_t)g.ntaps * a->Cin;
  MMG_CHECK_ARG(a->epilogue != MMG_EPI_GEGLU_TANH && a->epi.act != 2, "mmg_conv2d: GEGLU_TANH / ReLU epilogues are offered by mmg_linear only");
  int rc = validate_epilogue(a->epilogue, a->epi, N); if (rc) return rc;
  Epilogue epi; epi.p = a->epi; epi.kind = a->epilogue;
  TcGemmParams p{};
  const bool tc_ok = a->dtype == MMG_BF16 && a->kind != 3 && (a->Cin % 64 == 0) && (N % 64 == 0) && aligned16(a->x) && aligned16(a->w) &&
                     (a->epi.ldo % 8 == 0) && tile_geometry(g.Ho, g.Wo, &p) == 0;
  if (!tc_ok) {
    if (a->dtype == MMG_BF16) note_simt_fallback("mmg_conv2d", M, N, K);
    return launch_simt<true>(a->dtype, a->x, a->w, M, N, K, 0, K, g, epi, st);
  }
  p.epi = epi;
  rc = conv_operand(p, g, a->x, false, N); if (rc) return rc;
  return dispatch_tc(p, false, a->w, K, K, st);
}

// e4m3 convolutions: the conv mode of tc_gemm_kernel<BN, TC_EPI_REGS, fp8e4> at the tile geometry, tile width and tile order the bf16
// convolution of the same shape takes; the register epilogue first dequantises with x_scale[image] * w_scale[col].  Shapes the kernel
// does not take are argument errors: there is no other e4m3 convolution kernel.
extern "C" int mmg_conv2d_fp8(const mmg_conv2d_fp8_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->w && a->x_scale && a->w_scale, "mmg_conv2d_fp8: NULL operand or scale");
  MMG_CHECK_ARG(a->dtype == MMG_E4M3, "mmg_conv2d_fp8: dtype %d is not MMG_E4M3", a->dtype);
  MMG_CHECK_ARG(a->kind >= 0 && a->kind <= 2, "mmg_conv2d_fp8: kind %d (1x1, 3x3 or 4x4 stride 2 only)", a->kind);
  MMG_CHECK_ARG(a->B > 0 && a->H > 0 && a->W > 0 && a->Cin > 0 && a->Cout > 0, "mmg_conv2d_fp8: bad geometry");
  MMG_CHECK_ARG(a->kind != 2 || (a->H % 2 == 0 && a->W % 2 == 0), "mmg_conv2d_fp8: stride-2 conv needs even H, W");
  MMG_CHECK_ARG(a->Cin % 128 == 0 && a->Cout % 64 == 0, "mmg_conv2d_fp8: Cin %% 128 == 0 and Cout %% 64 == 0 (Cin=%d Cout=%d)", a->Cin, a->Cout);
  MMG_CHECK_ARG(aligned16(a->x) && aligned16(a->w) && aligned8(a->w_scale) && a->epi.ldo % 8 == 0,
                "mmg_conv2d_fp8: x and w need 16-byte alignment, w_scale 8-byte alignment, epi.ldo %% 8 == 0");
  MMG_CHECK_ARG(a->epilogue == MMG_EPI_STORE || a->epilogue == MMG_EPI_RESIDUAL || a->epilogue == MMG_EPI_GLU,
                "mmg_conv2d_fp8: epilogue %d (STORE, RESIDUAL or GLU)", a->epilogue);
  MMG_CHECK_ARG(a->epi.act != 2, "mmg_conv2d_fp8: ReLU epilogues are offered by mmg_linear only");
  ConvGeom g; conv_geom(a->kind, a->B, a->H, a->W, a->Cin, &g);
  const int64_t N = a->Cout, K = (int64_t)g.ntaps * a->Cin;
  int rc = validate_epilogue(a->epilogue, a->epi, N); if (rc) return rc;
  TcGemmParams p{};
  MMG_CHECK_ARG(tile_geometry(g.Ho, g.Wo, &p) == 0, "mmg_conv2d_fp8: no conv tile geometry for a %d x %d output", g.Ho, g.Wo);
  p.epi.p = a->epi; p.epi.kind = a->epilogue;
  p.a_scale = a->x_scale; p.w_scale = a->w_scale;
  rc = conv_operand(p, g, a->x, true, N); if (rc) return rc;
  return dispatch_tc(p, true, a->w, K, K, st);
}

extern "C" int mmg_conv_transpose2d_fp8(const mmg_conv_transpose2d_fp8_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->w && a->x_scale && a->w_scale, "mmg_conv_transpose2d_fp8: NULL operand or scale");
  MMG_CHECK_ARG(a->dtype == MMG_E4M3, "mmg_conv_transpose2d_fp8: dtype %d is not MMG_E4M3", a->dtype);
  MMG_CHECK_ARG(a->epilogue == MMG_EPI_CONVT || a->epilogue == MMG_EPI_CONVT_RGB, "mmg_conv_transpose2d_fp8: epilogue must be CONVT/CONVT_RGB");
  MMG_CHECK_ARG(a->B > 0 && a->H > 0 && a->W > 0 && a->Cin > 0 && a->Cout > 0, "mmg_conv_transpose2d_fp8: bad geometry");
  MMG_CHECK_ARG(a->Cin % 128 == 0 && a->Cout % 64 == 0, "mmg_conv_transpose2d_fp8: Cin %% 128 == 0 and Cout %% 64 == 0 (Cin=%d Cout=%d)", a->Cin, a->Cout);
  MMG_CHECK_ARG(aligned16(a->x) && aligned16(a->w) && aligned8(a->w_scale), "mmg_conv_transpose2d_fp8: x and w need 16-byte alignment, w_scale 8-byte alignment");
  MMG_CHECK_ARG(a->epilogue == MMG_EPI_CONVT_RGB ? (a->Cout == 64 || a->Cout == 128 || a->Cout == 256) : (a->epi.ldo % 8 == 0),
                "mmg_conv_transpose2d_fp8: CONVT_RGB needs Cout in {64, 128, 256}, CONVT epi.ldo %% 8 == 0");
  const int64_t N = a->Cout, K = 4 * (int64_t)a->Cin;
  int rc;
  { mmg_epilogue_args e = a->epi; e.H = a->H; e.W = a->W; rc = validate_epilogue(a->epilogue, e, N); if (rc) return rc; }
  TcGemmParams p{};
  MMG_CHECK_ARG(tile_geometry(a->H, a->W, &p) == 0, "mmg_conv_transpose2d_fp8: no conv tile geometry for a %d x %d input", a->H, a->W);
  p.a_scale = a->x_scale;
  ConvGeom g; conv_geom(CONVT_PARITY, a->B, a->H, a->W, a->Cin, &g);
  rc = conv_operand(p, g, a->x, true, N); if (rc) return rc;            // one A map: every parity class reads the same input grid
  for (int py = 0; py < 2; ++py) for (int px = 0; px < 2; ++px) {
    TcGemmParams q = p;
    q.epi.p = a->epi; q.epi.kind = a->epilogue;
    q.epi.p.H = a->H; q.epi.p.W = a->W; q.epi.p.py = py; q.epi.p.px = px;
    q.w_scale = a->w_scale + (size_t)(py * 2 + px) * N;
    conv_geom(CONVT_PARITY + py * 2 + px, a->B, a->H, a->W, a->Cin, &g); conv_taps(q, g);
    const uint8_t* wp = reinterpret_cast<const uint8_t*>(a->w) + (size_t)(py * 2 + px) * N * K;
    rc = dispatch_tc(q, true, wp, K, K, st); if (rc) return rc;
  }
  return MMG_OK;
}

extern "C" int mmg_conv_transpose2d(const mmg_conv_transpose2d_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->x && a->w, "mmg_conv_transpose2d: NULL operand");
  MMG_CHECK_ARG(a->epilogue == MMG_EPI_CONVT || a->epilogue == MMG_EPI_CONVT_RGB, "mmg_conv_transpose2d: epilogue must be CONVT/CONVT_RGB");
  const int64_t M = (int64_t)a->B * a->H * a->W, N = a->Cout, K = 4 * (int64_t)a->Cin;
  MMG_CHECK_ARG(a->B > 0 && a->H > 0 && a->W > 0 && a->Cin > 0 && a->Cout > 0, "mmg_conv_transpose2d: bad geometry");
  int rc;
  { mmg_epilogue_args e = a->epi; e.H = a->H; e.W = a->W; rc = validate_epilogue(a->epilogue, e, N); if (rc) return rc; }
  TcGemmParams p{};
  const bool tc_ok = a->dtype == MMG_BF16 && (a->Cin % 64 == 0) && (N % 64 == 0) && aligned16(a->x) && aligned16(a->w) &&
                     (a->epilogue == MMG_EPI_CONVT_RGB ? (N == 64 || N == 128 || N == 256) : (a->epi.ldo % 8 == 0)) &&
                     tile_geometry(a->H, a->W, &p) == 0;
  MMG_CHECK_ARG(tc_ok || a->epilogue != MMG_EPI_CONVT_RGB, "mmg_conv_transpose2d: CONVT_RGB needs the bf16 tensor-core path (N in {64, 128, 256}, a tile geometry)");
  const size_t esz = a->dtype == MMG_BF16 ? 2 : 4;
  if (!tc_ok && a->dtype == MMG_BF16) note_simt_fallback("mmg_conv_transpose2d", M, N, K);
  for (int py = 0; py < 2; ++py) for (int px = 0; px < 2; ++px) {
    Epilogue epi; epi.p = a->epi; epi.kind = a->epilogue;
    epi.p.H = a->H; epi.p.W = a->W; epi.p.py = py; epi.p.px = px;
    const uint8_t* wp = reinterpret_cast<const uint8_t*>(a->w) + (size_t)(py * 2 + px) * N * K * esz;
    ConvGeom g{}; conv_geom(CONVT_PARITY + py * 2 + px, a->B, a->H, a->W, a->Cin, &g);
    if (!tc_ok) {
      rc = launch_simt<true>(a->dtype, a->x, wp, M, N, K, 0, K, g, epi, st); if (rc) return rc;
      continue;
    }
    TcGemmParams q = p;
    q.epi = epi;
    rc = conv_operand(q, g, a->x, false, N); if (rc) return rc;
    rc = dispatch_tc(q, false, wp, K, K, st); if (rc) return rc;
  }
  return MMG_OK;
}

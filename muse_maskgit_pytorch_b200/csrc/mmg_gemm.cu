// mmg_linear / mmg_conv2d / mmg_conv_transpose2d: launchers for the wgmma GEMM (bf16) and the fp32 CUDA-core GEMM.
#include "mmg_gemm_tc.cuh"
#include "mmg_tmap.cuh"
#include <mutex>

namespace mmg {

int linear_impl(const mmg_linear_args* a, const int* skip_if_zero, void* stream);

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

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

static int pick_bn(int64_t M_tiles, int64_t N, int epilogue) {
  if (epilogue == MMG_EPI_CONVT_RGB) return (int)N;             // whole row in one tile
  if (N % 256 == 0 && M_tiles * (N / 256) >= 2 * num_sms()) return 256;
  if (N % 128 == 0 && M_tiles * (N / 128) >= num_sms()) return 128;
  if (N % 128 == 0 && N >= 1024) return 128;
  return (N % 64 == 0 && N % 128 != 0) ? 64 : ((M_tiles * ((N + 127) / 128) >= 96) ? 128 : 64);
}

// the output tensor maps of the QKV (q / k / v heads) and GEGLU (bf16 [M, N / 2]) tile epilogues
static int bf16_out_maps(TcGemmParams& p, int epi_mode) {
  const mmg_epilogue_args& e = p.epi.p;
  int rc = MMG_OK;
  if (epi_mode == TC_EPI_QKV) {
    const uint64_t seqs = (uint64_t)(p.M / e.tokens) * (uint64_t)e.heads;
    uint64_t str[1] = {128}; uint32_t box[2] = {64, 16};
    if (e.nq_heads) { uint64_t d[2] = {64, seqs * (uint64_t)e.q_rows}; rc = make_tmap_bf16(&p.tma_qkv[0], e.q_out, 2, d, str, box); if (rc) return rc; }
    if (e.nk_heads) {
      uint64_t d[2] = {64, seqs * (uint64_t)e.kv_rows};
      rc = make_tmap_bf16(&p.tma_qkv[1], e.k_out, 2, d, str, box); if (rc) return rc;
      rc = make_tmap_bf16(&p.tma_qkv[2], e.v_out, 2, d, str, box); if (rc) return rc;
    }
  } else if (epi_mode == TC_EPI_GEGLU) {
    uint64_t od[2] = {(uint64_t)(p.N / 2), (uint64_t)p.M}; uint64_t os[1] = {(uint64_t)e.ldo * 2}; uint32_t ob[2] = {64, 16};
    rc = make_tmap_bf16(&p.tma_out, e.out, 2, od, os, ob);
  }
  return rc;
}

static int dispatch_tc(TcGemmParams& p, int bn, const void* w, int64_t N, int64_t K, int64_t ldw, cudaStream_t st) {
  const mmg_epilogue_args& e = p.epi.p;
  const bool in_place = (p.epi.kind == MMG_EPI_LNFOLD_RESIDUAL || (p.epi.kind == MMG_EPI_RESIDUAL && e.act == 0)) && e.out_dtype == MMG_F32 &&
                        e.out == e.resid && e.ldo == e.ldr && (e.ldo % 4) == 0 && aligned16(e.out) && p.mode == 0;
  const bool plain_f32 = p.epi.kind == MMG_EPI_STORE && e.out_dtype == MMG_F32 && p.mode == 0 && !e.bias && e.act == 0 && (e.ldo % 4) == 0 && aligned16(e.out);
  const bool qkv_tiles = p.epi.kind == MMG_EPI_QKV && e.out_dtype == MMG_BF16 && p.mode == 0 && e.tokens % 32 == 0 && p.M % 128 == 0 && (bn == 128 || bn == 256) &&
                         (!e.nq_heads || aligned16(e.q_out)) && (!e.nk_heads || (aligned16(e.k_out) && aligned16(e.v_out))) && e.nk_heads == e.nv_heads;
  const bool geglu_tiles = p.epi.kind == MMG_EPI_GEGLU && e.out_dtype == MMG_BF16 && p.mode == 0 && bn == 256 && (e.ldo % 8) == 0 && aligned16(e.out);
  const int epi_mode = p.epi.is_act() ? TC_EPI_ACT : in_place ? TC_EPI_REDUCE : (plain_f32 && (bn == 256 || bn == 128)) ? TC_EPI_TSTORE :
                       qkv_tiles ? TC_EPI_QKV : geglu_tiles ? TC_EPI_GEGLU : TC_EPI_REGS;
  // 128 accumulator registers per thread at BN = 256 next to a 64-column row chunk would spill, so <256, TC_EPI_REGS> compiles only
  // the fused RGB epilogue, which reduces the fragments in place; every other register-epilogue kind runs at BN <= 128, and the T5
  // feed-forward epilogues (their own instantiation, kept out of the VAE's) at BN = 128 only
  if (epi_mode == TC_EPI_REGS && bn == 256 && p.epi.kind != MMG_EPI_CONVT_RGB) bn = 128;
  if (epi_mode == TC_EPI_ACT) bn = 128;
  // the tile epilogues write whole 32- / 64-column boxes: pick_bn's widths divide N (N % 64 == 0 on this path)
  MMG_CHECK_ARG(!tc_tile_epilogue(epi_mode) || N % bn == 0, "tile epilogue: tile width %d does not divide N = %lld", bn, (long long)N);
  p.num_n_tiles = (int)((N + bn - 1) / bn);
  p.n_fast = ((int64_t)N * K * 2 <= (8 << 20) && p.num_n_tiles > 1 && p.num_n_tiles <= 16) ? 1 : 0;
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)N}; uint64_t str[1] = {(uint64_t)ldw * 2}; uint32_t box[2] = {TC_BK, (uint32_t)bn};
  int rc = make_tmap_bf16(&p.tma_b, w, 2, dims, str, box); if (rc) return rc;
  if (epi_mode == TC_EPI_QKV) {
    rc = bf16_out_maps(p, epi_mode); if (rc) return rc;
    return bn == 256 ? launch_tc<256, TC_EPI_QKV>(p, st) : launch_tc<128, TC_EPI_QKV>(p, st);
  }
  if (epi_mode == TC_EPI_GEGLU) {
    rc = bf16_out_maps(p, epi_mode); if (rc) return rc;
    return launch_tc<256, TC_EPI_GEGLU>(p, st);
  }
  if (epi_mode == TC_EPI_ACT) return launch_tc<128, TC_EPI_ACT>(p, st);
  if (epi_mode != TC_EPI_REGS) {
    uint64_t od[2] = {(uint64_t)p.N, (uint64_t)p.M}; uint64_t os[1] = {(uint64_t)e.ldo * 4}; uint32_t ob[2] = {32, 16};
    rc = make_tmap_f32(&p.tma_out, e.out, 2, od, os, ob); if (rc) return rc;
  }
  if (epi_mode == TC_EPI_TSTORE) return bn == 256 ? launch_tc<256, TC_EPI_TSTORE>(p, st) : launch_tc<128, TC_EPI_TSTORE>(p, st);   // 128: the sample GEMM of the fused tail at small batch
  if (epi_mode == TC_EPI_REDUCE) {
    switch (bn) { case 64: return launch_tc<64, TC_EPI_REDUCE>(p, st); case 128: return launch_tc<128, TC_EPI_REDUCE>(p, st); case 256: return launch_tc<256, TC_EPI_REDUCE>(p, st); }
  }
  switch (bn) {
    case 64: return launch_tc<64, TC_EPI_REGS>(p, st);
    case 128: return launch_tc<128, TC_EPI_REGS>(p, st);
    case 256: return launch_tc<256, TC_EPI_REGS>(p, st);       // CONVT_RGB: the whole 256-column row in one tile
  }
  return fail(MMG_EINVAL, "unsupported tile width %d", bn);
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
static void conv_geom(int kind, int B, int H, int W, int Cin, ConvGeom* g) {
  const int k = kind == 0 ? 1 : kind == 1 ? 3 : kind == 2 ? 4 : 5;
  const int pad = kind == 0 ? 0 : kind == 1 ? 1 : kind == 2 ? 1 : 2;
  g->B = B; g->H = H; g->W = W; g->Cin = Cin; g->stride = (kind == 2) ? 2 : 1;
  g->Ho = H / g->stride; g->Wo = W / g->stride; g->ntaps = k * k;
  for (int r = 0; r < k; ++r) for (int s = 0; s < k; ++s) { g->tdy[r * k + s] = (int8_t)(r - pad); g->tdx[r * k + s] = (int8_t)(s - pad); }
}

// conv-transpose (k4 s2 p1) parity class (py,px): 2x2 taps, tap t = a*2+b, input offset dy = DY[py][a], kernel row r = R[py][a].
static const int CT_D[2][2] = {{0, -1}, {1, 0}};

static int tile_geometry(int Ho, int Wo, TcGemmParams* p) {
  int TW = Wo < 128 ? Wo : 128;
  if (128 % TW != 0 || Wo % TW != 0) return -1;
  int TH = 128 / TW; if (TH > Ho) TH = Ho;
  if (Ho % TH != 0 || 128 % (TW * TH) != 0) return -1;
  p->TW = TW; p->TH = TH; p->TB = 128 / (TW * TH);
  p->tiles_x = Wo / TW; p->tiles_y = Ho / TH;
  return 0;
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
                     aligned16(a->a) && aligned16(a->w) && (a->epi.ldo % 8 == 0 || a->epilogue == MMG_EPI_QKV || a->epilogue == MMG_EPI_CONVT_RGB || a->epilogue == MMG_EPI_LFQ_IDS || a->epilogue == MMG_EPI_ARGMIN);
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
  const int bn = pick_bn(p.num_m_tiles, a->N, a->epilogue);
  MMG_CHECK_ARG(bn == 64 || bn == 128 || bn == 256, "mmg_linear: unsupported N=%lld for this epilogue", (long long)a->N);
  return dispatch_tc(p, bn, a->w, a->N, a->K, a->ldw, st);
}

// e4m3 operands: the QKV and GEGLU tile epilogues only, at the tile widths and tile order the bf16 product of the same shape takes
extern "C" int mmg_linear_fp8(const mmg_linear_fp8_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MMG_CHECK_ARG(a && a->a && a->w && a->a_scale && a->w_scale, "mmg_linear_fp8: NULL operand or scale");
  MMG_CHECK_ARG(a->dtype == MMG_E4M3, "mmg_linear_fp8: dtype %d is not MMG_E4M3", a->dtype);
  MMG_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0 && a->K % 128 == 0, "mmg_linear_fp8: bad shape M=%lld N=%lld K=%lld (K %% 128 == 0)",
                (long long)a->M, (long long)a->N, (long long)a->K);
  MMG_CHECK_ARG(a->lda >= a->K && a->ldw >= a->K && a->lda % 16 == 0 && a->ldw % 16 == 0 && aligned16(a->a) && aligned16(a->w) &&
                (reinterpret_cast<uintptr_t>(a->w_scale) & 7) == 0, "mmg_linear_fp8: operands need 16-byte rows, w_scale 8-byte alignment");
  MMG_CHECK_ARG(a->epilogue == MMG_EPI_QKV || a->epilogue == MMG_EPI_GEGLU, "mmg_linear_fp8: epilogue %d (QKV or GEGLU only)", a->epilogue);
  int rc = validate_epilogue(a->epilogue, a->epi, a->N); if (rc) return rc;
  const mmg_epilogue_args& e = a->epi;
  const int64_t m_tiles = (a->M + TC_BM - 1) / TC_BM;
  int bn = 256, epi_mode = TC_EPI_GEGLU;
  if (a->epilogue == MMG_EPI_QKV) {
    MMG_CHECK_ARG(e.out_dtype == MMG_BF16 && e.tokens > 0 && e.tokens % 32 == 0 && a->M % 128 == 0 && a->N % 128 == 0 && e.nk_heads == e.nv_heads &&
                  (!e.nq_heads || aligned16(e.q_out)) && (!e.nk_heads || (aligned16(e.k_out) && aligned16(e.v_out))),
                  "mmg_linear_fp8: QKV needs bf16 outputs, tokens %% 32 == 0, M %% 128 == 0, N %% 128 == 0 (M=%lld N=%lld tokens=%d)",
                  (long long)a->M, (long long)a->N, e.tokens);
    bn = pick_bn(m_tiles, a->N, a->epilogue) == 256 ? 256 : 128;
    epi_mode = TC_EPI_QKV;
  } else {
    MMG_CHECK_ARG(e.out_dtype == MMG_BF16 && a->N % 256 == 0 && e.ldo % 8 == 0 && aligned16(e.out),
                  "mmg_linear_fp8: GEGLU needs bf16 out, N %% 256 == 0, ldo %% 8 == 0 (N=%lld)", (long long)a->N);
  }
  TcGemmParams p{};
  p.M = a->M; p.N = a->N; p.num_kb = (int)(a->K / 128); p.mode = 0;
  p.num_m_tiles = (int)m_tiles;
  p.num_n_tiles = (int)(a->N / bn);
  p.n_fast = ((int64_t)a->N * a->K * 2 <= (8 << 20) && p.num_n_tiles > 1 && p.num_n_tiles <= 16) ? 1 : 0;   // the bf16 product's tile order
  p.epi.p = a->epi; p.epi.kind = a->epilogue;
  p.a_scale = a->a_scale; p.w_scale = a->w_scale;
  { uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M}; uint64_t str[1] = {(uint64_t)a->lda}; uint32_t box[2] = {128, TC_BM};
    rc = make_tmap_u8(&p.tma_a[0], a->a, 2, dims, str, box); if (rc) return rc; }
  { uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->N}; uint64_t str[1] = {(uint64_t)a->ldw}; uint32_t box[2] = {128, (uint32_t)bn};
    rc = make_tmap_u8(&p.tma_b, a->w, 2, dims, str, box); if (rc) return rc; }
  rc = bf16_out_maps(p, epi_mode); if (rc) return rc;
  if (epi_mode == TC_EPI_GEGLU) return launch_tc<256, TC_EPI_GEGLU, fp8e4>(p, st);
  return bn == 256 ? launch_tc<256, TC_EPI_QKV, fp8e4>(p, st) : launch_tc<128, TC_EPI_QKV, fp8e4>(p, st);
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
  p.M = M; p.N = N; p.mode = 1; p.cchunks = a->Cin / 64; p.ntaps = g.ntaps; p.num_kb = p.ntaps * p.cchunks;
  p.Ho = g.Ho; p.Wo = g.Wo; p.B = a->B;
  p.num_m_tiles = p.tiles_x * p.tiles_y * ((a->B + p.TB - 1) / p.TB);
  p.epi = epi;
  const uint64_t C = a->Cin, W = a->W, H = a->H;
  uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TB};
  if (a->kind != 2) {
    uint64_t dims[4] = {C, W, H, (uint64_t)a->B}; uint64_t str[3] = {C * 2, W * C * 2, H * W * C * 2};
    rc = make_tmap_bf16(&p.tma_a[0], a->x, 4, dims, str, box); if (rc) return rc;
    for (int t = 0; t < g.ntaps; ++t) { p.tap_map[t] = 0; p.tap_dy[t] = g.tdy[t]; p.tap_dx[t] = g.tdx[t]; }
  } else {
    // stride 2: input row 2y + (r-1) = 2(y+dy) + py.  One tensor map per input parity (py,px) over the (H/2, W/2) grid.
    for (int py = 0; py < 2; ++py) for (int px = 0; px < 2; ++px) {
      const uint8_t* base = reinterpret_cast<const uint8_t*>(a->x) + ((uint64_t)py * W + px) * C * 2;
      uint64_t dims[4] = {C, W / 2, H / 2, (uint64_t)a->B}; uint64_t str[3] = {2 * C * 2, 2 * W * C * 2, H * W * C * 2};
      rc = make_tmap_bf16(&p.tma_a[py * 2 + px], base, 4, dims, str, box); if (rc) return rc;
    }
    for (int r = 0; r < 4; ++r) for (int s = 0; s < 4; ++s) {
      const int oy = r - 1, ox = s - 1;
      const int py = ((oy % 2) + 2) % 2, px = ((ox % 2) + 2) % 2;
      p.tap_map[r * 4 + s] = (int8_t)(py * 2 + px); p.tap_dy[r * 4 + s] = (int8_t)((oy - py) / 2); p.tap_dx[r * 4 + s] = (int8_t)((ox - px) / 2);
    }
  }
  const int bn = pick_bn(p.num_m_tiles, N, a->epilogue);
  return dispatch_tc(p, bn, a->w, N, K, K, st);
}

// ------------------------------------------------------------------------------------------------------------------
// e4m3 convolutions: the conv mode of tc_gemm_kernel<BN, TC_EPI_REGS, fp8e4> at the tile geometry, tile width and tile order the bf16
// convolution of the same shape takes.  A k-block is one tap x 128 channels (Cin % 128 == 0); the register epilogue first dequantises
// with x_scale[image] * w_scale[col].  Shapes the kernel does not take are argument errors: there is no other e4m3 convolution kernel.
// ------------------------------------------------------------------------------------------------------------------
static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

static int launch_conv_fp8(TcGemmParams& p, const void* w, int64_t N, int64_t K, cudaStream_t st) {
  int bn = pick_bn(p.num_m_tiles, N, p.epi.kind);
  if (bn == 256 && p.epi.kind != MMG_EPI_CONVT_RGB) bn = 128;        // dispatch_tc's register-epilogue width (<256, REGS>: RGB only)
  p.num_n_tiles = (int)((N + bn - 1) / bn);
  p.n_fast = ((int64_t)N * K * 2 <= (8 << 20) && p.num_n_tiles > 1 && p.num_n_tiles <= 16) ? 1 : 0;   // the bf16 product's tile order
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)N}; uint64_t str[1] = {(uint64_t)K}; uint32_t box[2] = {128, (uint32_t)bn};
  int rc = make_tmap_u8(&p.tma_b, w, 2, dims, str, box); if (rc) return rc;
  switch (bn) {
    case 64: return launch_tc<64, TC_EPI_REGS, fp8e4>(p, st);
    case 128: return launch_tc<128, TC_EPI_REGS, fp8e4>(p, st);
    case 256: return launch_tc<256, TC_EPI_REGS, fp8e4>(p, st);      // CONVT_RGB: the whole 256-column row in one tile
  }
  return fail(MMG_EINVAL, "e4m3 convolution: unsupported tile width %d", bn);
}

// the A tensor map(s) of an e4m3 NHWC map: one 4-D map (stride 1), or one per input parity over the (H/2, W/2) grid (stride 2)
static int fp8_image_maps(TcGemmParams& p, const void* x, int B, int H, int W, int Cin, bool stride2) {
  const uint64_t C = Cin, Wd = W, Hd = H;
  uint32_t box[4] = {128, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TB};
  if (!stride2) {
    uint64_t dims[4] = {C, Wd, Hd, (uint64_t)B}; uint64_t str[3] = {C, Wd * C, Hd * Wd * C};
    return make_tmap_u8(&p.tma_a[0], x, 4, dims, str, box);
  }
  for (int py = 0; py < 2; ++py) for (int px = 0; px < 2; ++px) {
    const uint8_t* base = reinterpret_cast<const uint8_t*>(x) + ((uint64_t)py * Wd + px) * C;
    uint64_t dims[4] = {C, Wd / 2, Hd / 2, (uint64_t)B}; uint64_t str[3] = {2 * C, 2 * Wd * C, Hd * Wd * C};
    const int rc = make_tmap_u8(&p.tma_a[py * 2 + px], base, 4, dims, str, box); if (rc) return rc;
  }
  return MMG_OK;
}

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
  const int64_t M = (int64_t)a->B * g.Ho * g.Wo, N = a->Cout, K = (int64_t)g.ntaps * a->Cin;
  int rc = validate_epilogue(a->epilogue, a->epi, N); if (rc) return rc;
  TcGemmParams p{};
  MMG_CHECK_ARG(tile_geometry(g.Ho, g.Wo, &p) == 0, "mmg_conv2d_fp8: no conv tile geometry for a %d x %d output", g.Ho, g.Wo);
  p.M = M; p.N = N; p.mode = 1; p.cchunks = a->Cin / 128; p.ntaps = g.ntaps; p.num_kb = p.ntaps * p.cchunks;
  p.Ho = g.Ho; p.Wo = g.Wo; p.B = a->B;
  p.num_m_tiles = p.tiles_x * p.tiles_y * ((a->B + p.TB - 1) / p.TB);
  p.epi.p = a->epi; p.epi.kind = a->epilogue;
  p.a_scale = a->x_scale; p.w_scale = a->w_scale;
  rc = fp8_image_maps(p, a->x, a->B, a->H, a->W, a->Cin, a->kind == 2); if (rc) return rc;
  if (a->kind != 2) {
    for (int t = 0; t < g.ntaps; ++t) { p.tap_map[t] = 0; p.tap_dy[t] = g.tdy[t]; p.tap_dx[t] = g.tdx[t]; }
  } else {
    for (int r = 0; r < 4; ++r) for (int s = 0; s < 4; ++s) {
      const int oy = r - 1, ox = s - 1;
      const int py = ((oy % 2) + 2) % 2, px = ((ox % 2) + 2) % 2;
      p.tap_map[r * 4 + s] = (int8_t)(py * 2 + px); p.tap_dy[r * 4 + s] = (int8_t)((oy - py) / 2); p.tap_dx[r * 4 + s] = (int8_t)((ox - px) / 2);
    }
  }
  return launch_conv_fp8(p, a->w, N, K, st);
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
  const int64_t M = (int64_t)a->B * a->H * a->W, N = a->Cout, K = 4 * (int64_t)a->Cin;
  int rc;
  { mmg_epilogue_args e = a->epi; e.H = a->H; e.W = a->W; rc = validate_epilogue(a->epilogue, e, N); if (rc) return rc; }
  TcGemmParams p{};
  MMG_CHECK_ARG(tile_geometry(a->H, a->W, &p) == 0, "mmg_conv_transpose2d_fp8: no conv tile geometry for a %d x %d input", a->H, a->W);
  p.M = M; p.N = N; p.mode = 1; p.cchunks = a->Cin / 128; p.ntaps = 4; p.num_kb = 4 * p.cchunks;
  p.Ho = a->H; p.Wo = a->W; p.B = a->B;
  p.num_m_tiles = p.tiles_x * p.tiles_y * ((a->B + p.TB - 1) / p.TB);
  p.a_scale = a->x_scale;
  rc = fp8_image_maps(p, a->x, a->B, a->H, a->W, a->Cin, false); if (rc) return rc;
  for (int py = 0; py < 2; ++py) for (int px = 0; px < 2; ++px) {
    TcGemmParams q = p;
    q.epi.p = a->epi; q.epi.kind = a->epilogue;
    q.epi.p.H = a->H; q.epi.p.W = a->W; q.epi.p.py = py; q.epi.p.px = px;
    q.w_scale = a->w_scale + (size_t)(py * 2 + px) * N;
    for (int t = 0; t < 4; ++t) { q.tap_map[t] = 0; q.tap_dy[t] = (int8_t)CT_D[py][t >> 1]; q.tap_dx[t] = (int8_t)CT_D[px][t & 1]; }
    const uint8_t* wp = reinterpret_cast<const uint8_t*>(a->w) + (size_t)(py * 2 + px) * N * K;
    rc = launch_conv_fp8(q, wp, N, K, st); if (rc) return rc;
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
    if (!tc_ok) {
      ConvGeom g{}; g.B = a->B; g.H = a->H; g.W = a->W; g.Cin = a->Cin; g.Ho = a->H; g.Wo = a->W; g.stride = 1; g.ntaps = 4;
      for (int t = 0; t < 4; ++t) { g.tdy[t] = (int8_t)CT_D[py][t >> 1]; g.tdx[t] = (int8_t)CT_D[px][t & 1]; }
      rc = launch_simt<true>(a->dtype, a->x, wp, M, N, K, 0, K, g, epi, st); if (rc) return rc;
      continue;
    }
    TcGemmParams q = p;
    q.M = M; q.N = N; q.mode = 1; q.cchunks = a->Cin / 64; q.ntaps = 4; q.num_kb = 4 * q.cchunks;
    q.Ho = a->H; q.Wo = a->W; q.B = a->B;
    q.num_m_tiles = q.tiles_x * q.tiles_y * ((a->B + q.TB - 1) / q.TB);
    q.epi = epi;
    const uint64_t C = a->Cin, W = a->W, H = a->H;
    uint64_t dims[4] = {C, W, H, (uint64_t)a->B}; uint64_t str[3] = {C * 2, W * C * 2, H * W * C * 2};
    uint32_t box[4] = {64, (uint32_t)q.TW, (uint32_t)q.TH, (uint32_t)q.TB};
    rc = make_tmap_bf16(&q.tma_a[0], a->x, 4, dims, str, box); if (rc) return rc;
    for (int t = 0; t < 4; ++t) { q.tap_map[t] = 0; q.tap_dy[t] = (int8_t)CT_D[py][t >> 1]; q.tap_dx[t] = (int8_t)CT_D[px][t & 1]; }
    const int bn = pick_bn(q.num_m_tiles, N, a->epilogue);
    rc = dispatch_tc(q, bn, wp, N, K, K, st); if (rc) return rc;
  }
  return MMG_OK;
}


/*
 * mmg.h — C-ABI of libmmg.so: hand-written sm_90a kernels for the MaskGit.generate() hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b, "lower face").  Every entry point is
 *     extern "C" int mmg_<op>(const mmg_<op>_args* a, void* cuda_stream);
 * with a POD argument block of raw DEVICE pointers + sizes.  Conventions:
 *   - returns 0 on success, a negative MMG_E* code otherwise; never throws, never allocates device memory,
 *     never synchronises the host; asynchronous on `cuda_stream` (a cudaStream_t) and CUDA-graph capturable;
 *   - no ownership transfer; the caller (PyTorch) owns all buffers;
 *   - mmg_last_error() returns a thread-local, human readable description of the last failure;
 *   - activations are row-major "token-major" matrices [rows, channels] (images: NHWC); `dtype` selects the
 *     operand type of a matrix product: MMG_BF16 -> wgmma tensor-core path (fp32 accumulate),
 *     MMG_F32 -> fp32 CUDA-core path ("parity precision").  There is no CPU path in this library.
 *
 * Each function cites the reference code it replaces (paths relative to /root/reference/muse_maskgit_pytorch/).
 */
#ifndef MMG_H_
#define MMG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMG_VERSION 101

/* error codes */
#define MMG_OK            0
#define MMG_EINVAL       -1   /* bad argument / unsupported shape */
#define MMG_ECUDA        -2   /* CUDA runtime / driver error (see mmg_last_error) */
#define MMG_EUNSUPPORTED -3   /* device is not sm_90 */

/* operand dtypes */
#define MMG_F32  0
#define MMG_BF16 1
#define MMG_E4M3 2   /* fp8 e4m3 (OCP E4M3FN: largest finite 448, no infinities): mmg_linear_fp8 / mmg_conv*_fp8 operands, mmg_layernorm_fp8 /
                          mmg_quantize_e4m3_images output */

int         mmg_version(void);
const char* mmg_last_error(void);
/* Number of kernel launches issued through this library by the calling process (bench.py "gpu_launches"). */
int64_t     mmg_launch_count(void);
/* Number of bf16 matrix products / convolutions of this process that fell off the wgmma path onto the CUDA-core kernel because of their shape
 * or alignment (K or Cin % 64, N % 64, 16-byte rows, conv tile geometry).  MMG_VERBOSE=1 logs each one to stderr. */
int64_t     mmg_simt_fallback_count(void);
/* Number of launches of the CUDA-core matrix-product / attention kernels (any dtype) by this process.  precision="fp32" runs its products on the
 * tensor cores as 3-way bf16 splits (mmg_split3), so this stays 0 for a model whose shapes the TMA path takes. */
int64_t     mmg_simt_launch_count(void);
/* sizeof() of the argument block of entry point `name` ("mmg_linear", ...; "mmg_epilogue" for mmg_epilogue_args): lets a
 * foreign-language binding verify its struct mirror. Returns 0 for unknown names. */
int         mmg_sizeof(const char* name);

/* ------------------------------------------------------------------------------------------------
 * Matrix product with fused epilogue:  C[M,N] = A[M,K] * W[N,K]^T  (+ epilogue)
 * replaces: every nn.Linear on the path (muse_maskgit_pytorch.py:85,88,118,119,124,225,233) and, through
 * mmg_conv2d / mmg_conv_transpose2d below, every nn.Conv2d / nn.ConvTranspose2d (vqgan_vae.py:224-232,255-277).
 * ---------------------------------------------------------------------------------------------- */
enum mmg_epilogue {
  MMG_EPI_STORE      = 0, /* out[r, c] = acc (+bias[c]) (+leaky_relu 0.1 if act==1); out dtype = out_dtype          */
  MMG_EPI_RESIDUAL   = 1, /* out[r, c] = acc (+bias[c]) + resid[r, c]; out/resid dtype = out_dtype (may alias)      */
  MMG_EPI_GEGLU      = 2, /* W rows interleaved in blocks of 32: [x(32) | gate(32)]; out[r, c/2] = gate*gelu_erf(x) */
  MMG_EPI_GLU        = 3, /* same interleave, with bias: out = (a+ba) * sigmoid(g+bg)         (nn.GLU, vqgan_vae.py:256) */
  MMG_EPI_QKV        = 4, /* N = (nq+nk+nv)*64 head-columns: l2norm(q)*q_scale, l2norm(k)*k_scale, v -> per-head layouts;
                             q_out / k_out / v_out / null_k / null_v 16-byte aligned (else MMG_EINVAL)                       */
  MMG_EPI_CONVT      = 5, /* conv-transpose parity scatter: out pixel (2y+py, 2x+px) = leaky(acc + bias)             */
  MMG_EPI_CONVT_RGB  = 6, /* CONVT followed by the fused final 1x1 conv (C -> channels<=4), fp32 NCHW output          */
  MMG_EPI_LNFOLD_RESIDUAL = 7, /* LayerNorm folded through the product: with W' = W*gamma, cvec[c] = sum_k W'[c,k] (passed as
                                  `bias`) and per-row (sum, sumsq) of the un-normalised A row in `row_stats`:
                                  out[r,c] = resid[r,c] + rstd_r * (acc - mean_r * cvec[c])   == resid + LN(a_r) W^T;
                                  out and resid 16-byte aligned (else MMG_EINVAL)                                                */
  MMG_EPI_LFQ_IDS    = 8, /* LFQ lookup fused into the projection: W rows = [hi(bits) | mid(bits) | lo(bits)] (a 3-way bf16 split
                             of the fp32 project_in weight, 3*bits <= 64 = N), bias = project_in bias [bits], ln_width = bits:
                             ids[r] = sum_i ((hi+mid+lo)_i + bias_i > 0) << (bits-1-i), written as int64 to out[r]                */
  MMG_EPI_ARGMIN     = 9, /* nearest codebook row: W = codebook [K, D], bias = ||e_k||^2 [K]; out = uint64 best[M], initialised to
                             all-ones by the caller, updated with atomicMin( orderkey(||e||^2 - 2 x.e) << 32 | k ): lowest k on ties */
  MMG_EPI_GEGLU_TANH = 10,/* GEGLU interleave (blocks of 32: [x(32) | gate(32)]), no bias, tanh-approximated GELU ("gelu_new" of T5 v1.1,
                             t5.py): out[r, c/2] = gelu_tanh(x) * gate; mmg_linear only                                        */
  MMG_EPI_QKV128     = 11,/* QKV with 128-column heads: the fields of MMG_EPI_QKV, with N = (nq+nk+nv)*128, q_scale / k_scale [128],
                             null_k / null_v [heads, 128], q_out [BH, q_rows, 128], k_out / v_out [BH, kv_rows, 128].  wgmma path only
                             (mmg_linear with bf16 operands that it takes, mmg_linear_fp8): any call that would run on the CUDA-core
                             kernel returns MMG_EINVAL and launches nothing                                                    */
};

typedef struct {
  void*        out;        /* see enum; [M, ldo]; any element offset (an unaligned out / resid is written element by element) */
  int64_t      ldo;        /* leading dimension of out (elements)                                                */
  int32_t      out_dtype;  /* MMG_F32 / MMG_BF16                                                                 */
  int32_t      act;        /* 0 none, 1 leaky_relu(0.1), 2 relu (STORE of mmg_linear only)                       */
  const float* bias;       /* [N] or NULL (for GEGLU/GLU: interleaved like W rows)                               */
  const void*  resid;      /* RESIDUAL: [M, ldr] of out_dtype                                                    */
  int64_t      ldr;
  /* QKV: q -> q_out[(b*heads+h), t, 64]; k,v -> k_out/v_out[(b*heads+h), key_off + t, 64] with row r = b*tokens + t */
  void*        q_out; void* k_out; void* v_out;   /* dtype = out_dtype                                            */
  const float* q_scale; const float* k_scale;     /* [64]                                                         */
  const void*  null_k; const void* null_v;        /* optional [heads, 64] of out_dtype: written to key row 0 of every
                                                     (b, h) by the thread that owns token 0 (learned null key/value) */
  int32_t      heads, tokens, q_rows, kv_rows, key_off, nq_heads, nk_heads, nv_heads;
  /* CONVT(_RGB): input geometry of the GEMM rows (b, y, x) and the output parity                                  */
  int32_t      H, W, py, px;
  float*       row_stats;  /* [M, stats_slots, 2] fp32 (sum, sum of squares) partials.  GEGLU: the epilogue WRITES the statistics of each
                              64-column accumulator chunk (32 outputs, as rounded to out_dtype) to slot col / 64 (stats_slots >= N / 64;
                              every slot of every row is written exactly once, no atomics); LNFOLD_RESIDUAL: adds the stats_slots partials
                              of its row in ascending order (statistics over ln_width columns, eps 1e-5) — bitwise reproducible           */
  int32_t      ln_width; int32_t stats_slots;
  const float* rgb_w;      /* CONVT_RGB: [channels, N] fp32 1x1 weights, rgb_b [channels]                          */
  const float* rgb_b;
  int32_t      rgb_channels;
  int32_t      _pad;
} mmg_epilogue_args;

typedef struct {
  const void* a;           /* [M, lda] operand dtype                                                             */
  const void* w;           /* [N, ldw] operand dtype (nn.Linear weight layout, K contiguous)                     */
  int64_t M, N, K, lda, ldw;
  int32_t dtype;           /* MMG_BF16: wgmma path when K % 64 == 0, N % 64 == 0, lda % 8 == 0, ldw % 8 == 0, a and w 16-byte aligned
                              and epi.ldo % 8 == 0 (not required for QKV, CONVT_RGB, LFQ_IDS, ARGMIN); any other bf16 call runs on the
                              CUDA-core kernel and counts in mmg_simt_fallback_count.  MMG_F32: CUDA cores                         */
  int32_t epilogue;        /* enum mmg_epilogue                                                                   */
  mmg_epilogue_args epi;
} mmg_linear_args;
int mmg_linear(const mmg_linear_args* a, void* stream);

/* The same product with e4m3 operands and one fp32 scale per row of A and per row of W (precision="fp8"):
 *   acc[r, c] = sum_k qa[r, k] qw[c, k]  (fp32 accumulation on the fp8 tensor cores),  C[r, c] = acc[r, c] * a_scale[r] * w_scale[c]
 * then the epilogue exactly as mmg_linear's tile epilogue: MMG_EPI_QKV (bf16 q / k / v, tokens % 32 == 0, M % 128 == 0, N % 128 == 0,
 * nk_heads == nv_heads) or MMG_EPI_GEGLU (bf16 out, N % 256 == 0, ldo % 8 == 0, optional row_stats partials of the dequantised outputs).
 * K % 128 == 0, lda / ldw % 16 == 0, 16-byte aligned operands, w_scale 8-byte aligned.  Any other shape or epilogue returns MMG_EINVAL;
 * there is no fallback kernel.                                                                                        */
typedef struct {
  const void*  a;          /* [M, lda] e4m3                                                                      */
  const void*  w;          /* [N, ldw] e4m3 (nn.Linear weight layout, K contiguous)                              */
  const float* a_scale;    /* [M] (mmg_layernorm_fp8 row_scale)                                                  */
  const float* w_scale;    /* [N]                                                                                */
  int64_t M, N, K, lda, ldw;
  int32_t dtype;           /* MMG_E4M3                                                                           */
  int32_t epilogue;        /* MMG_EPI_QKV or MMG_EPI_GEGLU                                                       */
  mmg_epilogue_args epi;
} mmg_linear_fp8_args;
int mmg_linear_fp8(const mmg_linear_fp8_args* a, void* stream);

/* Convolutions as implicit GEMM over NHWC activations; weights pre-packed [Cout, taps*Cin] (tap-major, Cin
 * contiguous).  kind: 0 = 1x1; 1 = 3x3 stride 1 pad 1; 2 = 4x4 stride 2 pad 1; 3 = 5x5 stride 1 pad 2.
 * replaces: nn.Conv2d at vqgan_vae.py:224,231,232,255,258,261,271,274,277.                                        */
typedef struct {
  const void* x;           /* [B, H, W, Cin]                                                                     */
  const void* w;           /* [Cout, taps*Cin]                                                                   */
  int32_t B, H, W, Cin, Cout, kind;
  int32_t dtype, epilogue; /* STORE / RESIDUAL / GLU                                                             */
  mmg_epilogue_args epi;   /* rows of `out` are output pixels (b, y, x) in NHWC order                            */
} mmg_conv2d_args;
int mmg_conv2d(const mmg_conv2d_args* a, void* stream);

/* ConvTranspose2d(k=4, s=2, p=1) as 4 parity-class GEMMs (K = 4*Cin each).  w: [4 parities][Cout, 4*Cin].
 * replaces: nn.ConvTranspose2d + LeakyReLU at vqgan_vae.py:225 (and, with CONVT_RGB, the 1x1 at vqgan_vae.py:232).
 * CONVT_RGB runs on the bf16 tensor-core kernel only: dtype MMG_BF16, Cout in {64, 128, 256}, Cin % 64 == 0, 16-byte aligned x and w, and
 * an (H, W) that the conv tile geometry takes (TW = min(W, 128) divides 128 and W; TH = min(128 / TW, H) divides H; TW * TH divides
 * 128).  Any other CONVT_RGB
 * call returns MMG_EINVAL and launches nothing.  mmg_conv2d and this call return MMG_EINVAL for B, H, W, Cin or Cout <= 0.           */
typedef struct {
  const void* x;           /* [B, H, W, Cin]                                                                     */
  const void* w;           /* [4, Cout, 4*Cin]                                                                   */
  int32_t B, H, W, Cin, Cout;
  int32_t dtype, epilogue; /* CONVT or CONVT_RGB                                                                 */
  mmg_epilogue_args epi;   /* out: [B, 2H, 2W, Cout] (CONVT) or fp32 [B, channels, 2H, 2W] (CONVT_RGB)           */
} mmg_conv_transpose2d_args;
int mmg_conv_transpose2d(const mmg_conv_transpose2d_args* a, void* stream);

/* The same convolutions with e4m3 operands (VQGanVAE precision="fp8"): one fp32 scale per IMAGE of x (mmg_quantize_e4m3_images) and one
 * per row of w (output channel; per parity class for the conv-transpose):
 *   acc[r, c] = sum_k qx[r, k] qw[c, k]  (fp8 tensor cores),  C[r, c] = acc[r, c] * x_scale[image of output row r] * w_scale[c]
 * then the register epilogue exactly as the bf16 call's: STORE (+ bias, LeakyReLU act = 1), RESIDUAL (bf16 resid), GLU (mmg_conv2d_fp8);
 * CONVT, CONVT_RGB (mmg_conv_transpose2d_fp8).  One k-block is one tap x 128 channels.  Requires Cin % 128 == 0, Cout % 64 == 0, x and w
 * 16-byte aligned, w_scale 8-byte aligned, an output (conv) / input (conv-transpose) grid the conv tile geometry takes, kind 0, 1 or 2,
 * epi.ldo % 8 == 0 (CONVT_RGB: Cout in {64, 128, 256}).  Any other call returns MMG_EINVAL and launches nothing: there is no fallback. */
typedef struct {
  const void*  x;          /* [B, H, W, Cin] e4m3                                                                */
  const void*  w;          /* [Cout, taps*Cin] e4m3                                                              */
  const float* x_scale;    /* [B]                                                                                */
  const float* w_scale;    /* [Cout]                                                                             */
  int32_t B, H, W, Cin, Cout, kind;
  int32_t dtype, epilogue; /* MMG_E4M3; STORE / RESIDUAL / GLU                                                   */
  mmg_epilogue_args epi;
} mmg_conv2d_fp8_args;
int mmg_conv2d_fp8(const mmg_conv2d_fp8_args* a, void* stream);

typedef struct {
  const void*  x;          /* [B, H, W, Cin] e4m3                                                                */
  const void*  w;          /* [4, Cout, 4*Cin] e4m3                                                              */
  const float* x_scale;    /* [B]                                                                                */
  const float* w_scale;    /* [4, Cout]                                                                          */
  int32_t B, H, W, Cin, Cout;
  int32_t dtype, epilogue; /* MMG_E4M3; CONVT or CONVT_RGB                                                       */
  mmg_epilogue_args epi;
} mmg_conv_transpose2d_fp8_args;
int mmg_conv_transpose2d_fp8(const mmg_conv_transpose2d_fp8_args* a, void* stream);

/* Per-image e4m3 quantisation of a bf16 NHWC map x [B * hw, C] (contiguous) for the calls above:
 *   amax_b = max |x| over image b (an integer max over the bits of |x|: order-independent, bitwise reproducible);
 *   inv = amax_b == 0 ? 0 : 448 / amax_b (IEEE division);  q = cvt.rn.satfinite.e4m3(x * inv);  scale[b] = amax_b / 448
 * An all-zero image gets scale 0 and zero bytes.  C % 8 == 0, x and q 16-byte aligned, B < 65536.                 */
typedef struct {
  const void* x;           /* [B * hw, C] bf16                                                                   */
  void*       q;           /* [B * hw, C] e4m3                                                                   */
  float*      scale;       /* [B]                                                                                */
  int64_t B, hw;
  int32_t C, _pad;
} mmg_quantize_e4m3_images_args;
int mmg_quantize_e4m3_images(const mmg_quantize_e4m3_images_args* a, void* stream);

/* First encoder conv: k x k (odd k <= 9, padding k / 2; the reference default is 5), Cin = channels (<= 4), fp32 NCHW image in, NHWC act
 * out.  replaces vqgan_vae.py:231.                                                                                  */
typedef struct {
  const float* img;        /* [B, C, H, W] fp32                                                                  */
  const float* w;          /* [Cout, C, k, k] fp32 (reference layout)                                            */
  const float* bias;       /* [Cout]                                                                             */
  void*        out;        /* [B, H, W, Cout] out_dtype                                                          */
  int32_t B, C, H, W, Cout, out_dtype;
  int32_t ksize, _pad;     /* k; 0 = 5                                                                           */
} mmg_conv_in_args;
int mmg_conv_in(const mmg_conv_in_args* a, void* stream);

/* GroupNorm(groups, eps 1e-5) over NHWC, in place, optional LeakyReLU(0.1).  replaces vqgan_vae.py:257,260,272-276. */
typedef struct {
  void*        x;          /* [B, HW, C] dtype, normalised in place                                              */
  const float* gamma; const float* beta;
  int32_t B, HW, C, groups, dtype, act;
} mmg_groupnorm_args;
int mmg_groupnorm(const mmg_groupnorm_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm (eps 1e-5, gamma only — beta is a zero buffer): muse_maskgit_pytorch.py:63-70.
 *   y[r, :] = LN(x[r, :width] (+ add[:]) ) * gamma, columns >= width are written as 0 up to ldy.
 *   If x_out != NULL the (x + add) sum is also written back (fp32) — used for the constant null-CFG cross-attn term.
 *   Mean, then the centred variance, in fp32 (two passes over the row, as F.layer_norm).  width <= 4096 when x and y are 16-byte aligned,
 *   ldx and ldy are multiples of 4 (fp32 x) / 8 (bf16 x), ldy <= 4096 and, with add or x_out, width is such a multiple too; otherwise
 *   width <= 2048 (any ldy).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const void*  x;  int32_t x_dtype;  int32_t y_dtype;
  void*        y;
  const float* gamma;      /* [width]                                                                            */
  const float* add;        /* [width] or NULL                                                                    */
  float*       x_out;      /* fp32 [rows, ldx] or NULL                                                           */
  float*       zero_stats; /* optional [rows, 2]: reset to 0 (kept for callers that accumulate their own row statistics; the GEGLU
                              epilogue writes per-chunk partials and needs no reset)                                          */
  int64_t      add_from;   /* `add` / `x_out` apply to rows >= add_from only (null-CFG branch rows of a 2-branch batch)   */
  int64_t rows, width, ldx, ldy;
} mmg_layernorm_args;
int mmg_layernorm(const mmg_layernorm_args* a, void* stream);

/* Quantising LayerNorm: the fp32 x -> fp32 y of mmg_layernorm (same arithmetic, same add / x_out / add_from handling), then per row
 *   amax = max_c |y[r, c]|;  inv = amax == 0 ? 0 : 448 / amax (IEEE division);  q[r, c] = cvt.rn.satfinite.e4m3(y[r, c] * inv);
 *   row_scale[r] = amax / 448
 * so that q * row_scale ~= y; columns [width, ldy) are written as 0.  x fp32, width % 4 == 0, width <= 2048, ldx % 4 == 0, ldy % 16 == 0,
 * x, y, add 16-byte aligned.                                                                                          */
typedef struct {
  const float* x;          /* [rows, ldx] fp32                                                                   */
  void*        y;          /* [rows, ldy] e4m3                                                                   */
  float*       row_scale;  /* [rows]                                                                             */
  const float* gamma;      /* [width]                                                                            */
  const float* add;        /* [width] or NULL                                                                    */
  float*       x_out;      /* fp32 [rows, ldx] or NULL                                                           */
  int64_t      add_from;   /* `add` / `x_out` apply to rows >= add_from only                                     */
  int64_t rows, width, ldx, ldy;
} mmg_layernorm_fp8_args;
int mmg_layernorm_fp8(const mmg_layernorm_fp8_args* a, void* stream);

/* x[r, :] = token_emb[ids[r]] + pos_emb[r % n]  (fp32): muse_maskgit_pytorch.py:322-323; `copies` replicas of the
 * whole [rows, dim] block are written back to back (cond / null CFG branches share the embedding).               */
typedef struct {
  const int64_t* ids; const float* token_emb; const float* pos_emb;
  float* x; int64_t rows, n, dim; int32_t copies; int32_t use_pos;
} mmg_embed_args;
int mmg_embed(const mmg_embed_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Attention core: out[b, t, h*64:(h+1)*64] = softmax(scale * q.k^T + key_mask) v   with dh = 64.
 * q [BH, Tq, 64], k/v [BH, Tk_alloc, 64] already l2-normalised/scaled (epilogue MMG_EPI_QKV); key 0 is the null key.
 * replaces: Attend.forward / flash_attn (attend.py:66-140) + the head split/merge in Attention.forward
 * (muse_maskgit_pytorch.py:143-161).  key_mask: [B, Tk - 1] uint8 (1 = attend) or NULL: one byte per REAL key, row b at
 * key_mask + b * (Tk - 1); the null key has no byte and is always attended.  Masked logits = -FLT_MAX.
 * Precondition: the tensor-core kernels (MMG_BF16 with aligned operands, and split3) multiply zero weights by the k/v rows between Tk
 * and the end of the last 32-key chunk.  Rows [Tk, Tk_alloc) of k and v must therefore hold finite values (zeros, or stale finite
 * data): a NaN or Inf there reaches the output.  Where the padding is shorter than the chunk the rows read are the next head's, and
 * reads past the end of the tensor give zeros.  The CUDA-core kernels never read past row Tk.                        */
typedef struct {
  const void* q; const void* k; const void* v; void* out;
  const uint8_t* key_mask;
  int32_t B, heads, Tq, Tk, Tk_alloc, dtype;
  int64_t ldo;             /* out row stride (elements) = heads*64 normally                                      */
  int32_t kv_batch_stride_zero;  /* 1: k/v are shared by all batch entries (per head only)                        */
  float   scale;
  float   logit_bound;     /* optional: a guaranteed upper bound on |q.k| (for l2-normalised q, k: max_i |q_scale_i k_scale_i|);
                              > 0 lets the tensor-core kernel run a single-pass softmax against that fixed maximum. 0 = unknown. */
  int32_t split3;          /* 1 (with dtype MMG_BF16): fp32 parity on the tensor cores.  q, k, v are mmg_split3 outputs of the fp32 [.., 64] tensors
                              (384 bf16 columns per row: q with side 0, k and v with side 1), out is fp32; exact two-pass softmax.      */
} mmg_attention_args;
int mmg_attention(const mmg_attention_args* a, void* stream);
/* The same attention for 128-wide heads: q [BH, Tq, 128], k / v [BH, Tk_alloc, 128] (MMG_EPI_QKV128 outputs), out rows
 * out[b, t, h*128 : (h+1)*128]; the same argument block, same key-mask, null-key, Tk_alloc and logit_bound conventions.
 * MMG_BF16 with 16-byte aligned q / k / v / out, ldo % 8 == 0 and 2 <= Tk <= 4096 runs the wgmma kernel; fp32, and any other bf16
 * call, the CUDA-core kernel.  split3 must be 0 (no split-precision kernel at this width: fp32 runs on the CUDA cores).           */
int mmg_attention_d128(const mmg_attention_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sampler.  replaces muse_maskgit_pytorch.py:556-609 (the per-step tail of MaskGit.generate).
 * ---------------------------------------------------------------------------------------------- */
/* re-mask: select the num_masked highest scores per batch row (ties: lowest position first), write mask_id there,
 * set all scores to -1e5, and emit the ascending list of masked positions (muse_maskgit_pytorch.py:561-563).     */
typedef struct {
  int64_t* ids; float* scores; int32_t* masked_pos;   /* [B, n], [B, n], [B, num_masked]                          */
  int32_t B, n, num_masked; int64_t mask_id;
} mmg_remask_args;
int mmg_remask(const mmg_remask_args* a, void* stream);

/* re-mask with frozen positions and a count per batch row (MaskGit.inpaint).  Row b ranks the scores of its non-frozen
 * positions only (ties: lowest position first) and selects c_b = min(num_masked[b], rows) of them: mask_id is written
 * there, every score of the row is set to -1e5, masked_pos[b, 0 .. c_b) gets the ascending selected positions and
 * masked_pos[b, c_b .. rows) the row's first frozen position (pad rows).  rows is the step's largest count over the batch;
 * a row with a smaller count must have a frozen position, so that with `only_masked` the sampler computes its pad rows but
 * writes no id for them, and their scores land on a position the next re-mask ignores.  num_masked is read on the device
 * (one launch per step, no host synchronisation).                                                                      */
typedef struct {
  int64_t* ids; float* scores; int32_t* masked_pos;   /* [B, n], [B, n], [B, rows]                                 */
  const uint8_t* frozen;                              /* [B, n], 1 = keep                                          */
  const int32_t* num_masked;                          /* [B] device counts for this step, each <= rows             */
  int32_t B, n, rows; int64_t mask_id;
} mmg_remask_frozen_args;
int mmg_remask_frozen(const mmg_remask_frozen_args* a, void* stream);

/* selection of one mask-free editing iteration (MaskGit.edit).  Row b takes one uniform key per position: u[b, p] when u != NULL,
 * else Philox4x32-10(counter = (0xFFFFFFFE, iteration, row_offset + b*n + p), key = seed + *seed_dev) >> 8 * 2^-24 (disjoint from
 * the gumbel stream, c0 = vocabulary index, and the critic stream, c0 = 0xFFFFFFFF).  Among its editable positions (keep == 0)
 * it selects the num_select[b] largest keys (ties: lowest position first), writes frozen_out[b, p] = 1 at every other position
 * and 0 at the selected ones, mask_id at the selected ids and 0 into every score of the row.  A following mmg_remask_frozen
 * with frozen = frozen_out and count num_select[b] re-masks exactly the selected positions.  num_select is read on the device. */
typedef struct {
  int64_t* ids; float* scores; uint8_t* frozen_out;   /* [B, n], [B, n], [B, n] (1 = keep)                         */
  const uint8_t* keep;                                /* [B, n], 1 = not editable                                  */
  const int32_t* num_select;                          /* [B] device counts, each <= n                              */
  const float* u;                                     /* [B, n] injected keys or NULL                              */
  uint64_t seed; const uint64_t* seed_dev;            /* seed_dev optional, as in mmg_logits_sample_args          */
  int64_t row_offset;                                 /* global position of this call's first token                */
  int32_t B, n, iteration, _pad; int64_t mask_id;
} mmg_edit_select_args;
int mmg_edit_select(const mmg_edit_select_args* a, void* stream);

/* Final LayerNorm + classifier-free-guidance combine on the masked rows only, in embedding space:
 *   e[j] = LN(x_null[r]) + (LN(x_cond[r]) - LN(x_null[r])) * cond_scale,  r = b*n + masked_pos[b, j]
 * (to_logits is linear and bias-free, so W e == null + (cond - null) * scale of muse_maskgit_pytorch.py:254).
 * cond_scale_dev != NULL: image b combines at cond_scale_dev[b] instead, and an image whose scale is exactly 1 takes LN(x_cond)
 * alone without reading x_null (bitwise the x_null == NULL launch).                                                 */
typedef struct {
  const float* x_cond; const float* x_null;  /* [B*n, dim] fp32; x_null may be NULL (cond_scale == 1)             */
  const float* gamma; const int32_t* masked_pos;
  void* e; int32_t e_dtype;
  int32_t B, n, num_masked, dim; float cond_scale;
  const float* cond_scale_dev;               /* [B] per-image scales or NULL (use cond_scale)                     */
} mmg_final_embed_args;
int mmg_final_embed(const mmg_final_embed_args* a, void* stream);

/* top-k filter + gumbel-argmax + confidence score for R logits rows (muse_maskgit_pytorch.py:576-609, 403-418):
 *   keep the k largest logits of each row (ties at the threshold: lowest index first);
 *   pred = argmax_v( logit_v / max(T, 1e-10) - log(-log(u_v)) ),   u clamped at 1e-20 as the reference's log();
 *   score = 1 - softmax(logits)[pred];  ids[b, pos] = pred;  scores[b, pos] = score.
 * Noise: `u` != NULL -> injected uniforms, u[(b*n + pos) * V + v] (parity mode: the tensor the reference would
 * draw); else Philox4x32-10(seed, counter = (global row, v)) so results do not depend on the GPU count.          */
typedef struct {
  const float* logits;     /* [R, V] fp32, R = B*num_masked, row j of batch b at b*num_masked + j                  */
  const int32_t* masked_pos;
  int64_t* ids; float* scores;             /* [B, n]                                                              */
  const float* u;          /* [B, n, V] or NULL                                                                   */
  int32_t B, n, num_masked, V, k;
  float temperature;
  uint64_t seed; uint64_t step; int64_t row_offset;  /* global row = row_offset + b*n + pos                        */
  const uint64_t* seed_dev;  /* optional device word added to `seed` at run time (lets a captured CUDA graph be replayed
                                with a fresh seed)                                                                   */
  int64_t mask_id; int32_t only_masked;         /* only_masked != 0: ids[b, pos] is replaced only where it equals mask_id (the
                                `where(is_mask, pred_ids, ids)` of :582-588 when rows of already-decoded positions are scored
                                too, can_remask_prev_masked = True); scores are written for every listed row              */
  int32_t rng_mode;          /* u == NULL only.  0: the keying above.  1: the stream ATen's CUDA `zeros_like(t).uniform_(0, 1)` draws
                                for the reference's [B_global, n, V] noise tensor (muse_maskgit_pytorch.py:407) from a generator with
                                seed (seed + *seed_dev) and offset (aten_offset + *aten_offset_dev): element i = t + aten_stride*k is
                                word k&3 of Philox(counter = offset/4 + k/4, subsequence = t) * 2^-32 + 2^-33, 1 -> 0; aten_stride =
                                256 * min(SMs * maxThreadsPerSM/256, ceil(numel/256)); accurate logf / IEEE division as with `u`  */
  uint64_t aten_offset; const uint64_t* aten_offset_dev; uint32_t aten_stride, _pad;
  /* optional row indirection (the fallback leg of mmg_logits_fused): logits row j belongs to sampled row row_index[j] (the index into
     masked_pos), only the first min(*row_count_dev, row_index_cap) rows are processed; the grid is row_index_cap CTAs               */
  const int32_t* row_index; const int32_t* row_count_dev; int32_t row_index_cap, _pad2;
  const float* temperature_dev;  /* [B] per-image temperatures or NULL (use `temperature`): sampled row j of image b = j / num_masked
                                    divides by max(temperature_dev[b], 1e-10)                                                       */
} mmg_logits_sample_args;
int mmg_logits_sample(const mmg_logits_sample_args* a, void* stream);

/* to_logits + the sampling tail of a decode step in one call, WITHOUT a [rows, V] logits buffer (muse_maskgit_pytorch.py:576-609 on the rows
 * listed in s.masked_pos; bf16 operands, wgmma): a 4096-column sample GEMM gives every row a candidate threshold, the logits GEMM's epilogue
 * keeps online-softmax partials and emits only the candidates >= threshold (~12 % of the logits) as per-row lists, a finishing kernel runs the
 * exact-rank perturbed argmax of mmg_logits_sample on the lists.  Rows whose threshold missed are redone through materialised logits inside the
 * same call (<= 128 rows per call; beyond that status[1] is raised and the caller must repeat the step with mmg_linear + mmg_logits_sample).
 * Same results as mmg_linear + mmg_logits_sample up to the summation order of the softmax denominator.                                        */
typedef struct {
  const void* e;           /* [rows, K] bf16: mmg_final_embed output, rows = s.B * s.num_masked                                 */
  const void* w;           /* [V, K] bf16 to_logits weight                                                                        */
  int32_t K, _pad;
  int64_t rows_capacity;   /* the R_max the workspace was sized for (0: rows of this call)                                        */
  mmg_logits_sample_args s;/* sampler arguments as for mmg_logits_sample; s.logits / s.row_index are ignored                      */
  void* workspace; uint64_t workspace_bytes;   /* >= mmg_logits_fused_workspace_bytes(rows_capacity, V, K, k), 256-byte aligned   */
  int32_t* status;         /* device int32[2], zeroed by the caller: [0] += rows redone through the materialised fallback,
                              [1] = 1 when a step had more such rows than the fallback holds (results of that step are incomplete)  */
} mmg_logits_fused_args;
/* 0 when the shape is not supported by the fused path (V % 256, V < 1024, K % 64, k too large for the candidate lists) */
uint64_t mmg_logits_fused_workspace_bytes(int64_t rows_capacity, int32_t V, int32_t K, int32_t k);
int mmg_logits_fused(const mmg_logits_fused_args* a, void* stream);

/* Cross-entropy of the labelled rows of MaskGit.forward (muse_maskgit_pytorch.py:335, 717-726) without a [rows, V] logits buffer:
 *   nll[r] = logsumexp_v(e_r . W_v) - e_r . W_labels[r]   (fp32; bf16 operands, wgmma)
 * The logits GEMM of mmg_logits_fused runs with an epilogue that keeps, per (row, split of the vocabulary, 64-column half), the
 * online-softmax partials (max, sum of exp) and the logit at the label column; a second kernel merges a row's records in split order,
 * so the result is bitwise the same on every run.  Labels must lie in [0, V) (a row whose label lies outside gets NaN).             */
typedef struct {
  const void* e;           /* [rows, K] bf16: final-LayerNormed embeddings of the labelled rows                                 */
  const void* w;           /* [V, K] bf16 to_logits weight                                                                        */
  const int32_t* labels;   /* [rows]                                                                                              */
  float* nll;              /* [rows] out                                                                                          */
  int64_t rows, rows_capacity;   /* rows_capacity: the row count the workspace was sized for (0: rows)                            */
  int32_t V, K;
  void* workspace; uint64_t workspace_bytes;   /* >= mmg_logits_xent_workspace_bytes(rows_capacity, V, K), 256-byte aligned        */
} mmg_logits_xent_args;
/* 0 when the shape is not supported by the fused path (V % 128, K % 64, K < 64): mmg_logits_xent then returns MMG_EINVAL */
uint64_t mmg_logits_xent_workspace_bytes(int64_t rows_capacity, int32_t V, int32_t K);
int mmg_logits_xent(const mmg_logits_xent_args* a, void* stream);

/* The same nll from materialised fp32 logits rows (precision="fp32", shapes mmg_logits_xent does not take, the token-critic branch of
 * MaskGit.forward): one CTA per row, a fixed reduction order.  A label outside [0, V) gives NaN.                                    */
typedef struct {
  const float* logits;     /* [rows, ld] fp32                                                                                     */
  int64_t ld;
  const int32_t* labels;   /* [rows]                                                                                              */
  float* nll;              /* [rows] out                                                                                          */
  int64_t rows; int32_t V, _pad;
} mmg_logits_xent_rows_args;
int mmg_logits_xent_rows(const mmg_logits_xent_rows_args* a, void* stream);

/* token-critic scoring branch of MaskGit.generate (muse_maskgit_pytorch.py:590-600; TokenCritic :383-386, SelfCritic :352-361):
 *   s[r] = dot(LayerNorm(x_cond[r]) * gamma, w) + bias;   x_null != NULL: s = s_null + (s - s_null) * cond_scale  (CFG, :257)
 *   scores[r] = s + (u[r] - 0.5) * noise_mul       noise_mul = critic_noise_scale * steps_until_x0 / timesteps
 * x_* are the residual streams after the critic's last block (the final LayerNorm and the 1-wide head are applied here).
 * u == NULL: u = Philox4x32-10(counter = (0xFFFFFFFF, step, row_offset + r), key = seed + *seed_dev) >> 8 * 2^-24.
 * cond_scale_dev / noise_mul_dev != NULL: row r reads its scale / noise multiplier from them instead of the scalars (a host expands
 * per-image settings over the image's rows); a row whose scale is exactly 1 keeps s from x_cond alone, as the x_null == NULL launch. */
typedef struct {
  const float* x_cond; const float* x_null;   /* [rows, dim] fp32; x_null may be NULL (cond_scale == 1, SelfCritic)   */
  const float* gamma; const float* w;         /* [dim] final LayerNorm gain, [dim] head weight (to_logits / to_pred)  */
  float bias, cond_scale, noise_mul; int32_t dim;
  const float* u;                             /* [rows] injected uniforms or NULL                                     */
  float* scores;                              /* [rows] out                                                           */
  int64_t rows, row_offset; uint64_t seed; const uint64_t* seed_dev; int32_t step;
  int32_t rng_mode;                           /* 1: ATen's `uniform(scores.shape)` stream (:598), see mmg_logits_sample_args */
  uint64_t aten_offset; const uint64_t* aten_offset_dev; uint32_t aten_stride, _pad;
  const float* cond_scale_dev; const float* noise_mul_dev;   /* [rows] per-row values or NULL (use cond_scale / noise_mul)      */
} mmg_critic_score_args;
int mmg_critic_score(const mmg_critic_score_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * VQ lookup.  replaces the quantizer calls at vqgan_vae.py:424 and 429-435.
 * ---------------------------------------------------------------------------------------------- */
/* LFQ: ids[t] = sum_i (x[t,:].w_in[i,:] + b_in[i] > 0) << (bits-1-i)  — the nearest-codebook L2 argmin over {+-1}^bits. */
typedef struct {
  const void* x; int32_t dtype;            /* [T, D] token-major fmap                                              */
  const float* w_in; const float* b_in;    /* [bits, D], [bits]; NULL -> identity (D == bits)                     */
  int64_t* ids; int64_t T; int32_t D, bits;
  const void* w_split;                     /* optional, bf16 tokens: [64, D] bf16, rows [hi(bits) | mid(bits) | lo(bits) | 0...] = the 3-way bf16
                                              split of w_in (hi + mid + lo == w_in in fp32; 3 * bits <= 64, D % 64 == 0): the projection then
                                              runs on the wgmma path (mmg_linear + MMG_EPI_LFQ_IDS), one TMA stream over the tokens      */
} mmg_vq_lfq_encode_args;
int mmg_vq_lfq_encode(const mmg_vq_lfq_encode_args* a, void* stream);

/* explicit codebook: ids[t] = argmin_k ||x_t - e_k||^2 (first index on ties); 64x64 tiles staged through shared memory with
 * coalesced loads, per-row packed (distance, code) atomicMin across code tiles.  (Large problems: mmg_linear + MMG_EPI_ARGMIN.) */
typedef struct {
  const float* x; const float* codebook;   /* [T, D], [K, D] fp32                                                  */
  int64_t* ids; int64_t T; int32_t K, D;
} mmg_vq_l2_argmin_args;
int mmg_vq_l2_argmin(const mmg_vq_l2_argmin_args* a, void* stream);

/* ids -> codes -> project_out: out[t, :] = sum_i (+-1)_i * w_out[:, i] + b_out  (LFQ.indices_to_codes)            */
typedef struct {
  const int64_t* ids; const float* w_out; const float* b_out;   /* w_out [D, bits]                                 */
  void* out; int32_t dtype; int64_t T; int32_t D, bits;
} mmg_vq_decode_codes_args;
int mmg_vq_decode_codes(const mmg_vq_decode_codes_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Composite entry points: the launch sequences of one FeedForward and of one whole decode step, for hosts that want one call
 * per step.  They only issue the entry points above on `stream` (no allocation, no host sync, CUDA-graph capturable).
 * ---------------------------------------------------------------------------------------------- */
/* FeedForward of a block on `rows` rows, in place on the fp32 residual stream (muse_maskgit_pytorch.py:72-89), bf16 operands:
 *   xn = LN(x [+ add on rows >= add_from, written back]) * ln_gamma;  h = gate * gelu_erf(xn W1^T);  x += LN(h) * gamma_inner W2^T
 * (the inner LayerNorm is folded through the second product: w2f = W2 * gamma_inner, cvec = rowsum(w2f), MMG_EPI_LNFOLD_RESIDUAL). */
typedef struct {
  float* x; int64_t rows; int32_t dim, F, Fp;     /* x [rows, dim]; F = inner width int(dim*mult*2/3), Fp = F padded to a multiple of 64 */
  const float* ln_gamma;                          /* [dim]                                                                  */
  const void* w1;                                 /* [2*Fp, dim] bf16, rows interleaved in blocks of 32: [x(32) | gate(32)] */
  const void* w2f; const float* cvec;             /* [dim, Fp] bf16, [dim]                                                  */
  const float* add; int64_t add_from;             /* optional [dim] constant (to_out(null_v) of an all-masked cross-attention) */
  void* xn; void* h; float* stats;                /* workspace: [rows, dim] bf16, [rows, Fp] bf16, [rows, Fp / 32, 2] fp32   */
} mmg_ff_geglu_args;
int mmg_ff_geglu(const mmg_ff_geglu_args* a, void* stream);

/* One step of MaskGit.generate (muse_maskgit_pytorch.py:556-609) for the default path (bf16, no token critic, no self-conditioning):
 * re-mask -> embed -> depth x [self-attention, cross-attention, FeedForward] over `branches` copies of the batch (1, or 2 = cond + null
 * CFG; the first `live_branches` attend to the context, the others take the constant to_out(null_v)) -> final LayerNorm + CFG combine
 * on the masked rows -> logits GEMM -> top-k / gumbel argmax / confidence.  ids / scores / masked_pos are updated in place. */
typedef struct {
  const float* ln_gamma; const void* w_qkv;       /* self: [3*heads*64, dim]; cross: [heads*64, dim] (q only)                */
  const void* w_out;                              /* [dim, heads*64]                                                         */
  const float* q_scale; const float* k_scale;     /* [64]; k_scale, null_k, null_v: self-attention only                      */
  const void* null_k; const void* null_v;         /* [heads, 64] bf16: l2norm(null_k)*k_scale, null_v                        */
  float logit_bound; int32_t _pad;                /* max_i |q_scale_i k_scale_i| (+ slack), see mmg_attention_args           */
} mmg_attn_weights;
typedef struct {
  mmg_attn_weights self_attn, cross_attn;
  const void* ctx_k; const void* ctx_v;           /* this layer's context K/V [live*b*heads, ctx_alloc, 64] bf16 (null key at row 0), computed
                                                     once per generate() with mmg_linear + MMG_EPI_QKV                       */
  const float* cross_null_out;                    /* [dim] to_out(null_v)                                                    */
  const float* ff_ln_gamma; const void* ff_w1; const void* ff_w2f; const float* ff_cvec;
} mmg_layer_weights;
typedef struct {
  int32_t depth, dim, heads, n, V, F, Fp, b, branches, live_branches;
  const mmg_layer_weights* layers;                /* HOST array [depth]                                                      */
  const float* tok_emb; const float* pos_emb; const float* final_gamma; const void* w_logits;   /* fp32, fp32, fp32, [V, dim] bf16 */
  const uint8_t* ctx_key_mask; int32_t ctx_keys, ctx_alloc;   /* [live*b, ctx_keys] (1 = attend); keys incl. the null key = ctx_keys + 1 */
  int64_t* ids; float* scores; int32_t* masked_pos; int64_t mask_id;     /* [b, n], [b, n], [b, n] */
  int32_t num_masked, k_keep, step; float temperature, cond_scale; int32_t _pad;
  const float* u; uint64_t seed; const uint64_t* seed_dev; int64_t row_offset;   /* noise: see mmg_logits_sample_args        */
  void* workspace; uint64_t workspace_bytes;      /* >= mmg_decode_step_workspace_bytes(...), 256-byte aligned, ZERO-INITIALISED once by
                                                     the caller (the padding rows of the self-attention K/V stay zero)        */
  const float* cond_scale_dev; const float* temperature_dev;   /* [b] per-image settings or NULL (use cond_scale / temperature): passed
                                                     to mmg_final_embed_args.cond_scale_dev / mmg_logits_sample_args.temperature_dev */
} mmg_decode_step_args;
uint64_t mmg_decode_step_workspace_bytes(int32_t b, int32_t branches, int32_t n, int32_t dim, int32_t heads, int32_t Fp, int32_t V, int32_t max_masked);
int mmg_decode_step(const mmg_decode_step_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * T5 text encoder (HF T5EncoderModel, eval mode; the text step of MaskGit.generate, t5.py:60-99).
 * ---------------------------------------------------------------------------------------------- */
/* T5 self-attention with d_kv = 64:  out[b*T + i, h*64 : h*64+64] = softmax_j( q_i . k_j + rel_bias[rel_bucket[j - i + T - 1], h] + m_j ) v_j
 * over the T keys of sequence b: no 1/sqrt(d) scaling, m_j = 0 for a live key and -FLT_MAX (finfo(fp32).min) for a masked one, softmax in fp32
 * (a row with no live key gets uniform weights over the T keys, as in HF).  q, k, v are read straight from the token-major output of one
 * fused [3*heads*64, d_model] projection: row b*T + t = [q (heads*64) | k (heads*64) | v (heads*64)].
 * dtype MMG_BF16: wgmma kernel (TMA loads, exact two-pass softmax, bias staged per CTA in shared memory); MMG_F32: CUDA-core fp32 kernel.  */
typedef struct {
  const void*    qkv;        /* [B*T, ldqkv] of dtype                                                                   */
  void*          out;        /* [B*T, ldo] of dtype                                                                     */
  const uint8_t* key_mask;   /* [B, T] (1 = attend) or NULL                                                             */
  const int32_t* rel_bucket; /* [2T-1] int32: bucket of the relative position key - query, at index key - query + T - 1 */
  const float*   rel_bias;   /* [num_buckets, heads] fp32 (relative_attention_bias.weight as stored)                    */
  int32_t B, T, heads, num_buckets, dtype, _pad;  /* T <= 512                                                           */
  int64_t ldqkv, ldo;        /* row strides (elements); ldqkv >= 3*heads*64                                             */
} mmg_t5_attention_args;
int mmg_t5_attention(const mmg_t5_attention_args* a, void* stream);

/* T5 RMSNorm (T5LayerNorm): y[r, :] = w * (x[r, :] * rsqrt(mean(x[r, :]^2) + eps)), statistics in fp32, no mean, no bias;
 * rows with row_mask[r] == 0 are written as zeros (the padding zero-fill of t5_encode_text).                          */
typedef struct {
  const float*   x;          /* [rows, ldx] fp32                                                                        */
  void*          y;          /* [rows, ldy] of y_dtype                                                                  */
  const float*   w;          /* [d]                                                                                     */
  const uint8_t* row_mask;   /* [rows] or NULL                                                                          */
  int64_t rows, d, ldx, ldy;
  float   eps; int32_t y_dtype;
} mmg_rmsnorm_args;
int mmg_rmsnorm(const mmg_rmsnorm_args* a, void* stream);

/* dtype conversion / layout helpers used by the host mirror */
typedef struct { const void* src; void* dst; int64_t n; int32_t src_dtype, dst_dtype; } mmg_cast_args;
int mmg_cast(const mmg_cast_args* a, void* stream);

/* fp32 on the tensor cores (precision="fp32"): dst[r, 6K] bf16 = the hi / mid / lo bf16 terms of src[r, K] (hi + mid + lo == src to 24 bits),
 * ordered per `side` (0: left operand [lo|hi|mid|mid|hi|hi], 1: right operand [hi|lo|mid|hi|mid|hi]) so that one bf16 product of the two
 * 6K-wide operands accumulates lo*hi + hi*lo + mid*mid + mid*hi + hi*mid + hi*hi in fp32 = the fp32 product to ~2^-24.  An NHWC activation
 * is split per pixel (rows = B*H*W, K = Cin -> 6*Cin channels), a packed conv weight per (output channel, tap).
 * replaces: the fp32 arithmetic of nn.Linear / nn.Conv2d when parity with the fp32 reference is asked for (no reference counterpart). */
typedef struct { const float* src; void* dst; int64_t rows, K, lds; int32_t side, _pad; } mmg_split3_args;
int mmg_split3(const mmg_split3_args* a, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MMG_H_ */

// mmg_ff_geglu / mmg_decode_step: the launch sequences of one FeedForward and of one whole MaskGit decode step, composed from the
// entry points of this library on the caller's stream (no allocation, no host synchronisation, CUDA-graph capturable), so a host in
// any language drives the path with one call per step.  The Python mirror issues the same sequence call by call
// (muse_maskgit.py: Transformer._run_blocks / MaskGit._generate_body); tests/test_gpu_models.py checks the two are bit-identical.
#include "mmg_common.cuh"

using namespace mmg;

namespace {
inline uint64_t up256(uint64_t x) { return (x + 255) & ~uint64_t(255); }
inline int32_t round8(int32_t x) { return (x + 7) / 8 * 8; }

struct StepWs {            // carve-up of the decode-step workspace (all offsets 256-byte aligned)
  uint64_t x, xn, q, k, v, ao, h, stats, e, logits, total;
};
StepWs carve(int32_t b, int32_t branches, int32_t n, int32_t dim, int32_t heads, int32_t Fp, int32_t V, int32_t max_masked) {
  const uint64_t R = (uint64_t)branches * b * n, BH = (uint64_t)branches * b * heads, inner = (uint64_t)heads * 64, tk = round8(n + 1);
  StepWs w{}; uint64_t o = 0;
  w.x = o;      o += up256(R * dim * 4);
  w.xn = o;     o += up256(R * dim * 2);
  w.q = o;      o += up256(BH * n * 64 * 2);
  w.k = o;      o += up256(BH * tk * 64 * 2);
  w.v = o;      o += up256(BH * tk * 64 * 2);
  w.ao = o;     o += up256(R * inner * 2);
  w.h = o;      o += up256(R * (uint64_t)Fp * 2);
  w.stats = o;  o += up256(R * (uint64_t)(Fp / 32) * 2 * 4);
  w.e = o;      o += up256((uint64_t)b * n * dim * 2);
  w.logits = o; o += up256((uint64_t)b * max_masked * V * 4);
  w.total = o;
  return w;
}

int linear_bf16(const void* a, const void* w, int64_t M, int64_t N, int64_t K, int epilogue, const mmg_epilogue_args& epi, void* stream) {
  mmg_linear_args l{};
  l.a = a; l.w = w; l.M = M; l.N = N; l.K = K; l.lda = K; l.ldw = K; l.dtype = MMG_BF16; l.epilogue = epilogue; l.epi = epi;
  return mmg_linear(&l, stream);
}
}  // namespace

extern "C" int mmg_ff_geglu(const mmg_ff_geglu_args* a, void* stream) {
  MMG_CHECK_ARG(a && a->x && a->ln_gamma && a->w1 && a->w2f && a->cvec && a->xn && a->h && a->stats, "mmg_ff_geglu: NULL pointer");
  MMG_CHECK_ARG(a->rows >= 0 && a->dim > 0 && a->F > 0 && a->Fp >= a->F && a->Fp % 64 == 0 && a->dim % 64 == 0, "mmg_ff_geglu: dim=%d F=%d Fp=%d", a->dim, a->F, a->Fp);
  if (a->rows == 0) return MMG_OK;
  int rc;
  {   // xn = LN(x [+ add]) * gamma
    mmg_layernorm_args ln{};
    ln.x = a->x; ln.x_dtype = MMG_F32; ln.y = a->xn; ln.y_dtype = MMG_BF16; ln.gamma = a->ln_gamma;
    ln.add = a->add; ln.x_out = a->add ? a->x : nullptr; ln.add_from = a->add ? a->add_from : 0;
    ln.rows = a->rows; ln.width = a->dim; ln.ldx = a->dim; ln.ldy = a->dim;
    if ((rc = mmg_layernorm(&ln, stream))) return rc;
  }
  {   // h = gate * gelu(x); the epilogue writes the (sum, sumsq) of every 32-output chunk of h to its own slot
    mmg_epilogue_args e{};
    e.out = a->h; e.ldo = a->Fp; e.out_dtype = MMG_BF16; e.row_stats = a->stats; e.stats_slots = a->Fp / 32;
    if ((rc = linear_bf16(a->xn, a->w1, a->rows, 2 * (int64_t)a->Fp, a->dim, MMG_EPI_GEGLU, e, stream))) return rc;
  }
  {   // x += LN(h) * gamma_inner W2^T, LayerNorm folded through the product
    mmg_epilogue_args e{};
    e.out = a->x; e.ldo = a->dim; e.out_dtype = MMG_F32; e.resid = a->x; e.ldr = a->dim; e.bias = a->cvec; e.row_stats = a->stats; e.stats_slots = a->Fp / 32; e.ln_width = a->F;
    if ((rc = linear_bf16(a->h, a->w2f, a->rows, a->dim, a->Fp, MMG_EPI_LNFOLD_RESIDUAL, e, stream))) return rc;
  }
  return MMG_OK;
}

extern "C" uint64_t mmg_decode_step_workspace_bytes(int32_t b, int32_t branches, int32_t n, int32_t dim, int32_t heads, int32_t Fp, int32_t V,
                                                     int32_t max_masked) {
  if (b <= 0 || branches <= 0 || n <= 0 || dim <= 0 || heads <= 0 || Fp <= 0 || V <= 0 || max_masked <= 0) return 0;
  return carve(b, branches, n, dim, heads, Fp, V, max_masked).total;
}

extern "C" int mmg_decode_step(const mmg_decode_step_args* a, void* stream) {
  MMG_CHECK_ARG(a && a->layers && a->tok_emb && a->pos_emb && a->final_gamma && a->w_logits && a->ids && a->scores && a->masked_pos && a->workspace,
                "mmg_decode_step: NULL pointer");
  MMG_CHECK_ARG(a->depth > 0 && a->dim % 64 == 0 && a->heads > 0 && a->n > 0 && a->b > 0 && (a->branches == 1 || a->branches == 2) &&
                a->live_branches >= 0 && a->live_branches <= a->branches && a->num_masked >= 1 && a->num_masked <= a->n,
                "mmg_decode_step: depth=%d dim=%d heads=%d n=%d b=%d branches=%d live=%d num_masked=%d", a->depth, a->dim, a->heads, a->n, a->b,
                a->branches, a->live_branches, a->num_masked);
  MMG_CHECK_ARG(a->live_branches == 0 || (a->layers[0].ctx_k && a->layers[0].ctx_v && a->ctx_alloc >= a->ctx_keys + 1), "mmg_decode_step: context K/V");
  const StepWs w = carve(a->b, a->branches, a->n, a->dim, a->heads, a->Fp, a->V, a->num_masked);
  MMG_CHECK_ARG(a->workspace_bytes >= w.total, "mmg_decode_step: workspace %llu < %llu bytes", (unsigned long long)a->workspace_bytes, (unsigned long long)w.total);
  MMG_CHECK_ARG((reinterpret_cast<uintptr_t>(a->workspace) & 255) == 0, "mmg_decode_step: workspace must be 256-byte aligned");
  uint8_t* base = static_cast<uint8_t*>(a->workspace);
  float* x = reinterpret_cast<float*>(base + w.x);
  void *xn = base + w.xn, *q = base + w.q, *k = base + w.k, *v = base + w.v, *ao = base + w.ao, *h = base + w.h, *e = base + w.e;
  float* stats = reinterpret_cast<float*>(base + w.stats);
  float* logits = reinterpret_cast<float*>(base + w.logits);
  const int64_t bn = (int64_t)a->b * a->n, R = a->branches * bn, Rl = a->live_branches * bn;
  const int32_t inner = a->heads * 64, tk = round8(a->n + 1);
  int rc;

  {   // re-mask the num_masked least confident positions (muse_maskgit_pytorch.py:561-563)
    mmg_remask_args r{}; r.ids = a->ids; r.scores = a->scores; r.masked_pos = a->masked_pos; r.B = a->b; r.n = a->n; r.num_masked = a->num_masked; r.mask_id = a->mask_id;
    if ((rc = mmg_remask(&r, stream))) return rc;
  }
  {   // token + position embedding, one copy per CFG branch (:322-323)
    mmg_embed_args m{}; m.ids = a->ids; m.token_emb = a->tok_emb; m.pos_emb = a->pos_emb; m.x = x; m.rows = bn; m.n = a->n; m.dim = a->dim; m.copies = a->branches; m.use_pos = 1;
    if ((rc = mmg_embed(&m, stream))) return rc;
  }
  for (int32_t li = 0; li < a->depth; ++li) {
    const mmg_layer_weights& L = a->layers[li];
    // ---- self attention over every branch (:187-189, 91-162) ----
    { mmg_layernorm_args ln{}; ln.x = x; ln.x_dtype = MMG_F32; ln.y = xn; ln.y_dtype = MMG_BF16; ln.gamma = L.self_attn.ln_gamma; ln.rows = R; ln.width = a->dim; ln.ldx = a->dim; ln.ldy = a->dim;
      if ((rc = mmg_layernorm(&ln, stream))) return rc; }
    { mmg_epilogue_args ep{}; ep.out_dtype = MMG_BF16; ep.heads = a->heads; ep.tokens = a->n; ep.key_off = 1;
      ep.q_out = q; ep.q_scale = L.self_attn.q_scale; ep.q_rows = a->n; ep.nq_heads = a->heads;
      ep.k_out = k; ep.k_scale = L.self_attn.k_scale; ep.kv_rows = tk; ep.nk_heads = a->heads; ep.v_out = v; ep.nv_heads = a->heads;
      ep.null_k = L.self_attn.null_k; ep.null_v = L.self_attn.null_v;
      if ((rc = linear_bf16(xn, L.self_attn.w_qkv, R, 3 * (int64_t)inner, a->dim, MMG_EPI_QKV, ep, stream))) return rc; }
    { mmg_attention_args at{}; at.q = q; at.k = k; at.v = v; at.out = ao; at.B = a->branches * a->b; at.heads = a->heads; at.Tq = a->n; at.Tk = a->n + 1; at.Tk_alloc = tk;
      at.dtype = MMG_BF16; at.ldo = inner; at.scale = 8.0f; at.logit_bound = L.self_attn.logit_bound;
      if ((rc = mmg_attention(&at, stream))) return rc; }
    { mmg_epilogue_args ep{}; ep.out = x; ep.ldo = a->dim; ep.out_dtype = MMG_F32; ep.resid = x; ep.ldr = a->dim;
      if ((rc = linear_bf16(ao, L.self_attn.w_out, R, a->dim, inner, MMG_EPI_RESIDUAL, ep, stream))) return rc; }
    // ---- cross attention: only the branches that still see context keys (:190-191) ----
    if (Rl > 0) {
      { mmg_layernorm_args ln{}; ln.x = x; ln.x_dtype = MMG_F32; ln.y = xn; ln.y_dtype = MMG_BF16; ln.gamma = L.cross_attn.ln_gamma; ln.rows = Rl; ln.width = a->dim; ln.ldx = a->dim; ln.ldy = a->dim;
        if ((rc = mmg_layernorm(&ln, stream))) return rc; }
      { mmg_epilogue_args ep{}; ep.out_dtype = MMG_BF16; ep.heads = a->heads; ep.tokens = a->n; ep.key_off = 0;
        ep.q_out = q; ep.q_scale = L.cross_attn.q_scale; ep.q_rows = a->n; ep.nq_heads = a->heads;
        if ((rc = linear_bf16(xn, L.cross_attn.w_qkv, Rl, inner, a->dim, MMG_EPI_QKV, ep, stream))) return rc; }
      { mmg_attention_args at{}; at.q = q; at.k = L.ctx_k; at.v = L.ctx_v; at.out = ao; at.key_mask = a->ctx_key_mask; at.B = a->live_branches * a->b; at.heads = a->heads;
        at.Tq = a->n; at.Tk = a->ctx_keys + 1; at.Tk_alloc = a->ctx_alloc; at.dtype = MMG_BF16; at.ldo = inner; at.scale = 8.0f; at.logit_bound = L.cross_attn.logit_bound;
        if ((rc = mmg_attention(&at, stream))) return rc; }
      { mmg_epilogue_args ep{}; ep.out = x; ep.ldo = a->dim; ep.out_dtype = MMG_F32; ep.resid = x; ep.ldr = a->dim;
        if ((rc = linear_bf16(ao, L.cross_attn.w_out, Rl, a->dim, inner, MMG_EPI_RESIDUAL, ep, stream))) return rc; }
    }
    // ---- feed forward; rows of an all-masked (null CFG) branch first receive their constant cross-attention term to_out(null_v) ----
    { mmg_ff_geglu_args f{}; f.x = x; f.rows = R; f.dim = a->dim; f.F = a->F; f.Fp = a->Fp; f.ln_gamma = L.ff_ln_gamma; f.w1 = L.ff_w1; f.w2f = L.ff_w2f; f.cvec = L.ff_cvec;
      if (a->live_branches < a->branches) { f.add = L.cross_null_out; f.add_from = Rl; MMG_CHECK_ARG(f.add, "mmg_decode_step: cross_null_out is NULL"); }
      f.xn = xn; f.h = h; f.stats = stats;
      if ((rc = mmg_ff_geglu(&f, stream))) return rc; }
  }
  {   // final LayerNorm + CFG combine in embedding space, masked rows only (:195, 254)
    mmg_final_embed_args f{}; f.x_cond = x; f.x_null = a->branches == 2 ? x + bn * a->dim : nullptr; f.gamma = a->final_gamma; f.masked_pos = a->masked_pos; f.e = e; f.e_dtype = MMG_BF16;
    f.B = a->b; f.n = a->n; f.num_masked = a->num_masked; f.dim = a->dim; f.cond_scale = a->cond_scale; f.cond_scale_dev = a->cond_scale_dev;
    if ((rc = mmg_final_embed(&f, stream))) return rc;
  }
  const int64_t Rm = (int64_t)a->b * a->num_masked;
  { mmg_epilogue_args ep{}; ep.out = logits; ep.ldo = a->V; ep.out_dtype = MMG_F32;
    if ((rc = linear_bf16(e, a->w_logits, Rm, a->V, a->dim, MMG_EPI_STORE, ep, stream))) return rc; }
  {   // top-k filter + gumbel argmax + confidence (:576-609)
    mmg_logits_sample_args s{}; s.logits = logits; s.masked_pos = a->masked_pos; s.ids = a->ids; s.scores = a->scores; s.u = a->u;
    s.B = a->b; s.n = a->n; s.num_masked = a->num_masked; s.V = a->V; s.k = a->k_keep; s.temperature = a->temperature; s.temperature_dev = a->temperature_dev; s.image_seed = a->image_seed; s.k_dev = a->k_dev;
    s.seed = a->seed; s.step = (uint64_t)a->step; s.row_offset = a->row_offset; s.seed_dev = a->seed_dev;
    if ((rc = mmg_logits_sample(&s, stream))) return rc;
  }
  return MMG_OK;
}

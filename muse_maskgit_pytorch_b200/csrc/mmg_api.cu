// Library-level entry points of libmmg.so.
#include "mmg_common.cuh"

extern "C" int mmg_version(void) { return MMG_VERSION; }
extern "C" const char* mmg_last_error(void) { return mmg::err_buf(); }
extern "C" int64_t mmg_launch_count(void) { return mmg::launch_counter().load(); }
extern "C" int64_t mmg_simt_fallback_count(void) { return mmg::simt_fallback_counter().load(); }
extern "C" int64_t mmg_simt_launch_count(void) { return mmg::simt_launch_counter().load(); }

// ABI self-check for language bindings: size of an argument block by entry-point name (0 if unknown).
#include <string.h>
extern "C" int mmg_sizeof(const char* name) {
#define SZ(n) if (!strcmp(name, "mmg_" #n)) return (int)sizeof(mmg_##n##_args)
  SZ(linear); SZ(conv2d); SZ(conv_transpose2d); SZ(conv_in); SZ(groupnorm); SZ(layernorm); SZ(embed); SZ(attention);
  SZ(remask); SZ(final_embed); SZ(logits_sample); SZ(vq_lfq_encode); SZ(vq_l2_argmin); SZ(vq_decode_codes); SZ(cast); SZ(split3); SZ(critic_score); SZ(ff_geglu); SZ(decode_step); SZ(logits_fused);
  SZ(t5_attention); SZ(rmsnorm); SZ(remask_frozen); SZ(edit_select); SZ(extrapolate_window); SZ(logits_xent); SZ(logits_xent_rows); SZ(linear_fp8); SZ(layernorm_fp8);
  SZ(conv2d_fp8); SZ(conv_transpose2d_fp8); SZ(quantize_e4m3_images);
#undef SZ
  if (!strcmp(name, "mmg_attention_d128")) return (int)sizeof(mmg_attention_args);
  if (!strcmp(name, "mmg_epilogue")) return (int)sizeof(mmg_epilogue_args);
  if (!strcmp(name, "mmg_attn_weights")) return (int)sizeof(mmg_attn_weights);
  if (!strcmp(name, "mmg_layer_weights")) return (int)sizeof(mmg_layer_weights);
  return 0;
}

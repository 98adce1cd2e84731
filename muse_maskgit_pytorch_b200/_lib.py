"""ctypes binding of libmmg.so (include/mmg.h).  The product path fails loudly if the CUDA library is missing —
there is no PyTorch or CPU fallback behind these calls."""
import ctypes as C
import os
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MMG_LIB") or os.path.join(_HERE, "libmmg.so")     # MMG_LIB: an alternative build of the library

F32, BF16, E4M3 = 0, 1, 2
EPI_STORE, EPI_RESIDUAL, EPI_GEGLU, EPI_GLU, EPI_QKV, EPI_CONVT, EPI_CONVT_RGB, EPI_LNFOLD_RESIDUAL, EPI_LFQ_IDS, EPI_ARGMIN, EPI_GEGLU_TANH, \
    EPI_QKV128 = range(12)

vp, i32, i64, f32, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_uint64


class EpilogueArgs(C.Structure):
    _fields_ = [("out", vp), ("ldo", i64), ("out_dtype", i32), ("act", i32), ("bias", vp), ("resid", vp), ("ldr", i64),
                ("q_out", vp), ("k_out", vp), ("v_out", vp), ("q_scale", vp), ("k_scale", vp), ("null_k", vp), ("null_v", vp),
                ("heads", i32), ("tokens", i32), ("q_rows", i32), ("kv_rows", i32), ("key_off", i32),
                ("nq_heads", i32), ("nk_heads", i32), ("nv_heads", i32),
                ("H", i32), ("W", i32), ("py", i32), ("px", i32),
                ("row_stats", vp), ("ln_width", i32), ("stats_slots", i32),
                ("rgb_w", vp), ("rgb_b", vp), ("rgb_channels", i32), ("_pad", i32)]


class LinearArgs(C.Structure):
    _fields_ = [("a", vp), ("w", vp), ("M", i64), ("N", i64), ("K", i64), ("lda", i64), ("ldw", i64),
                ("dtype", i32), ("epilogue", i32), ("epi", EpilogueArgs)]


class LinearFp8Args(C.Structure):
    _fields_ = [("a", vp), ("w", vp), ("a_scale", vp), ("w_scale", vp), ("M", i64), ("N", i64), ("K", i64), ("lda", i64), ("ldw", i64),
                ("dtype", i32), ("epilogue", i32), ("epi", EpilogueArgs)]


class Conv2dArgs(C.Structure):
    _fields_ = [("x", vp), ("w", vp), ("B", i32), ("H", i32), ("W", i32), ("Cin", i32), ("Cout", i32), ("kind", i32),
                ("dtype", i32), ("epilogue", i32), ("epi", EpilogueArgs)]


class ConvTranspose2dArgs(C.Structure):
    _fields_ = [("x", vp), ("w", vp), ("B", i32), ("H", i32), ("W", i32), ("Cin", i32), ("Cout", i32),
                ("dtype", i32), ("epilogue", i32), ("epi", EpilogueArgs)]


class Conv2dFp8Args(C.Structure):
    _fields_ = [("x", vp), ("w", vp), ("x_scale", vp), ("w_scale", vp), ("B", i32), ("H", i32), ("W", i32), ("Cin", i32), ("Cout", i32),
                ("kind", i32), ("dtype", i32), ("epilogue", i32), ("epi", EpilogueArgs)]


class ConvTranspose2dFp8Args(C.Structure):
    _fields_ = [("x", vp), ("w", vp), ("x_scale", vp), ("w_scale", vp), ("B", i32), ("H", i32), ("W", i32), ("Cin", i32), ("Cout", i32),
                ("dtype", i32), ("epilogue", i32), ("epi", EpilogueArgs)]


class QuantizeE4m3ImagesArgs(C.Structure):
    _fields_ = [("x", vp), ("q", vp), ("scale", vp), ("B", i64), ("hw", i64), ("C", i32), ("_pad", i32)]


class ConvInArgs(C.Structure):
    _fields_ = [("img", vp), ("w", vp), ("bias", vp), ("out", vp), ("B", i32), ("C", i32), ("H", i32), ("W", i32),
                ("Cout", i32), ("out_dtype", i32), ("ksize", i32), ("_pad", i32)]


class GroupNormArgs(C.Structure):
    _fields_ = [("x", vp), ("gamma", vp), ("beta", vp), ("B", i32), ("HW", i32), ("C", i32), ("groups", i32),
                ("dtype", i32), ("act", i32)]


class LayerNormArgs(C.Structure):
    _fields_ = [("x", vp), ("x_dtype", i32), ("y_dtype", i32), ("y", vp), ("gamma", vp), ("add", vp), ("x_out", vp), ("zero_stats", vp), ("add_from", i64),
                ("rows", i64), ("width", i64), ("ldx", i64), ("ldy", i64)]


class LayerNormFp8Args(C.Structure):
    _fields_ = [("x", vp), ("y", vp), ("row_scale", vp), ("gamma", vp), ("add", vp), ("x_out", vp), ("add_from", i64),
                ("rows", i64), ("width", i64), ("ldx", i64), ("ldy", i64)]


class EmbedArgs(C.Structure):
    _fields_ = [("ids", vp), ("token_emb", vp), ("pos_emb", vp), ("x", vp), ("rows", i64), ("n", i64), ("dim", i64),
                ("copies", i32), ("use_pos", i32)]


class AttentionArgs(C.Structure):
    _fields_ = [("q", vp), ("k", vp), ("v", vp), ("out", vp), ("key_mask", vp),
                ("B", i32), ("heads", i32), ("Tq", i32), ("Tk", i32), ("Tk_alloc", i32), ("dtype", i32),
                ("ldo", i64), ("kv_batch_stride_zero", i32), ("scale", f32), ("logit_bound", f32), ("split3", i32)]


class RemaskArgs(C.Structure):
    _fields_ = [("ids", vp), ("scores", vp), ("masked_pos", vp), ("B", i32), ("n", i32), ("num_masked", i32),
                ("mask_id", i64)]


class RemaskFrozenArgs(C.Structure):
    _fields_ = [("ids", vp), ("scores", vp), ("masked_pos", vp), ("frozen", vp), ("num_masked", vp), ("B", i32), ("n", i32), ("rows", i32),
                ("mask_id", i64)]


class EditSelectArgs(C.Structure):
    _fields_ = [("ids", vp), ("scores", vp), ("frozen_out", vp), ("keep", vp), ("num_select", vp), ("u", vp), ("seed", u64), ("seed_dev", vp),
                ("row_offset", i64), ("B", i32), ("n", i32), ("iteration", i32), ("_pad", i32), ("mask_id", i64),
                ("image_seed", vp)]


class ExtrapolateWindowArgs(C.Structure):
    _fields_ = [("canvas", vp), ("ids", vp), ("scores", vp), ("B", i32), ("f", i32), ("canvas_h", i32), ("canvas_w", i32), ("row0", i32),
                ("col0", i32), ("direction", i32), ("stride", i32), ("store", i32), ("_pad", i32), ("mask_id", i64)]


class FinalEmbedArgs(C.Structure):
    _fields_ = [("x_cond", vp), ("x_null", vp), ("gamma", vp), ("masked_pos", vp), ("e", vp), ("e_dtype", i32),
                ("B", i32), ("n", i32), ("num_masked", i32), ("dim", i32), ("cond_scale", f32), ("cond_scale_dev", vp)]


class LogitsSampleArgs(C.Structure):
    _fields_ = [("logits", vp), ("masked_pos", vp), ("ids", vp), ("scores", vp), ("u", vp),
                ("B", i32), ("n", i32), ("num_masked", i32), ("V", i32), ("k", i32), ("temperature", f32),
                ("seed", u64), ("step", u64), ("row_offset", i64), ("seed_dev", vp), ("mask_id", i64), ("only_masked", i32), ("rng_mode", i32),
                ("aten_offset", u64), ("aten_offset_dev", vp), ("aten_stride", C.c_uint32), ("_pad", i32),
                ("row_index", vp), ("row_count_dev", vp), ("row_index_cap", i32), ("_pad2", i32), ("temperature_dev", vp), ("image_seed", vp),
                ("k_dev", vp)]


class LogitsFusedArgs(C.Structure):
    _fields_ = [("e", vp), ("w", vp), ("K", i32), ("_pad", i32), ("rows_capacity", i64), ("s", LogitsSampleArgs),
                ("workspace", vp), ("workspace_bytes", u64), ("status", vp)]


class LogitsXentArgs(C.Structure):
    _fields_ = [("e", vp), ("w", vp), ("labels", vp), ("nll", vp), ("rows", i64), ("rows_capacity", i64), ("V", i32), ("K", i32),
                ("workspace", vp), ("workspace_bytes", u64)]


class LogitsXentRowsArgs(C.Structure):
    _fields_ = [("logits", vp), ("ld", i64), ("labels", vp), ("nll", vp), ("rows", i64), ("V", i32), ("_pad", i32)]


class CriticScoreArgs(C.Structure):
    _fields_ = [("x_cond", vp), ("x_null", vp), ("gamma", vp), ("w", vp), ("bias", f32), ("cond_scale", f32), ("noise_mul", f32),
                ("dim", i32), ("u", vp), ("scores", vp), ("rows", i64), ("row_offset", i64), ("seed", u64), ("seed_dev", vp),
                ("step", i32), ("rng_mode", i32), ("aten_offset", u64), ("aten_offset_dev", vp), ("aten_stride", C.c_uint32), ("_pad", i32),
                ("cond_scale_dev", vp), ("noise_mul_dev", vp), ("row_key", vp)]


class FfGegluArgs(C.Structure):
    _fields_ = [("x", vp), ("rows", i64), ("dim", i32), ("F", i32), ("Fp", i32), ("ln_gamma", vp), ("w1", vp), ("w2f", vp), ("cvec", vp),
                ("add", vp), ("add_from", i64), ("xn", vp), ("h", vp), ("stats", vp)]


class AttnWeights(C.Structure):
    _fields_ = [("ln_gamma", vp), ("w_qkv", vp), ("w_out", vp), ("q_scale", vp), ("k_scale", vp), ("null_k", vp), ("null_v", vp),
                ("logit_bound", f32), ("_pad", i32)]


class LayerWeights(C.Structure):
    _fields_ = [("self_attn", AttnWeights), ("cross_attn", AttnWeights), ("ctx_k", vp), ("ctx_v", vp), ("cross_null_out", vp),
                ("ff_ln_gamma", vp), ("ff_w1", vp), ("ff_w2f", vp), ("ff_cvec", vp)]


class DecodeStepArgs(C.Structure):
    _fields_ = [("depth", i32), ("dim", i32), ("heads", i32), ("n", i32), ("V", i32), ("F", i32), ("Fp", i32), ("b", i32), ("branches", i32),
                ("live_branches", i32), ("layers", C.POINTER(LayerWeights)), ("tok_emb", vp), ("pos_emb", vp), ("final_gamma", vp), ("w_logits", vp),
                ("ctx_key_mask", vp), ("ctx_keys", i32), ("ctx_alloc", i32), ("ids", vp), ("scores", vp), ("masked_pos", vp), ("mask_id", i64),
                ("num_masked", i32), ("k_keep", i32), ("step", i32), ("temperature", f32), ("cond_scale", f32), ("_pad", i32),
                ("u", vp), ("seed", u64), ("seed_dev", vp), ("row_offset", i64), ("workspace", vp), ("workspace_bytes", u64),
                ("cond_scale_dev", vp), ("temperature_dev", vp), ("image_seed", vp), ("k_dev", vp)]


class LfqEncodeArgs(C.Structure):
    _fields_ = [("x", vp), ("dtype", i32), ("w_in", vp), ("b_in", vp), ("ids", vp), ("T", i64), ("D", i32), ("bits", i32), ("w_split", vp)]


class L2ArgminArgs(C.Structure):
    _fields_ = [("x", vp), ("codebook", vp), ("ids", vp), ("T", i64), ("K", i32), ("D", i32)]


class DecodeCodesArgs(C.Structure):
    _fields_ = [("ids", vp), ("w_out", vp), ("b_out", vp), ("out", vp), ("dtype", i32), ("T", i64), ("D", i32), ("bits", i32)]


class CastArgs(C.Structure):
    _fields_ = [("src", vp), ("dst", vp), ("n", i64), ("src_dtype", i32), ("dst_dtype", i32)]


class Split3Args(C.Structure):
    _fields_ = [("src", vp), ("dst", vp), ("rows", i64), ("K", i64), ("lds", i64), ("side", i32), ("_pad", i32)]


class T5AttentionArgs(C.Structure):
    _fields_ = [("qkv", vp), ("out", vp), ("key_mask", vp), ("rel_bucket", vp), ("rel_bias", vp),
                ("B", i32), ("T", i32), ("heads", i32), ("num_buckets", i32), ("dtype", i32), ("_pad", i32), ("ldqkv", i64), ("ldo", i64)]


class RmsNormArgs(C.Structure):
    _fields_ = [("x", vp), ("y", vp), ("w", vp), ("row_mask", vp), ("rows", i64), ("d", i64), ("ldx", i64), ("ldy", i64),
                ("eps", f32), ("y_dtype", i32)]


EXPORTS = {
    "mmg_linear": LinearArgs, "mmg_conv2d": Conv2dArgs, "mmg_conv_transpose2d": ConvTranspose2dArgs,
    "mmg_conv_in": ConvInArgs, "mmg_groupnorm": GroupNormArgs, "mmg_layernorm": LayerNormArgs, "mmg_embed": EmbedArgs,
    "mmg_attention": AttentionArgs, "mmg_attention_d128": AttentionArgs, "mmg_remask": RemaskArgs, "mmg_final_embed": FinalEmbedArgs,
    "mmg_logits_sample": LogitsSampleArgs, "mmg_vq_lfq_encode": LfqEncodeArgs, "mmg_vq_l2_argmin": L2ArgminArgs,
    "mmg_vq_decode_codes": DecodeCodesArgs, "mmg_cast": CastArgs, "mmg_split3": Split3Args, "mmg_critic_score": CriticScoreArgs,
    "mmg_ff_geglu": FfGegluArgs, "mmg_decode_step": DecodeStepArgs, "mmg_logits_fused": LogitsFusedArgs,
    "mmg_t5_attention": T5AttentionArgs, "mmg_rmsnorm": RmsNormArgs, "mmg_remask_frozen": RemaskFrozenArgs, "mmg_edit_select": EditSelectArgs,
    "mmg_extrapolate_window": ExtrapolateWindowArgs, "mmg_logits_xent": LogitsXentArgs, "mmg_logits_xent_rows": LogitsXentRowsArgs,
    "mmg_linear_fp8": LinearFp8Args, "mmg_layernorm_fp8": LayerNormFp8Args,
    "mmg_conv2d_fp8": Conv2dFp8Args, "mmg_conv_transpose2d_fp8": ConvTranspose2dFp8Args, "mmg_quantize_e4m3_images": QuantizeE4m3ImagesArgs,
}
PLAIN_EXPORTS = ("mmg_version", "mmg_last_error", "mmg_launch_count", "mmg_sizeof", "mmg_decode_step_workspace_bytes", "mmg_logits_fused_workspace_bytes",
                 "mmg_logits_xent_workspace_bytes", "mmg_simt_fallback_count", "mmg_simt_launch_count")

_lib = None


class MMGError(RuntimeError):
    pass


def lib():
    """Load libmmg.so (built in-tree by build.py / __graft_entry__.build()).  Raises if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MMGError(f"{LIB_PATH} not found: build it with `python -m muse_maskgit_pytorch_b200.build` "
                           "(there is no fallback path)")
        l = C.CDLL(LIB_PATH)
        for name, st in EXPORTS.items():
            fn = getattr(l, name)
            fn.argtypes = [C.POINTER(st), vp]
            fn.restype = C.c_int
        l.mmg_version.restype = C.c_int
        l.mmg_last_error.restype = C.c_char_p
        l.mmg_launch_count.restype = C.c_int64
        l.mmg_simt_fallback_count.restype = C.c_int64
        l.mmg_simt_launch_count.restype = C.c_int64
        l.mmg_sizeof.argtypes = [C.c_char_p]
        l.mmg_sizeof.restype = C.c_int
        l.mmg_decode_step_workspace_bytes.argtypes = [i32] * 8
        l.mmg_decode_step_workspace_bytes.restype = u64
        l.mmg_logits_fused_workspace_bytes.argtypes = [i64, i32, i32, i32]
        l.mmg_logits_fused_workspace_bytes.restype = u64
        l.mmg_logits_xent_workspace_bytes.argtypes = [i64, i32, i32]
        l.mmg_logits_xent_workspace_bytes.restype = u64
        for name, st in list(EXPORTS.items()) + [("mmg_epilogue", EpilogueArgs), ("mmg_attn_weights", AttnWeights), ("mmg_layer_weights", LayerWeights)]:
            if l.mmg_sizeof(name.encode()) != C.sizeof(st):
                raise MMGError(f"ABI mismatch for {name}: C {l.mmg_sizeof(name.encode())} vs ctypes {C.sizeof(st)}")
        _lib = l
    return _lib


def call(name, args, stream=None):
    l = lib()
    if stream is None:
        stream = torch.cuda.current_stream().cuda_stream
    rc = getattr(l, name)(C.byref(args), vp(stream))
    if rc != 0:
        raise MMGError(f"{name} failed ({rc}): {l.mmg_last_error().decode()}")


def launch_count():
    return int(lib().mmg_launch_count())


def simt_launch_count():
    """launches of the CUDA-core GEMM / attention kernels (any dtype) so far"""
    return int(lib().mmg_simt_launch_count())


def simt_fallback_count():
    """bf16 products that left the wgmma path for the CUDA-core kernel (shape / alignment): should stay 0 on the benchmark configs."""
    return int(lib().mmg_simt_fallback_count())


def dt(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"unsupported dtype {t.dtype}")


def ptr(t):
    return None if t is None else t.data_ptr()

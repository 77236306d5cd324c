"""ctypes binding of libvqa_b200.so (the C ABI declared in include/vqa_b200.h).

The shared library is built in-tree by `__graft_entry__.build()` / `python -m t2v_metrics_b200.build`. There is no
fallback: if the library is missing or does not export the ABI, importing the engine fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libvqa_b200.so"

ABI_SYMBOLS = [
    "vqa_version", "vqa_create_clipt5", "vqa_bind_weights", "vqa_finalize_weights", "vqa_clipt5_workspace_bytes",
    "vqa_clipt5_score", "vqa_set_profile", "vqa_profile_read", "vqa_last_launch_count", "vqa_last_error", "vqa_destroy", "vqa_op_gemm_bf16",
    "vqa_op_lmhead_logprob", "vqa_op_attention_d64", "vqa_op_norm", "vqa_op_attention_d128",
    "vqa_create_qwen25vl", "vqa_qwen25vl_set_rope", "vqa_qwen25vl_workspace_bytes", "vqa_qwen25vl_score",
    "vqa_clip_preprocess_workspace_bytes", "vqa_clip_preprocess", "vqa_resample_table", "vqa_qwen_preprocess_plan",
    "vqa_qwen_preprocess", "vqa_clipt5_debug_layout", "vqa_qwen25vl_debug_layout", "vqa_set_gemm_schedule",
    "vqa_qwen25vl_topk", "vqa_op_gemm_bf16_normfuse",
    "vqa_debug_max_active_clusters", "vqa_debug_pdl_enabled", "vqa_op_attention_d128_ex", "vqa_op_gemm_bf16_grouped", "vqa_op_gemm_bf16_splitk",
    "vqa_qwen25vl_generate_workspace_bytes", "vqa_qwen25vl_generate_prefill", "vqa_qwen25vl_generate_step",
    "vqa_clipt5_generate_workspace_bytes", "vqa_clipt5_generate_prefill", "vqa_clipt5_generate_step",
    "vqa_op_answer_logprob",
    "vqa_op_kv_cache_write", "vqa_op_decode_attention_d128", "vqa_op_greedy_select", "vqa_t5_bucket_lut", "vqa_op_t5_decoder_self_attn",
    "vqa_op_t5_decode_self_attn", "vqa_op_gemm_bf16_f32acc", "vqa_op_gemm_bf16_batched", "vqa_op_t5_cross_attention", "vqa_op_layernorm_f32",
    "vqa_op_clip_embed_ln", "vqa_qwen_preprocess_video_plan", "vqa_qwen_preprocess_video",
    "vqa_op_qwen_rope", "vqa_op_gather_rows", "vqa_op_qwen_embed", "vqa_op_token_bitmap", "vqa_op_topk_softmax",
    "vqa_op_patchify", "vqa_op_splice_embed", "vqa_op_decoder_embed", "vqa_op_t5_bias_table", "vqa_op_lmhead_score", "vqa_op_row_ssq",
    "vqa_qwen_preprocess_video_aa_plan", "vqa_qwen_preprocess_video_aa", "vqa_debug_set_preprocess_tiles", "vqa_debug_preprocess_geometry",
]

VQA_DTYPE_BF16, VQA_DTYPE_F32, VQA_DTYPE_I32 = 0, 1, 2


class VqaClipT5Config(C.Structure):
    _fields_ = [
        ("image_size", C.c_int32), ("patch_size", C.c_int32), ("vit_hidden", C.c_int32), ("vit_heads", C.c_int32),
        ("vit_mlp", C.c_int32), ("vit_layers_run", C.c_int32), ("vit_ln_eps", C.c_float),
        ("d_model", C.c_int32), ("n_heads", C.c_int32), ("d_ff", C.c_int32), ("enc_layers", C.c_int32),
        ("dec_layers", C.c_int32), ("vocab", C.c_int32), ("rel_buckets", C.c_int32), ("rel_max_distance", C.c_int32),
        ("t5_ln_eps", C.c_float), ("image_token_id", C.c_int32), ("pad_token_id", C.c_int32),
        ("decoder_start_id", C.c_int32), ("emulate_bf16_rounding", C.c_int32), ("cross_attention_mode", C.c_int32),
    ]


class VqaQwen25VLConfig(C.Structure):
    _fields_ = [
        ("vit_depth", C.c_int32), ("vit_hidden", C.c_int32), ("vit_heads", C.c_int32), ("vit_head_dim", C.c_int32),
        ("vit_mlp", C.c_int32), ("patch_dim", C.c_int32), ("spatial_merge", C.c_int32), ("out_hidden", C.c_int32),
        ("fullatt_mask", C.c_uint64), ("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32),
        ("kv_heads", C.c_int32), ("mlp", C.c_int32), ("vocab", C.c_int32), ("rms_eps", C.c_float),
        ("emulate_bf16_rounding", C.c_int32),
    ]


# The Qwen2.5-VL call structs, field for field as include/vqa_b200.h declares them (tests/test_abi.py checks the layout). Pointer fields
# hold device addresses (ints); VqaQwen25VLGeneration.score points to a VqaQwen25VLAnswerScore the caller keeps alive.
class VqaQwen25VLPrompts(C.Structure):
    _fields_ = [
        ("pixel_patches", C.c_void_p), ("pixel_dtype", C.c_int32), ("n_patches", C.c_int32), ("vis_pos_hw", C.c_void_p),
        ("window_index", C.c_void_p), ("reverse_index", C.c_void_p), ("cu_window", C.c_void_p), ("n_windows", C.c_int32),
        ("max_window_len", C.c_int32), ("cu_frames", C.c_void_p), ("n_frames", C.c_int32), ("max_frame_len", C.c_int32),
        ("input_ids", C.c_void_p), ("seq_lens", C.c_void_p), ("feat_index", C.c_void_p), ("position_ids", C.c_void_p),
        ("batch", C.c_int32), ("seq_len", C.c_int32),
    ]


class VqaQwen25VLPacked(C.Structure):
    _fields_ = [
        ("total_rows", C.c_int32), ("cu_seqlens", C.c_void_p), ("kv_prefix", C.c_void_p), ("n_seq", C.c_int32), ("max_seq_len", C.c_int32),
        ("pair_row", C.c_void_p), ("pair_seq", C.c_void_p), ("max_prompt_len", C.c_int32),
    ]


class VqaQwen25VLAnswerScore(C.Structure):
    _fields_ = [
        ("answer_ids", C.c_void_p), ("answer_counts", C.c_void_p), ("n_max", C.c_int32), ("temperature", C.c_float), ("top_k", C.c_int32),
        ("out_logp", C.c_void_p), ("out_topk_ids", C.c_void_p), ("out_topk_probs", C.c_void_p),
    ]


class VqaQwen25VLGeneration(C.Structure):
    _fields_ = [
        ("seq_lens", C.c_void_p), ("first_position", C.c_void_p), ("eos_ids", C.c_void_p), ("n_eos", C.c_int32),
        ("max_new_tokens", C.c_int32), ("repetition_penalty", C.c_float), ("out_tokens", C.c_void_p), ("out_lengths", C.c_void_p),
        ("all_done", C.c_void_p), ("score", C.POINTER(VqaQwen25VLAnswerScore)),
    ]


class VqaTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("shape", C.c_int64 * 4), ("ndim", C.c_int32),
                ("dtype", C.c_int32)]


_lib = None


def load() -> C.CDLL:
    """dlopen libvqa_b200.so and declare prototypes. Raises if the library is absent (no CPU fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("VQA_B200_LIB", LIB_PATH))
    if not path.exists():
        raise ImportError(
            f"{path} not found: build it first (python -c 'import __graft_entry__ as g; g.build()'). "
            "t2v_metrics_b200 has no CPU or PyTorch fallback for the scoring path.")
    lib = C.CDLL(str(path))
    for sym in ABI_SYMBOLS:
        if not hasattr(lib, sym):
            raise ImportError(f"{path} does not export {sym}")
    vp, i32, f32, i64 = C.c_void_p, C.c_int32, C.c_float, C.c_int64
    lib.vqa_version.restype = C.c_char_p
    lib.vqa_create_clipt5.argtypes = [C.POINTER(VqaClipT5Config), C.c_int, C.POINTER(vp)]
    lib.vqa_create_clipt5.restype = C.c_int
    lib.vqa_bind_weights.argtypes = [vp, C.POINTER(VqaTensor), i32]
    lib.vqa_bind_weights.restype = C.c_int
    lib.vqa_finalize_weights.argtypes = [vp]
    lib.vqa_finalize_weights.restype = C.c_int
    lib.vqa_clipt5_workspace_bytes.argtypes = [vp, i32, i32, i32, i32]
    lib.vqa_clipt5_workspace_bytes.restype = C.c_size_t
    lib.vqa_clipt5_score.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, i32, i32, i32, vp, vp, vp, C.c_size_t, vp]
    lib.vqa_clipt5_score.restype = C.c_int
    lib.vqa_set_profile.argtypes = [vp, i32]
    lib.vqa_set_profile.restype = C.c_int
    lib.vqa_profile_read.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    lib.vqa_profile_read.restype = C.c_int
    lib.vqa_last_launch_count.argtypes = [vp]
    lib.vqa_last_launch_count.restype = i64
    lib.vqa_last_error.argtypes = [vp]
    lib.vqa_last_error.restype = C.c_char_p
    lib.vqa_destroy.argtypes = [vp]
    lib.vqa_destroy.restype = None
    lib.vqa_op_gemm_bf16.argtypes = [vp, i32, vp, i32, i32, vp, i32, i32, i32, i32, vp, vp, i32, i32, i32, i32, vp]
    lib.vqa_op_gemm_bf16.restype = C.c_int
    lib.vqa_op_gemm_bf16_normfuse.argtypes = [vp, i32, vp, i32, i32, vp, i32, i32, i32, i32, vp, i32, i32, i32, vp, vp, i32, i32, f32,
                                              C.POINTER(i32), vp]
    lib.vqa_op_gemm_bf16_normfuse.restype = C.c_int
    lib.vqa_op_lmhead_logprob.argtypes = [vp, i32, vp, i32, i32, i32, i32, vp, f32, vp, f32, vp, vp, C.c_size_t, C.POINTER(C.c_size_t), vp]
    lib.vqa_op_lmhead_logprob.restype = C.c_int
    lib.vqa_op_attention_d64.argtypes = [vp, vp, i32, i32, i32, vp, vp, f32, i32, i32, vp]
    lib.vqa_op_attention_d64.restype = C.c_int
    lib.vqa_op_norm.argtypes = [vp, vp, vp, i32, i32, f32, vp]
    lib.vqa_op_norm.restype = C.c_int
    lib.vqa_op_attention_d128.argtypes = [vp, i32, i64, i32, i32, i32, vp, i32, i32, i32, i32, i32, i32, vp, vp, f32, i32, vp]
    lib.vqa_op_attention_d128.restype = C.c_int
    lib.vqa_create_qwen25vl.argtypes = [C.POINTER(VqaQwen25VLConfig), C.c_int, C.POINTER(vp)]
    lib.vqa_create_qwen25vl.restype = C.c_int
    lib.vqa_qwen25vl_set_rope.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(i32), i32, C.POINTER(C.c_float), C.POINTER(i32), i32]
    lib.vqa_qwen25vl_set_rope.restype = C.c_int
    lib.vqa_qwen25vl_workspace_bytes.argtypes = [vp, i32, i64, i32]
    lib.vqa_qwen25vl_workspace_bytes.restype = C.c_size_t
    lib.vqa_qwen25vl_score.argtypes = [vp, C.POINTER(VqaQwen25VLPrompts), C.POINTER(VqaQwen25VLPacked), vp, f32, f32, vp, vp, vp, C.c_size_t, vp]
    lib.vqa_qwen25vl_score.restype = C.c_int
    lib.vqa_qwen25vl_topk.argtypes = [vp, i32, i64, i32, i32, f32, f32, vp, vp, vp, C.c_size_t, vp]
    lib.vqa_qwen25vl_topk.restype = C.c_int
    lib.vqa_qwen25vl_generate_workspace_bytes.argtypes = [vp, i32, i32, i32, i32]
    lib.vqa_qwen25vl_generate_workspace_bytes.restype = C.c_size_t
    lib.vqa_qwen25vl_generate_prefill.argtypes = [vp, C.POINTER(VqaQwen25VLPrompts), C.POINTER(VqaQwen25VLGeneration), vp, C.c_size_t, vp]
    lib.vqa_qwen25vl_generate_prefill.restype = C.c_int
    lib.vqa_qwen25vl_generate_step.argtypes = [vp, C.POINTER(VqaQwen25VLGeneration), i32, i32, i32, vp, C.c_size_t, vp]
    lib.vqa_qwen25vl_generate_step.restype = C.c_int
    lib.vqa_op_answer_logprob.argtypes = [vp, i32, i32, vp, f32, f32, vp, vp, i32, i32, vp, vp, i32, vp, vp, vp, vp]
    lib.vqa_op_answer_logprob.restype = C.c_int
    lib.vqa_op_kv_cache_write.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, i32, vp]
    lib.vqa_op_kv_cache_write.restype = C.c_int
    lib.vqa_op_decode_attention_d128.argtypes = [vp, i32, vp, vp, i32, vp, vp, i32, i32, i32, f32, i32, vp, C.c_size_t, C.POINTER(i32), vp,
                                                 i32, vp]
    lib.vqa_op_decode_attention_d128.restype = C.c_int
    lib.vqa_op_greedy_select.argtypes = [vp, i32, i32, vp, f32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.vqa_op_greedy_select.restype = C.c_int
    lib.vqa_t5_bucket_lut.argtypes = [i32, i32, i32, C.POINTER(i32)]
    lib.vqa_t5_bucket_lut.restype = C.c_int
    lib.vqa_op_t5_decoder_self_attn.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]
    lib.vqa_op_t5_decoder_self_attn.restype = C.c_int
    lib.vqa_op_t5_decode_self_attn.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.vqa_op_t5_decode_self_attn.restype = C.c_int
    lib.vqa_op_gemm_bf16_f32acc.argtypes = [vp, i32, vp, i32, i32, vp, i32, i32, i32, i32, vp, i32, vp]
    lib.vqa_op_gemm_bf16_f32acc.restype = C.c_int
    lib.vqa_op_gemm_bf16_batched.argtypes = [vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i64, i64, i64, i64, i64, i32, vp]
    lib.vqa_op_gemm_bf16_batched.restype = C.c_int
    lib.vqa_op_t5_cross_attention.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, C.c_size_t, C.POINTER(C.c_size_t), vp]
    lib.vqa_op_t5_cross_attention.restype = C.c_int
    lib.vqa_op_layernorm_f32.argtypes = [vp, vp, vp, vp, i32, i32, f32, vp]
    lib.vqa_op_layernorm_f32.restype = C.c_int
    lib.vqa_op_clip_embed_ln.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, f32, vp]
    lib.vqa_op_clip_embed_ln.restype = C.c_int
    lib.vqa_op_qwen_rope.argtypes = [vp, i32, vp, vp, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    lib.vqa_op_qwen_rope.restype = C.c_int
    lib.vqa_op_gather_rows.argtypes = [vp, vp, vp, i32, i32, i32, vp]
    lib.vqa_op_gather_rows.restype = C.c_int
    lib.vqa_op_qwen_embed.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, vp]
    lib.vqa_op_qwen_embed.restype = C.c_int
    lib.vqa_op_token_bitmap.argtypes = [vp, vp, i32, i32, vp, vp, vp, i32, i32, vp, vp]
    lib.vqa_op_token_bitmap.restype = C.c_int
    lib.vqa_op_topk_softmax.argtypes = [vp, i64, i32, i32, f32, vp, f32, i32, vp, vp, vp]
    lib.vqa_op_topk_softmax.restype = C.c_int
    lib.vqa_op_patchify.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp]
    lib.vqa_op_patchify.restype = C.c_int
    lib.vqa_op_splice_embed.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, vp, vp, i32, i32, i32, i32, i32, vp]
    lib.vqa_op_splice_embed.restype = C.c_int
    lib.vqa_op_decoder_embed.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp]
    lib.vqa_op_decoder_embed.restype = C.c_int
    lib.vqa_op_t5_bias_table.argtypes = [vp, vp, i32, vp, i32, i32, vp]
    lib.vqa_op_t5_bias_table.restype = C.c_int
    lib.vqa_op_lmhead_score.argtypes = [vp, i32, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp, C.c_size_t, C.POINTER(C.c_size_t), vp]
    lib.vqa_op_lmhead_score.restype = C.c_int
    lib.vqa_op_row_ssq.argtypes = [vp, vp, i32, i32, i32, vp]
    lib.vqa_op_row_ssq.restype = C.c_int
    lib.vqa_clipt5_generate_workspace_bytes.argtypes = [vp, i32, i32, i32, i32]
    lib.vqa_clipt5_generate_workspace_bytes.restype = C.c_size_t
    lib.vqa_clipt5_generate_prefill.argtypes = [vp, vp, i32, i32, vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, vp, vp, C.c_size_t, vp]
    lib.vqa_clipt5_generate_prefill.restype = C.c_int
    lib.vqa_clipt5_generate_step.argtypes = [vp, i32, i32, i32, vp, i32, i32, vp, vp, vp, vp, C.c_size_t, vp]
    lib.vqa_clipt5_generate_step.restype = C.c_int
    lib.vqa_clip_preprocess_workspace_bytes.argtypes = [C.POINTER(i32), C.POINTER(i32), i32, i32, i32]
    lib.vqa_clip_preprocess_workspace_bytes.restype = C.c_size_t
    lib.vqa_clip_preprocess.argtypes = [vp, C.POINTER(i64), C.POINTER(i32), C.POINTER(i32), i32, i32, i32, C.POINTER(C.c_uint8),
                                        C.POINTER(C.c_float), C.POINTER(C.c_float), vp, i32, vp, C.c_size_t, vp, vp]
    lib.vqa_clip_preprocess.restype = C.c_int
    lib.vqa_qwen_preprocess_plan.argtypes = [C.POINTER(i32), C.POINTER(i32), i32, i32, i32, i64, i64, C.POINTER(i32), C.POINTER(i64),
                                             C.POINTER(C.c_size_t)]
    lib.vqa_qwen_preprocess_plan.restype = C.c_int
    lib.vqa_qwen_preprocess.argtypes = [vp, C.POINTER(i64), C.POINTER(i32), C.POINTER(i32), i32, i32, i32, i32, i64, i64,
                                        C.POINTER(C.c_float), C.POINTER(C.c_float), vp, i32, vp, C.c_size_t, vp, vp]
    lib.vqa_qwen_preprocess.restype = C.c_int
    lib.vqa_qwen_preprocess_video_plan.argtypes = [C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), i32, i32, i32, i32, i64, i64,
                                                   C.POINTER(i32), C.POINTER(i64), C.POINTER(C.c_size_t)]
    lib.vqa_qwen_preprocess_video_plan.restype = C.c_int
    lib.vqa_qwen_preprocess_video.argtypes = [vp, C.POINTER(i64), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), i32, i32, i32,
                                              i32, i64, i64, C.POINTER(C.c_float), C.POINTER(C.c_float), vp, i32, vp, C.c_size_t, vp, vp]
    lib.vqa_qwen_preprocess_video.restype = C.c_int
    lib.vqa_qwen_preprocess_video_aa_plan.argtypes = [i32, i32, i32, i32, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, i32, i32, i32,
                                                      C.POINTER(i64), C.POINTER(C.c_size_t)]
    lib.vqa_qwen_preprocess_video_aa_plan.restype = C.c_int
    lib.vqa_qwen_preprocess_video_aa.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, C.POINTER(i32), C.POINTER(C.c_float), i32,
                                                 C.POINTER(i32), C.POINTER(C.c_float), i32, i32, i32, i32, C.POINTER(C.c_float),
                                                 C.POINTER(C.c_float), vp, i32, vp, C.c_size_t, vp, vp]
    lib.vqa_qwen_preprocess_video_aa.restype = C.c_int
    lib.vqa_clipt5_debug_layout.argtypes = [vp, i32, i32, i32, i32, C.POINTER(C.c_size_t), i32]
    lib.vqa_clipt5_debug_layout.restype = C.c_int
    lib.vqa_qwen25vl_debug_layout.argtypes = [vp, i32, i64, i32, C.POINTER(C.c_size_t), i32]
    lib.vqa_qwen25vl_debug_layout.restype = C.c_int
    lib.vqa_set_gemm_schedule.argtypes = [i32, i32]
    lib.vqa_set_gemm_schedule.restype = C.c_int
    lib.vqa_op_attention_d128_ex.argtypes = [vp, i32, i64, i32, i32, i32, vp, i32, i32, i32, i32, i32, vp, vp, f32, i32, i32, i32, i32, vp]
    lib.vqa_op_attention_d128_ex.restype = C.c_int
    lib.vqa_op_gemm_bf16_grouped.argtypes = [vp, i32, vp, i32, i32, vp, i32, i32, i32, i32, vp, i32, i32, i32, vp]
    lib.vqa_op_gemm_bf16_grouped.restype = C.c_int
    lib.vqa_op_gemm_bf16_splitk.argtypes = [vp, i32, vp, i32, i32, vp, i32, i32, i32, i32, vp, vp, i32, i32, vp, C.c_size_t, C.POINTER(i32), vp]
    lib.vqa_op_gemm_bf16_splitk.restype = C.c_int
    lib.vqa_debug_max_active_clusters.argtypes = [i32]
    lib.vqa_debug_max_active_clusters.restype = C.c_int
    lib.vqa_debug_pdl_enabled.argtypes = []
    lib.vqa_debug_pdl_enabled.restype = C.c_int
    lib.vqa_debug_set_preprocess_tiles.argtypes = [i32, i32, i32]
    lib.vqa_debug_set_preprocess_tiles.restype = C.c_int
    lib.vqa_debug_preprocess_geometry.argtypes = [i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), i32, i32, i32, i32, i32,
                                                  i32, i64, i64, C.POINTER(i32)]
    lib.vqa_debug_preprocess_geometry.restype = C.c_int
    lib.vqa_resample_table.argtypes = [i32, i32, i32, i32, C.POINTER(i32), C.POINTER(i32)]
    lib.vqa_resample_table.restype = i32
    _lib = lib
    return lib


def last_error(handle=None) -> str:
    msg = load().vqa_last_error(handle)
    return msg.decode() if msg else ""

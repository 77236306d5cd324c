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

VQA_DTYPE_BF16, VQA_DTYPE_F32, VQA_DTYPE_I32 = 0, 1, 2
VQA_OK, VQA_ERR_INVALID_ARG, VQA_ERR_MISSING_WEIGHT, VQA_ERR_CUDA, VQA_ERR_WORKSPACE, VQA_ERR_UNSUPPORTED = 0, -1, -2, -3, -4, -5   # vqa_status


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


class VqaQwen25VLSampling(C.Structure):
    # top_p is a double: the kernels compare against fp32(1 - top_p) of the caller's value, as HF does
    _fields_ = [("seeds", C.c_void_p), ("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_double)]


class VqaTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("shape", C.c_int64 * 4), ("ndim", C.c_int32),
                ("dtype", C.c_int32)]


# Every function include/vqa_b200.h declares: name -> (restype, argtypes). tests/test_abi.py checks each entry against the header.
_vp, _i32, _i64, _f32, _sz, _P = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_size_t, C.POINTER
PROTOTYPES = {
    "vqa_version": (C.c_char_p, []),
    "vqa_create_clipt5": (_i32, [_P(VqaClipT5Config), _i32, _P(_vp)]),
    "vqa_bind_weights": (_i32, [_vp, _P(VqaTensor), _i32]),
    "vqa_finalize_weights": (_i32, [_vp]),
    "vqa_clipt5_workspace_bytes": (_sz, [_vp, _i32, _i32, _i32, _i32]),
    "vqa_clipt5_score": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "vqa_clipt5_generate_workspace_bytes": (_sz, [_vp, _i32, _i32, _i32, _i32]),
    "vqa_clipt5_generate_prefill": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vqa_clipt5_generate_step": (_i32, [_vp, _i32, _i32, _i32, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vqa_clipt5_generate_prefill_sampled": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _vp,
                                                   _P(VqaQwen25VLSampling), _vp, _sz, _vp]),
    "vqa_clipt5_generate_step_sampled": (_i32, [_vp, _i32, _i32, _i32, _vp, _i32, _i32, _vp, _vp, _vp, _P(VqaQwen25VLSampling), _vp, _sz, _vp]),
    "vqa_create_qwen25vl": (_i32, [_P(VqaQwen25VLConfig), _i32, _P(_vp)]),
    "vqa_qwen25vl_set_rope": (_i32, [_vp, _P(_f32), _P(_i32), _i32, _P(_f32), _P(_i32), _i32]),
    "vqa_qwen25vl_workspace_bytes": (_sz, [_vp, _i32, _i64, _i32]),
    "vqa_qwen25vl_score": (_i32, [_vp, _P(VqaQwen25VLPrompts), _P(VqaQwen25VLPacked), _vp, _f32, _f32, _vp, _vp, _vp, _sz, _vp]),
    "vqa_qwen25vl_topk": (_i32, [_vp, _i32, _i64, _i32, _i32, _f32, _f32, _vp, _vp, _vp, _sz, _vp]),
    "vqa_qwen25vl_generate_workspace_bytes": (_sz, [_vp, _i32, _i32, _i32, _i32]),
    "vqa_qwen25vl_generate_prefill": (_i32, [_vp, _P(VqaQwen25VLPrompts), _P(VqaQwen25VLGeneration), _vp, _sz, _vp]),
    "vqa_qwen25vl_generate_step": (_i32, [_vp, _P(VqaQwen25VLGeneration), _i32, _i32, _i32, _vp, _sz, _vp]),
    "vqa_qwen25vl_generate_prefill_sampled": (_i32, [_vp, _P(VqaQwen25VLPrompts), _P(VqaQwen25VLGeneration), _P(VqaQwen25VLSampling), _vp, _sz,
                                                     _vp]),
    "vqa_qwen25vl_generate_step_sampled": (_i32, [_vp, _P(VqaQwen25VLGeneration), _P(VqaQwen25VLSampling), _i32, _i32, _i32, _vp, _sz, _vp]),
    "vqa_last_launch_count": (_i64, [_vp]),
    "vqa_set_profile": (_i32, [_vp, _i32]),
    "vqa_profile_read": (_i32, [_vp, _P(_f32), _P(C.c_double), _P(C.c_double), _P(_i64)]),
    "vqa_clipt5_debug_layout": (_i32, [_vp, _i32, _i32, _i32, _i32, _P(_sz), _i32]),
    "vqa_qwen25vl_debug_layout": (_i32, [_vp, _i32, _i64, _i32, _P(_sz), _i32]),
    "vqa_set_gemm_schedule": (_i32, [_i32, _i32]),
    "vqa_debug_max_active_clusters": (_i32, [_i32]),
    "vqa_debug_pdl_enabled": (_i32, []),
    "vqa_debug_set_preprocess_tiles": (_i32, [_i32, _i32, _i32]),
    "vqa_debug_preprocess_geometry": (_i32, [_i32, _P(_i32), _P(_i32), _P(_i32), _P(_i32), _i32, _i32, _i32, _i32, _i32, _i32, _i64, _i64,
                                             _P(_i32)]),
    "vqa_debug_set_preprocess_aa_rows": (_i32, [_i32]),
    "vqa_debug_preprocess_aa_geometry": (_i32, [_i32, _i32, _i32, _i32, _P(_i32), _i32, _P(_i32), _i32, _i32, _i32, _P(_i32)]),
    "vqa_last_error": (C.c_char_p, [_vp]),
    "vqa_destroy": (None, [_vp]),
    "vqa_clip_preprocess_workspace_bytes": (_sz, [_P(_i32), _P(_i32), _i32, _i32, _i32]),
    "vqa_clip_preprocess": (_i32, [_vp, _P(_i64), _P(_i32), _P(_i32), _i32, _i32, _i32, _P(C.c_uint8), _P(_f32), _P(_f32), _vp, _i32, _vp, _sz,
                                   _vp, _vp]),
    "vqa_qwen_preprocess_video_plan": (_i32, [_P(_i32), _P(_i32), _P(_i32), _P(_i32), _i32, _i32, _i32, _i32, _i64, _i64, _P(_i32), _P(_i64),
                                              _P(_sz)]),
    "vqa_qwen_preprocess_video": (_i32, [_vp, _P(_i64), _P(_i32), _P(_i32), _P(_i32), _P(_i32), _i32, _i32, _i32, _i32, _i64, _i64, _P(_f32),
                                         _P(_f32), _vp, _i32, _vp, _sz, _vp, _vp]),
    "vqa_qwen_preprocess_video_aa_plan": (_i32, [_i32, _i32, _i32, _i32, _P(_i32), _i32, _P(_i32), _i32, _i32, _i32, _i32, _i32, _P(_i64),
                                                 _P(_sz)]),
    "vqa_qwen_preprocess_video_aa": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _P(_i32), _P(_f32), _i32, _P(_i32), _P(_f32), _i32,
                                            _i32, _i32, _i32, _P(_f32), _P(_f32), _vp, _i32, _vp, _sz, _vp, _vp]),
    "vqa_resample_table": (_i32, [_i32, _i32, _i32, _i32, _P(_i32), _P(_i32)]),
    "vqa_op_gemm_bf16": (_i32, [_vp, _i32, _vp, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "vqa_op_gemm_bf16_normfuse": (_i32, [_vp, _i32, _vp, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _vp, _vp, _i32, _i32,
                                         _f32, _P(_i32), _vp]),
    "vqa_op_lmhead_logprob": (_i32, [_vp, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _f32, _vp, _f32, _vp, _vp, _sz, _P(_sz), _vp]),
    "vqa_op_answer_logprob": (_i32, [_vp, _i32, _i32, _vp, _f32, _f32, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp]),
    "vqa_op_kv_cache_write": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _vp]),
    "vqa_op_decode_attention_d128": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _f32, _i32, _vp, _sz, _P(_i32), _vp, _i32,
                                            _vp]),
    "vqa_op_greedy_select": (_i32, [_vp, _i32, _i32, _vp, _f32, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqa_op_sample_select": (_i32, [_vp, _i32, _i32, _vp, _f32, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                    _P(VqaQwen25VLSampling), _vp, _vp]),
    "vqa_debug_sample_terms": (_i32, [_vp, _i32, _i32, _vp, _f32, _vp, _P(VqaQwen25VLSampling), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqa_op_clipt5_expand_prompts": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "vqa_t5_bucket_lut": (_i32, [_i32, _i32, _i32, _P(_i32)]),
    "vqa_op_t5_decoder_self_attn": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "vqa_op_t5_decode_self_attn": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "vqa_op_attention_d64": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _f32, _i32, _i32, _vp]),
    "vqa_op_norm": (_i32, [_vp, _vp, _vp, _i32, _i32, _f32, _vp]),
    "vqa_op_attention_d128": (_i32, [_vp, _i32, _i64, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _f32, _i32, _vp]),
    "vqa_op_attention_d128_ex": (_i32, [_vp, _i32, _i64, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _f32, _i32, _i32, _i32,
                                        _i32, _vp]),
    "vqa_op_gemm_bf16_splitk": (_i32, [_vp, _i32, _vp, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _i32, _vp, _sz, _P(_i32), _vp]),
    "vqa_op_gemm_bf16_grouped": (_i32, [_vp, _i32, _vp, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _vp]),
    "vqa_op_gemm_bf16_f32acc": (_i32, [_vp, _i32, _vp, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _vp]),
    "vqa_op_gemm_bf16_batched": (_i32, [_vp, _i32, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _i64,
                                        _i64, _i32, _vp]),
    "vqa_op_t5_cross_attention": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _sz, _P(_sz), _vp]),
    "vqa_op_layernorm_f32": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _f32, _vp]),
    "vqa_op_clip_embed_ln": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp]),
    "vqa_op_patchify": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "vqa_op_splice_embed": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "vqa_op_decoder_embed": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "vqa_op_t5_bias_table": (_i32, [_vp, _vp, _i32, _vp, _i32, _i32, _vp]),
    "vqa_op_lmhead_score": (_i32, [_vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _P(_sz), _vp]),
    "vqa_op_row_ssq": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp]),
    "vqa_op_qwen_rope": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "vqa_op_gather_rows": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "vqa_op_qwen_embed": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "vqa_op_token_bitmap": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "vqa_op_topk_softmax": (_i32, [_vp, _i64, _i32, _i32, _f32, _vp, _f32, _i32, _vp, _vp, _vp]),
}

_lib = None


def load() -> C.CDLL:
    """dlopen libvqa_b200.so and declare PROTOTYPES. Raises if the library is absent (no CPU fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("VQA_B200_LIB", LIB_PATH))
    if not path.exists():
        raise ImportError(
            f"{path} not found: build it first (python -c 'import __graft_entry__ as g; g.build()'). "
            "t2v_metrics_b200 has no CPU or PyTorch fallback for the scoring path.")
    lib = C.CDLL(str(path))
    for name, (restype, argtypes) in PROTOTYPES.items():
        if not hasattr(lib, name):
            raise ImportError(f"{path} does not export {name}")
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def last_error(handle=None) -> str:
    msg = load().vqa_last_error(handle)
    return msg.decode() if msg else ""

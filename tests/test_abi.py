"""The C-ABI shared library loads without a GPU and exports every symbol include/vqa_b200.h declares."""
import ctypes
import os
import re

from t2v_metrics_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    text = open(os.path.join(ROOT, "include", "vqa_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vqa_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported():
    lib = _lib.load()
    names = declared_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(_lib.ABI_SYMBOLS) == names


def test_qwen_struct_layout_matches_header():
    # field names in header order, and the sizes and last-field offsets vqa_b200.cu static_asserts, for the Qwen2.5-VL call structs
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqa_b200.h")).read(), flags=re.S)
    for cls, name, size, offset in [(_lib.VqaQwen25VLPrompts, "vqa_qwen25vl_prompts", 112, 108), (_lib.VqaQwen25VLPacked, "vqa_qwen25vl_packed", 56, 48),
                                    (_lib.VqaQwen25VLAnswerScore, "vqa_qwen25vl_answer_score", 56, 48),
                                    (_lib.VqaQwen25VLGeneration, "vqa_qwen25vl_generation", 72, 64)]:
        body = re.search(r"typedef struct \{([^}]*)\} " + name + ";", text).group(1)
        assert [f[0] for f in cls._fields_] == re.findall(r"(\w+);", body), name
        assert ctypes.sizeof(cls) == size and getattr(cls, cls._fields_[-1][0]).offset == offset, name


def test_version_and_null_handling():
    lib = _lib.load()
    assert b"sm_90a" in lib.vqa_version()
    assert lib.vqa_finalize_weights(None) != 0
    assert lib.vqa_last_launch_count(None) == 0
    lib.vqa_destroy(None)  # no-op


def test_create_fails_cleanly_without_device():
    import torch
    if torch.cuda.is_available():
        return
    lib = _lib.load()
    cfg = _lib.VqaClipT5Config(image_size=336, patch_size=14, vit_hidden=1024, vit_heads=16, vit_mlp=4096, vit_layers_run=23,
                               vit_ln_eps=1e-5, d_model=4096, n_heads=64, d_ff=10240, enc_layers=24, dec_layers=24, vocab=32128,
                               rel_buckets=32, rel_max_distance=128, t5_ln_eps=1e-6, image_token_id=-200, pad_token_id=0,
                               decoder_start_id=0, emulate_bf16_rounding=1)
    h = ctypes.c_void_p()
    rc = lib.vqa_create_clipt5(ctypes.byref(cfg), 0, ctypes.byref(h))
    assert rc != 0 and not h.value
    assert _lib.last_error(None)

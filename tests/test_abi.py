"""The C-ABI shared library loads without a GPU and exports every symbol include/vqa_b200.h declares."""
import ctypes
import os
import re

from t2v_metrics_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_text():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqa_b200.h")).read(), flags=re.S)


def declared_functions():
    return sorted(set(re.findall(r"\b(vqa_[a-z0-9_]+)\s*\(", header_text())))


def declared_prototypes():
    """{name: (return kind, [parameter kinds])} of every function declaration in the header."""
    out = {}
    for ret, name, params in re.findall(r"^\s*([A-Za-z_][\w\s]*?\**)\s*\b(vqa_\w+)\s*\(([^)]*)\)\s*;", header_text(), flags=re.M):
        params = [p.strip() for p in params.split(",")]
        args = [] if params == ["void"] else [c_kind(re.sub(r"\w+$", "", p)) for p in params]     # drop the parameter name
        out[name] = (c_kind(ret), args)
    return out


C_KINDS = {"void": None, "int": "i32", "int32_t": "i32", "uint32_t": "i32", "int64_t": "i64", "size_t": "u64", "uint64_t": "u64",
           "float": "f32", "double": "f64"}


def c_kind(decl: str):
    """The kind of a C type as written in the header (parameter name already removed)."""
    if "*" in decl:
        return "ptr"
    return C_KINDS[decl.replace("const", "").strip()]


def ctypes_kind(t):
    """The kind of a ctypes type; on Linux c_size_t is c_uint64, so size_t and uint64_t are one kind."""
    if t is None:
        return None
    if isinstance(t, type) and issubclass(t, (ctypes._Pointer, ctypes.c_void_p, ctypes.c_char_p)):
        return "ptr"
    code = t._type_
    if code in "fd":
        return {"f": "f32", "d": "f64"}[code]
    assert code in "iIlLqQ", t
    if ctypes.sizeof(t) == 4:
        return "i32"
    return "i64" if code.islower() else "u64"


def test_header_symbols_exported():
    lib = _lib.load()
    names = declared_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(_lib.PROTOTYPES) == names


def test_prototypes_match_header():
    # a wrong integer width or a missing argument is undefined behaviour at the foreign-call boundary: every entry of the ctypes table must
    # have the header's return kind and parameter kinds, in order
    declared = declared_prototypes()
    assert sorted(declared) == declared_functions()
    for name, (restype, argtypes) in _lib.PROTOTYPES.items():
        ret, args = declared[name]
        assert ctypes_kind(restype) == ret, f"{name}: return type"
        assert [ctypes_kind(t) for t in argtypes] == args, f"{name}: parameters"


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

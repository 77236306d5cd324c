"""Architecture descriptions for the engine (the HF config objects the reference loads with `from_pretrained`,
t2v_metrics/models/vqascore_models/mm_utils.py:182-241, reduced to what the kernels need)."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass


@dataclass
class ClipT5Config:
    # CLIP ViT-L/14-336 vision tower
    image_size: int = 336
    patch_size: int = 14
    vit_hidden: int = 1024
    vit_heads: int = 16
    vit_mlp: int = 4096
    vit_layers: int = 24           # layers in the checkpoint; mm_vision_select_layer=-2 => vit_layers - 1 are executed
    vit_ln_eps: float = 1e-5
    # FlanT5 encoder-decoder
    d_model: int = 4096
    n_heads: int = 64
    d_kv: int = 64
    d_ff: int = 10240
    enc_layers: int = 24
    dec_layers: int = 24
    vocab: int = 32128
    rel_buckets: int = 32
    rel_max_distance: int = 128
    t5_ln_eps: float = 1e-6
    pad_token_id: int = 0
    decoder_start_id: int = 0

    @property
    def num_patches(self) -> int:
        return (self.image_size // self.patch_size) ** 2

    @staticmethod
    def xxl() -> "ClipT5Config":
        """clip-flant5-xxl (google/flan-t5-xxl + openai/clip-vit-large-patch14-336), SURVEY App. A."""
        return ClipT5Config()

    @staticmethod
    def xl() -> "ClipT5Config":
        return ClipT5Config(d_model=2048, n_heads=32, d_ff=5120)


CLIPT5_MODELS = {
    # public names of the reference's (v3.0) model table; checkpoints: zhiqiulin/clip-flant5-{xxl,xl}
    "clip-flant5-xxl": dict(config=ClipT5Config.xxl, tokenizer="google/flan-t5-xxl", weights="zhiqiulin/clip-flant5-xxl"),
    "clip-flant5-xl": dict(config=ClipT5Config.xl, tokenizer="google/flan-t5-xl", weights="zhiqiulin/clip-flant5-xl"),
}


@dataclass
class Qwen25VLConfig:
    """Qwen2.5-VL dims (7B defaults; transformers configuration_qwen2_5_vl.py:51-64,106-125, SURVEY App. B)."""
    vit_depth: int = 32
    vit_hidden: int = 1280
    vit_heads: int = 16
    vit_mlp: int = 3420
    patch_size: int = 14
    temporal_patch_size: int = 2
    spatial_merge_size: int = 2
    window_size: int = 112
    fullatt_block_indexes: tuple = (7, 15, 23, 31)
    out_hidden: int = 3584
    tokens_per_second: int = 2
    hidden: int = 3584
    layers: int = 28
    heads: int = 28
    kv_heads: int = 4
    mlp: int = 18944
    vocab: int = 152064
    rms_eps: float = 1e-6
    rope_theta: float = 1e6
    mrope_section: tuple = (16, 24, 24)
    image_token_id: int = 151655
    video_token_id: int = 151656
    # lm_head shares the embedding matrix (the checkpoint then stores no `lm_head.weight`)
    tie_word_embeddings: bool = False

    @property
    def head_dim(self) -> int:
        return self.hidden // self.heads

    @property
    def vit_head_dim(self) -> int:
        return self.vit_hidden // self.vit_heads

    @property
    def patch_dim(self) -> int:
        return 3 * self.temporal_patch_size * self.patch_size ** 2

    @property
    def vit_mlp_padded(self) -> int:
        return (self.vit_mlp + 127) // 128 * 128

    @staticmethod
    def qwen25_vl_7b() -> "Qwen25VLConfig":
        return Qwen25VLConfig()

    @staticmethod
    def qwen25_vl_3b() -> "Qwen25VLConfig":
        """Qwen/Qwen2.5-VL-3B-Instruct's config.json: hidden_size 2048, num_hidden_layers 36, num_attention_heads 16,
        num_key_value_heads 2, intermediate_size 11008, vocab_size 151936, tie_word_embeddings true; vision_config as the 7B's with
        out_hidden_size 2048. A checkpoint directory's own config.json is compared against these values when it is loaded
        (Qwen2VLModel.load_model), so a disagreement raises instead of binding wrong shapes."""
        return Qwen25VLConfig(out_hidden=2048, hidden=2048, layers=36, heads=16, kv_heads=2, mlp=11008, vocab=151936,
                              tie_word_embeddings=True)

    @staticmethod
    def from_hf_config(path_or_dict) -> "Qwen25VLConfig":
        """The dims of a checkpoint's config.json (a path to the file or to its directory, or the parsed dict). Accepts both layouts
        transformers reads: the published flat one (text fields at the top level, `rope_scaling`) and transformers 5.5.0's
        `Qwen2_5_VLConfig.to_dict()` (text fields under `text_config`, `rope_parameters`); `vision_config` holds the tower in both.
        Fields a file leaves out keep this class's defaults."""
        import json
        import os
        d = path_or_dict
        if not isinstance(d, dict):
            path = os.path.join(d, "config.json") if os.path.isdir(d) else d
            with open(path) as f:
                d = json.load(f)
        text = dict(d)
        text.update(d.get("text_config") or {})
        vis = d.get("vision_config") or {}
        rope = text.get("rope_parameters") or text.get("rope_scaling") or {}
        base = Qwen25VLConfig()
        kw = dict(
            vit_depth=vis.get("depth"), vit_hidden=vis.get("hidden_size"), vit_heads=vis.get("num_heads"), vit_mlp=vis.get("intermediate_size"),
            patch_size=vis.get("patch_size"), temporal_patch_size=vis.get("temporal_patch_size"), spatial_merge_size=vis.get("spatial_merge_size"),
            window_size=vis.get("window_size"), out_hidden=vis.get("out_hidden_size"), tokens_per_second=vis.get("tokens_per_second"),
            hidden=text.get("hidden_size"), layers=text.get("num_hidden_layers"), heads=text.get("num_attention_heads"),
            kv_heads=text.get("num_key_value_heads"), mlp=text.get("intermediate_size"), vocab=text.get("vocab_size"),
            rms_eps=text.get("rms_norm_eps"), rope_theta=rope.get("rope_theta", text.get("rope_theta")),
            image_token_id=d.get("image_token_id"), video_token_id=d.get("video_token_id"),
            tie_word_embeddings=d.get("tie_word_embeddings", text.get("tie_word_embeddings")))
        if vis.get("fullatt_block_indexes") is not None:
            kw["fullatt_block_indexes"] = tuple(vis["fullatt_block_indexes"])
        if rope.get("mrope_section") is not None:
            kw["mrope_section"] = tuple(rope["mrope_section"])
        kw = {k: v for k, v in kw.items() if v is not None}
        for k in ("rms_eps", "rope_theta"):
            if k in kw:
                kw[k] = float(kw[k])
        if "tie_word_embeddings" in kw:
            kw["tie_word_embeddings"] = bool(kw["tie_word_embeddings"])
        return dataclasses.replace(base, **kw)

    def mismatches(self, other: "Qwen25VLConfig") -> dict:
        """{field: (self's value, other's value)} over every field that decides a kernel shape, a weight binding or the arithmetic."""
        return {f.name: (getattr(self, f.name), getattr(other, f.name)) for f in dataclasses.fields(self)
                if getattr(self, f.name) != getattr(other, f.name)}


# listed: the name appears in list_all_models(). That listing holds the sizes bench.py measures, so that every listed name is a bench.py
# workload. The 3B is not a bench.py workload; VQAScore and get_score_model accept it by name.
QWEN25VL_MODELS = {
    "qwen2.5-vl-3b": dict(config=Qwen25VLConfig.qwen25_vl_3b, weights="Qwen/Qwen2.5-VL-3B-Instruct", listed=False),
    "qwen2.5-vl-7b": dict(config=Qwen25VLConfig.qwen25_vl_7b, weights="Qwen/Qwen2.5-VL-7B-Instruct", listed=True),
}

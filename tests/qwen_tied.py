"""Tied-embedding Qwen2.5-VL fixtures (Qwen2.5-VL-3B ties lm_head to the token embedding and has 8 query heads per K/V head).

Synthetic tied weights are the untied ones of oracle.qwen25vl_oracle.make_synthetic_state_dict with the drawn lm_head taking the
embedding's place: the checkpoint then carries no `lm_head.weight`, as a published tied checkpoint does. The oracle and HF builders of
oracle/ read `lm_head.weight`; `with_lm_head` hands them the embedding under that name (the same tensor)."""
import dataclasses
import hashlib
import os

import torch

from oracle import qwen25vl_oracle as qo

# head_dim 128 and 16 query heads over 2 K/V heads, the attention layout of Qwen2.5-VL-3B, at two layers
TINY_GQA8 = dict(hidden=2048, heads=16, kv_heads=2, out_hidden=2048, mrope_section=(16, 24, 24))
EMBED = "model.language_model.embed_tokens.weight"


def tie(sd):
    """An untied synthetic state dict -> the tied one: the embedding is the drawn lm_head (std hidden^-0.5), lm_head.weight is dropped."""
    sd = dict(sd)
    sd[EMBED] = sd.pop("lm_head.weight")
    return sd


def tied_state_dict(cfg, seed=0, gen_device="cpu"):
    return tie(qo.make_synthetic_state_dict(cfg, seed=seed, gen_device=gen_device))


def with_lm_head(sd):
    """The tied state dict with `lm_head.weight` bound to the embedding tensor, for the oracle (which reads that name)."""
    return dict(sd, **{"lm_head.weight": sd[EMBED]})


def sd_checksum(sd):
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def engine_config(cfg):
    """The engine's config with the oracle config's fields, tied."""
    from t2v_metrics_b200.config import Qwen25VLConfig
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    return Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(cfg).items() if k in fields}, tie_word_embeddings=True)


def build_hf_qwen_tied(cfg, sd, dtype=torch.float32, device="cpu", attn="eager"):
    """The real Qwen2_5_VLForConditionalGeneration with tie_word_embeddings=True carrying the tied `sd`: its lm_head IS its embedding
    module's weight (transformers' tie_weights), so this is the reference's own tied arithmetic, calibration edits included."""
    from transformers import Qwen2_5_VLForConditionalGeneration
    from oracle.hf_reference import _construct_on, _cast_keep_float_buffers, hf_qwen_config
    c = hf_qwen_config(cfg)
    c.tie_word_embeddings = True
    c._attn_implementation = attn
    if torch.device(device).type == "cuda":
        prev = torch.get_default_dtype()
        torch.set_default_dtype(dtype)
        try:
            with _construct_on(device):
                m = Qwen2_5_VLForConditionalGeneration(c)
        finally:
            torch.set_default_dtype(prev)
        missing, unexpected = m.load_state_dict({k: v.to(device, dtype) for k, v in sd.items()}, strict=False)
    else:
        m = Qwen2_5_VLForConditionalGeneration(c)
        missing, unexpected = m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
        _cast_keep_float_buffers(m, dtype, device)
    assert missing == ["lm_head.weight"] and not unexpected, (missing, unexpected)
    m.tie_weights()
    assert m.lm_head.weight.data_ptr() == m.model.language_model.embed_tokens.weight.data_ptr()
    return m.eval().requires_grad_(False)


def load_tied_golden(golden_dir):
    """tests/golden/qwen_tied_gqa8_tiny.pt (tools/make_golden_qwen_3b.py) with its weights regenerated from their seed."""
    blob = torch.load(os.path.join(golden_dir, "qwen_tied_gqa8_tiny.pt"), weights_only=False)
    cfg = qo.Qwen25VLConfig(**blob["config"])
    sd = tied_state_dict(cfg, seed=blob["weights_seed"])
    assert sd_checksum(sd) == blob["weights_sha256"], "synthetic weights differ from the ones the golden was generated with"
    return blob, cfg, sd

"""The Qwen2.5-VL size a tool measures (`--model`): its dims from the engine's model table, seeded synthetic weights drawn on the device
(tied, without lm_head.weight, for a size that ties its embeddings), the engine carrying them, and the real transformers model with the
same weights for the HF arm."""
import dataclasses
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import qwen25vl_oracle as qo
from t2v_metrics_b200.config import QWEN25VL_MODELS


def add_model_arg(ap):
    ap.add_argument("--model", default="qwen2.5-vl-7b", choices=sorted(QWEN25VL_MODELS))


def model_config(name):
    """(the oracle's config with the table entry's dims, the table entry)."""
    ecfg = QWEN25VL_MODELS[name]["config"]()
    fields = {f.name for f in dataclasses.fields(qo.Qwen25VLConfig)}
    return qo.Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(ecfg).items() if k in fields}), ecfg


def synthetic_weights(cfg, ecfg, dev, seed=0):
    if ecfg.tie_word_embeddings:
        from qwen_tied import tied_state_dict
        return tied_state_dict(cfg, seed=seed, gen_device=dev)
    return qo.make_synthetic_state_dict(cfg, seed=seed, gen_device=dev)


def engine(ecfg, sd, dev):
    from t2v_metrics_b200.engine import QwenVLEngine
    eng = QwenVLEngine(ecfg, dev)
    eng.load_state_dict(sd)
    return eng


def hf_model(cfg, ecfg, sd, dev):
    """HF Qwen2_5_VLForConditionalGeneration in bf16 with sdpa, as the reference loads it."""
    import torch
    if ecfg.tie_word_embeddings:
        from qwen_tied import build_hf_qwen_tied
        return build_hf_qwen_tied(cfg, sd, dtype=torch.bfloat16, device=dev, attn="sdpa")
    import hf_reference as hf
    return hf.build_hf_qwen(cfg, sd, dtype=torch.bfloat16, device=dev, attn="sdpa", assign=True)

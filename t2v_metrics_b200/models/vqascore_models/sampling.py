"""How both generating plugins resolve the sampling parameters of a `generate` call, as the reference's generate does."""
from __future__ import annotations

from typing import Optional

import torch

# Warpers transformers adds for generate(do_sample=True) when generation_config.json enables them (generation/utils.py:1197-1230), with the
# value that leaves each one off. The engine samples with repetition penalty, temperature, top-k and top-p only; a checkpoint that turns
# one of these on is refused rather than sampled from another distribution.
_UNSUPPORTED_WARPERS = {"min_p": None, "typical_p": 1.0, "epsilon_cutoff": 0.0, "eta_cutoff": 0.0, "top_h": None}
HF_DEFAULT_TOP_K = 50      # GenerationConfig's top_k when neither the call nor generation_config.json sets one


def sampling_params(checkpoint_path: str, do_sample: Optional[bool], temperature: float, top_p: float) -> Optional[tuple]:
    """(temperature, top_k, top_p) of the reference's generate (qwen2vl_model.py:512-551), or None for greedy decoding. do_sample None means
    temperature > 0, and only do_sample with temperature > 0 samples. The call passes temperature and top_p, so top_k is the one of the
    generation_config.json beside the checkpoint, else transformers' default 50 (0 = off). A file that enables another warper raises."""
    from ...checkpoint import generation_config_value
    if do_sample is None:
        do_sample = temperature > 0
    if not (do_sample and temperature > 0):
        return None
    for key, off in _UNSUPPORTED_WARPERS.items():
        v = generation_config_value(checkpoint_path, key, off)
        if v != off:
            raise NotImplementedError(f"generation_config.json sets {key} = {v!r}: sampling supports the repetition penalty, temperature, "
                                      "top_k and top_p warpers only")
    if not (0.0 < top_p <= 1.0) or not torch.isfinite(torch.tensor(float(temperature))):
        raise ValueError(f"sampling needs a finite temperature > 0 and 0 < top_p <= 1 (got temperature {temperature}, top_p {top_p})")
    top_k = int(generation_config_value(checkpoint_path, "top_k", HF_DEFAULT_TOP_K))
    if top_k < 0:
        raise ValueError(f"generation_config.json sets top_k = {top_k}")
    return float(temperature), top_k, float(top_p)

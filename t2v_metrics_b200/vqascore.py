"""`VQAScore`: the public scorer class, i.e. `Score` wired to the registry of engine-backed VQAScore plugins
(the reference keeps the same split: t2v_metrics/vqascore.py:9-23 on top of t2v_metrics/score.py)."""
from __future__ import annotations

from typing import List

from . import constants
from .models import vqascore_models as _registry
from .models.vqascore_models import list_all_vqascore_models      # re-exported: the package __init__ imports it from here
from .score import Score

__all__ = ["VQAScore", "list_all_vqascore_models"]


class VQAScore(Score):
    def prepare_scoremodel(self, model: str = "clip-flant5-xxl", device: str = "cuda", cache_dir: str = constants.HF_CACHE_DIR, **kwargs):
        """Instantiate the plugin registered under `model`; extra keyword arguments (checkpoint=, state_dict=, tokenizer=, ...) go to it."""
        return _registry.get_vqascore_model(model, device=device, cache_dir=cache_dir, **kwargs)

    def list_all_models(self) -> List[str]:
        """The names this scorer accepts: list_all_vqascore_models() and the sizes accepted by name only (qwen2.5-vl-3b)."""
        return _registry.accepted_vqascore_models()

"""t2v_metrics_b200 -- H100-native (sm_90a) drop-in for the VQAScore scoring hot path of linzhiqiu/t2v_metrics.

Public surface mirrors the reference package (t2v_metrics/__init__.py:23-33): VQAScore, list_all_models,
get_score_model. The ffmpeg import gate of the reference is not reproduced: video decoding is outside this engine.
"""
from .constants import HF_CACHE_DIR
from .models.vqascore_models import accepted_vqascore_models
from .vqascore import VQAScore, list_all_vqascore_models

__all__ = ["VQAScore", "list_all_models", "get_score_model", "HF_CACHE_DIR"]


def list_all_models():
    return list_all_vqascore_models()


def get_score_model(model='clip-flant5-xxl', device='cuda', cache_dir=HF_CACHE_DIR, **kwargs):
    if model in accepted_vqascore_models():
        return VQAScore(model, device=device, cache_dir=cache_dir, **kwargs)
    raise NotImplementedError()

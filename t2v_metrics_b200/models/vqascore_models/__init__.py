"""Registry + factory, same surface as the reference's t2v_metrics/models/vqascore_models/__init__.py:14-53."""
from ...constants import HF_CACHE_DIR
from .clip_t5_model import CLIP_T5_MODELS, CLIPT5Model
from .qwen2vl_model import QWEN2_VL_MODELS, Qwen2VLModel

ALL_VQA_MODELS = [CLIP_T5_MODELS, QWEN2_VL_MODELS]


def list_all_vqascore_models():
    """The listed models (the ones bench.py measures); config.QWEN25VL_MODELS marks which Qwen2.5-VL sizes are listed."""
    return [model for models in ALL_VQA_MODELS for model, spec in models.items() if spec.get("listed", True)]


def accepted_vqascore_models():
    """Every model name the factory builds: the listed ones and the sizes accepted by name only (qwen2.5-vl-3b)."""
    return [model for models in ALL_VQA_MODELS for model in models]


def get_vqascore_model(model_name, device='cuda', cache_dir=HF_CACHE_DIR, **kwargs):
    assert model_name in accepted_vqascore_models()
    if model_name in CLIP_T5_MODELS:
        return CLIPT5Model(model_name, device=device, cache_dir=cache_dir, **kwargs)
    if model_name in QWEN2_VL_MODELS:
        return Qwen2VLModel(model_name, device=device, cache_dir=cache_dir, **kwargs)
    raise NotImplementedError()

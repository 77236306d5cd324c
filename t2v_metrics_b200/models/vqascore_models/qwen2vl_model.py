"""Qwen2.5-VL VQAScore plugin backed by the H100 engine (image inputs).

Same plugin contract as the reference's `Qwen2VLModel` (t2v_metrics/models/vqascore_models/qwen2vl_model.py:93-301): class
attributes, `forward(images, texts, question_template, answer_template, temperature) -> CPU fp32 Tensor[n]` with
score = softmax(last-position logits / temperature)[first answer token]. The reference loops over samples and calls
`generate(max_new_tokens=1)`; here the whole batch is ONE prefill in libvqa_b200.so and identical images are encoded once.
Video inputs (decord / qwen_vl_utils frame sampling) are outside this engine's scope and raise.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from ...config import QWEN25VL_MODELS as _TABLE, Qwen25VLConfig
from ...constants import HF_CACHE_DIR
from .qwen_utils import qwen_image_to_patches, build_prompt_ids, default_question_template, default_answer_template
from .vqa_model import VQAScoreModel

QWEN2_VL_MODELS: Dict[str, dict] = {name: dict(model=dict(path=spec["weights"]), config=spec["config"]) for name, spec in _TABLE.items()}


# Pixel bounds of the resize the reference applies BEFORE the HF processor: `process_vision_info` (qwen_vl_utils.vision_process.fetch_image)
# calls smart_resize(h, w, factor=28, min_pixels=MIN_PIXELS, max_pixels=MAX_PIXELS) with MIN_PIXELS = 4 * 28 * 28 and
# MAX_PIXELS = 16384 * 28 * 28, and the processor then runs with do_resize=False (reference qwen2vl_model.py:201-216), so the processor's own
# 14*14*4*1280 ceiling never applies. qwen_vl_utils is an unpinned dependency that is not installed here: the two values are restated from
# its source and exposed as constructor arguments (`min_pixels=`, `max_pixels=`) for other versions.
QWEN_VL_UTILS_MIN_PIXELS = 4 * 28 * 28
QWEN_VL_UTILS_MAX_PIXELS = 16384 * 28 * 28


def _generation_config_penalty(checkpoint_path: str) -> float:
    """repetition_penalty of the generation_config.json stored beside the checkpoint (what `from_pretrained` would attach to
    `model.generation_config` in the reference, qwen2vl_model.py:116-130); 1.0 when there is none."""
    from ...checkpoint import generation_config_value
    return float(generation_config_value(checkpoint_path, "repetition_penalty", 1.0) or 1.0)


class Qwen2VLModel(VQAScoreModel):
    video_mode = "direct"
    allows_image = True
    supports_trace = True

    def __init__(self, model_name="qwen2.5-vl-7b", device="cuda", cache_dir=HF_CACHE_DIR, tokenizer=None,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, config: Optional[Qwen25VLConfig] = None,
                 checkpoint: Optional[str] = None, repetition_penalty: Optional[float] = None,
                 min_pixels: int = QWEN_VL_UTILS_MIN_PIXELS, max_pixels: int = QWEN_VL_UTILS_MAX_PIXELS, **kwargs):
        assert model_name in QWEN2_VL_MODELS
        self.min_pixels, self.max_pixels = int(min_pixels), int(max_pixels)
        # The reference's scores come out of `generate(..., output_scores=True)`, i.e. AFTER the logits processors the checkpoint's
        # generation_config.json configures (SURVEY F8; Qwen2.5-VL-Instruct ships repetition_penalty 1.05). None = read it from the
        # generation_config.json next to `checkpoint` when there is one, else 1.0 (off).
        self.repetition_penalty = repetition_penalty
        self._tokenizer_override, self._state_dict, self._config_override, self._checkpoint = tokenizer, state_dict, config, checkpoint
        super().__init__(model_name=model_name, device=device, cache_dir=cache_dir)

    def load_model(self):
        from ...engine import QwenVLEngine
        spec = QWEN2_VL_MODELS[self.model_name]
        self.cfg: Qwen25VLConfig = self._config_override or spec["config"]()
        if self._tokenizer_override is not None:
            self.tokenizer = self._tokenizer_override
        else:
            from transformers import AutoTokenizer
            self.tokenizer = AutoTokenizer.from_pretrained(spec["model"]["path"], cache_dir=self.cache_dir)
        from ...checkpoint import load_state_dict, normalise_qwen_keys
        sd = self._state_dict
        if sd is None:
            # a local file or a downloaded repository directory (index json + shards), as `from_pretrained(path)` takes (qwen2vl_model.py:116-130)
            sd = load_state_dict(self._checkpoint or spec["model"]["path"])
        sd = normalise_qwen_keys(sd)      # published checkpoints use `visual.*` / `model.layers.*`; transformers renames them while loading
        if self.repetition_penalty is None:
            self.repetition_penalty = _generation_config_penalty(self._checkpoint or spec["model"]["path"])
        dev = torch.device(self.device if self.device != "cuda" else "cuda:0")
        self.engine = QwenVLEngine(self.cfg, dev)
        self.engine.load_state_dict(sd)
        self._state_dict = None

    def load_images(self, image: List[str]):
        """-> (patches fp32 [sum P, 1176] on the device, [(1, gh, gw), ...])"""
        if any(p[-4:].lower() in (".mp4", ".avi", ".mov", ".mkv") for p in image):
            raise NotImplementedError("video inputs are outside the engine's hot-path scope")
        # PIL decode on the host, everything else (smart_resize, PIL-exact bicubic, normalise, frame duplication, merge-order patch
        # rows) in ONE device kernel -- bit-identical to qwen_utils.qwen_image_to_patches, the CPU path the reference runs per image
        import numpy as np
        from PIL import Image
        from ...engine import qwen_preprocess_u8
        raw = []
        for p in image:
            if p.lower().endswith(".npy"):
                # the reference's Qwen path takes the array as RGB, no channel flip (qwen2vl_model.py:146-153); 4-D arrays are frame stacks
                arr = np.load(p)
                if arr.ndim == 4:
                    raise NotImplementedError("4-D .npy frame stacks are video inputs: outside the engine's hot-path scope")
                if arr.ndim != 3:
                    raise ValueError(f"Unexpected shape for NumPy array in {p}")
                arr = np.asarray(Image.fromarray(arr.astype("uint8"), "RGB"), dtype=np.uint8)
            else:
                with Image.open(p) as im:
                    arr = np.asarray(im.convert("RGB"), dtype=np.uint8)
            raw.append(torch.from_numpy(np.ascontiguousarray(arr)))
        return qwen_preprocess_u8(raw, self.engine.device, self.cfg.patch_size, self.cfg.temporal_patch_size, self.cfg.spatial_merge_size,
                                  min_pixels=self.min_pixels, max_pixels=self.max_pixels)

    @torch.no_grad()
    def forward_with_trace(self, images: List[str], texts: List[str], fps=None, question_template: str = default_question_template,
                           answer_template: str = default_answer_template, max_new_tokens: int = 1, temperature: float = 1.0,
                           score_position: str = "end", debug: bool = False, repetition_penalty: Optional[float] = None):
        """Scores plus the per-sample trace dictionaries of the reference's forward_with_trace (qwen2vl_model.py:303-493; schema at
        :469-487): the greedy token, the answer token's probability and the five most probable alternatives. With one generated position
        `score_position` "start" and "end" coincide. The alternatives come from a top-k pass over the last position's logits
        (engine.topk_last) under the same temperature / repetition penalty as the score."""
        assert score_position in ("start", "end"), f"score_position must be 'start' or 'end', got '{score_position}'"
        probs = self.forward(images, texts, fps=fps, question_template=question_template, answer_template=answer_template,
                             max_new_tokens=max_new_tokens, temperature=temperature, debug=False, repetition_penalty=repetition_penalty)
        pen = self.repetition_penalty if repetition_penalty is None else repetition_penalty
        ids, top_p = self.engine.topk_last(5, temperature=temperature, repetition_penalty=pen)
        ids, top_p = ids.cpu().tolist(), top_p.cpu().tolist()
        dec = lambda t: self.tokenizer.decode([t]) if hasattr(self.tokenizer, "decode") else str(t)
        special = {getattr(self.tokenizer, n, None) for n in ("eos_token_id", "bos_token_id", "pad_token_id")} - {None}
        traces = []
        for b, (p, answer_id) in enumerate(zip(probs.tolist(), self._last_answer_ids)):
            generated = ids[b][0]                                   # generate(max_new_tokens=1, do_sample=False) emits the arg-max
            if generated in special:
                # the reference drops a trailing special token and then has nothing left to score (qwen2vl_model.py:395-419)
                raise ValueError("No tokens available to score at the specified position")
            alternatives = [dict(token_id=t, token_text=dec(t), probability=q) for t, q in zip(ids[b], top_p[b])]
            detail = dict(position=0, expected_token_id=answer_id, expected_token_text=dec(answer_id), probability=p, top_alternatives=alternatives)
            traces.append(dict(generated_text=dec(generated), generated_length=1, score_position=score_position, score_start_idx=0,
                               scored_indices=[0], scored_tokens_text=dec(generated), probability=p, token_details=[detail]))
            if debug:
                print(f"sample {b}: generated {dec(generated)!r}; P(answer {dec(answer_id)!r}) = {p:.6f}; top-5 "
                      f"{[(a['token_text'], round(a['probability'], 6)) for a in alternatives]}")
        return probs, traces

    def _eos_ids(self) -> List[int]:
        """generation_config.json's eos_token_id beside the checkpoint (an id or a list), else the tokenizer's."""
        from ...checkpoint import generation_config_value
        spec = QWEN2_VL_MODELS[self.model_name]
        eos = generation_config_value(self._checkpoint or spec["model"]["path"], "eos_token_id", None)
        if eos is None:
            eos = getattr(self.tokenizer, "eos_token_id", None)
        if eos is None:
            return []
        return [int(e) for e in eos] if isinstance(eos, (list, tuple)) else [int(eos)]

    @torch.no_grad()
    def generate(self, images: List[str], texts: List[str], fps=None, max_new_tokens: int = 2048, temperature: float = 0.0,
                 do_sample: Optional[bool] = None, top_p: float = 0.9, eos_token_ids: Optional[List[int]] = None) -> List[str]:
        """Greedy text generation, the reference's Qwen2VLModel.generate (qwen2vl_model.py:495-563) with its default temperature 0: per
        sample, the chat prompt of the raw text and the image, generate(do_sample=False) under the checkpoint's repetition penalty, the
        prompt cut off, decoded with skip_special_tokens and stripped. Here the whole batch is one prefill and one decode loop on the
        device; identical images are encoded once. Sampling (temperature > 0 or do_sample=True, top-p) is not implemented."""
        assert len(images) == len(texts), "Number of images/videos and texts must match"
        if do_sample is None:
            do_sample = temperature > 0
        if do_sample or temperature > 0:
            raise NotImplementedError("only greedy decoding is supported (temperature=0.0, do_sample=False); top-p sampling is not implemented")
        uniq: Dict[str, int] = {}
        index = [uniq.setdefault(p, len(uniq)) for p in images]
        patches, grids = self.load_images(list(uniq.keys()))
        unit = self.cfg.spatial_merge_size ** 2
        cache = self.__dict__.setdefault("_prompt_cache", {})
        if len(cache) > 65536:
            cache.clear()
        prompts = []
        for text, img in zip(texts, index):
            t, gh, gw = grids[img]
            prompts.append(build_prompt_ids(self.tokenizer, text, t * gh * gw // unit, self.cfg.image_token_id, cache))
        eos = self._eos_ids() if eos_token_ids is None else [int(e) for e in eos_token_ids]
        ids = self.engine.generate_prompts(patches, grids, prompts, max_new_tokens, eos, image_of_sample=index,
                                           repetition_penalty=self.repetition_penalty)
        return [self.tokenizer.decode(x, skip_special_tokens=True, clean_up_tokenization_spaces=False).strip() for x in ids]

    @torch.no_grad()
    def forward(self, images: List[str], texts: List[str], fps=None, question_template: str = default_question_template,
                answer_template: str = default_answer_template, max_new_tokens: int = 1, temperature: float = 1.0,
                debug: bool = False, repetition_penalty: Optional[float] = None) -> torch.Tensor:
        assert len(images) == len(texts), "Number of images/videos and texts must match"
        if max_new_tokens != 1:
            # With max_new_tokens = k > 1 the reference scores answer token i on the logits of generation step len(scores) - n + i, i.e.
            # conditioned on its own GREEDY continuation (qwen2vl_model.py:259-289) -- a decode loop, not the single prefill this engine runs.
            raise NotImplementedError("the engine scores the first generated position only (max_new_tokens=1, the reference default)")
        questions = [question_template.format(t) for t in texts]
        answers = [answer_template.format(t) for t in texts]
        uniq: Dict[str, int] = {}
        index = [uniq.setdefault(p, len(uniq)) for p in images]
        patches, grids = self.load_images(list(uniq.keys()))
        unit = self.cfg.spatial_merge_size ** 2
        prompts, answer_ids = [], []
        cache = self.__dict__.setdefault("_prompt_cache", {})
        if len(cache) > 65536:
            cache.clear()
        for q, a, img in zip(questions, answers, index):
            t, gh, gw = grids[img]
            prompts.append(build_prompt_ids(self.tokenizer, q, t * gh * gw // unit, self.cfg.image_token_id, cache))
            ids = cache.get(("answer", a))
            if ids is None:
                ids = cache[("answer", a)] = tuple(self.tokenizer.encode(a, add_special_tokens=False))
            if not ids:
                raise ValueError("empty answer")
            # one generated position => the reference truncates a multi-token answer to its first token ("Generated 1 tokens but need n,
            # adjusting", qwen2vl_model.py:259-263) and the geometric mean over one token is that token's probability
            answer_ids.append(ids[0])
        self._last_answer_ids = list(answer_ids)
        probs = self.engine.score_prompts(patches, grids, prompts, answer_ids, image_of_sample=index, temperature=temperature,
                                          repetition_penalty=self.repetition_penalty if repetition_penalty is None else repetition_penalty)
        return probs.float().cpu()

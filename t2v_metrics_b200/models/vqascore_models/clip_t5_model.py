"""CLIP-FlanT5 VQAScore plugin backed by the H100 engine.

Same plugin contract as the reference's (v3.0) `CLIPT5Model(VQAScoreModel)` -- class attributes `video_mode`,
`allows_image`, `forward(images, texts, question_template, answer_template) -> CPU fp32 Tensor[n]` -- which is what
`Score.forward` calls once per image (reference t2v_metrics/score.py:104-106). The forward itself is one call into
libvqa_b200.so (engine.ClipT5Engine.score_tensors); nothing on this path runs through transformers or torch ops.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from ...config import CLIPT5_MODELS as _MODEL_TABLE, ClipT5Config
from ...constants import HF_CACHE_DIR, CONTEXT_LEN, SYSTEM_MSG, IGNORE_INDEX, DEFAULT_IMAGE_TOKEN, IMAGE_TOKEN_INDEX
from .mm_utils import t5_tokenizer_image_token, clip_preprocess, video_canvas
from .sampling import sampling_params
from .vqa_model import VQAScoreModel

default_question_template = 'Does this figure show "{}"? Please answer yes or no.'  # V_3.0_README.md:211-215
default_answer_template = "Yes"
VIDEO_EXTENSIONS = ('.mp4', '.avi', '.mov', '.mkv')      # the suffixes the reference's score.py:72 treats as videos

CLIP_T5_MODELS: Dict[str, dict] = {
    name: dict(tokenizer=dict(path=spec["tokenizer"], model_max_length=CONTEXT_LEN, padding_side="right"),
               model=dict(path=spec["weights"], conversation="t5_chat", image_aspect_ratio="pad"),
               config=spec["config"])
    for name, spec in _MODEL_TABLE.items()
}


def format_question(question: str, conversation_style: str = "t5_chat") -> str:
    """v3.0 format_question: SYSTEM_MSG + ' USER: <image>\\n' + question + ' ASSISTANT: ' (SURVEY App. A)."""
    if conversation_style == "t5_chat":
        return SYSTEM_MSG + " USER: " + DEFAULT_IMAGE_TOKEN + "\n" + question + " ASSISTANT: "
    if conversation_style == "t5_plain":
        return DEFAULT_IMAGE_TOKEN + "\n" + question
    raise NotImplementedError(conversation_style)


def format_answer(answer: str, conversation_style: str = "t5_chat") -> str:
    return answer


def prompt_token_ids(tokenizer, questions: List[str], context_len: int, vocab: int, cache: dict) -> List[List[int]]:
    """t5_tokenizer_image_token of each formatted prompt, truncated to context_len. The splice kernel replaces exactly ONE image slot per
    prompt and embeds every other id: a caption that itself contains the literal "<image>" would add a second slot (t5_tokenizer_image_token
    splits on it), and an id outside the vocabulary would index past the embedding table. Refuse both on the host."""
    ids = [t5_tokenizer_image_token(q, tokenizer, chunk_cache=cache)[:context_len] for q in questions]
    for q, row in zip(questions, ids):
        if sum(1 for t in row if t == IMAGE_TOKEN_INDEX) != 1:
            raise ValueError(f"each prompt must contain exactly one {DEFAULT_IMAGE_TOKEN!r} placeholder (the caption must not contain it): {q!r}")
        if any((t < 0 and t != IMAGE_TOKEN_INDEX) or t >= vocab for t in row):
            raise ValueError("token id outside [0, vocab)")
    return ids


class CLIPT5Model(VQAScoreModel):
    """VQAScore with CLIP-FlanT5 on the H100 engine."""
    video_mode = "concat"
    # video files may be passed to forward(): the plugin concatenates their frames into one canvas per video itself (Score.forward hands
    # a "concat" plugin video files only when it sets this)
    builds_video_canvases = True
    allows_image = True

    def __init__(self, model_name="clip-flant5-xxl", device="cuda", cache_dir=HF_CACHE_DIR, tokenizer=None,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, config: Optional[ClipT5Config] = None,
                 checkpoint: Optional[str] = None, vision_tower_checkpoint: Optional[str] = None, cuda_graph_max_pairs: int = 16, **kwargs):
        assert model_name in CLIP_T5_MODELS
        # calls with at most this many pairs replay a CUDA graph captured per (pairs, images, padded text length, answer length): the
        # ~700 launches of a forward cost more host time than device time at batch 1 (0 disables)
        self.cuda_graph_max_pairs = int(cuda_graph_max_pairs)
        self._vision_checkpoint = vision_tower_checkpoint
        self._tokenizer_override = tokenizer
        self._state_dict = state_dict
        self._config_override = config
        self._checkpoint = checkpoint
        super().__init__(model_name=model_name, device=device, cache_dir=cache_dir)

    # ---- loading -------------------------------------------------------------------------------------------------
    def load_model(self):
        """Tokenizer via transformers (slow SentencePiece tokenizer, as mm_utils.py:198), weights from a local
        HF-named state dict (`state_dict=` / `checkpoint=` safetensors or .pt) cast to bf16 on the device
        (mm_utils.py:228) and bound into the engine."""
        from ...engine import ClipT5Engine

        spec = CLIP_T5_MODELS[self.model_name]
        self.conversational_style = spec["model"]["conversation"]
        self.image_aspect_ratio = spec["model"]["image_aspect_ratio"]
        self.context_len = spec["tokenizer"]["model_max_length"]
        self.cfg: ClipT5Config = self._config_override or spec["config"]()
        if self._tokenizer_override is not None:
            self.tokenizer = self._tokenizer_override
        else:
            from transformers import AutoTokenizer
            self.tokenizer = AutoTokenizer.from_pretrained(spec["tokenizer"]["path"], use_fast=False, cache_dir=self.cache_dir,
                                                           model_max_length=self.context_len, padding_side="right")
        sd = self._state_dict
        if sd is None:
            sd = self._load_checkpoint(self._checkpoint or spec["model"]["path"])
        dev = torch.device(self.device if self.device != "cuda" else "cuda:0")
        self.engine = ClipT5Engine(self.cfg, dev)
        self.engine.load_state_dict(sd)
        self._state_dict = None

    def _load_checkpoint(self, path: str) -> Dict[str, torch.Tensor]:
        """`path`: a local weights file or a downloaded repository directory (index json + shards) of zhiqiulin/clip-flant5-*;
        `vision_tower_checkpoint=`: the CLIP tower the reference loads separately when the checkpoint does not carry it
        (openai/clip-vit-large-patch14-336, mm_utils.py:226-227)."""
        from ...checkpoint import load_state_dict, normalise_clipt5_keys
        vision = load_state_dict(self._vision_checkpoint) if self._vision_checkpoint else None
        return normalise_clipt5_keys(load_state_dict(path), vision)

    # ---- pre-processing ------------------------------------------------------------------------------------------
    def load_images(self, image: List[str], num_frames: int = 8) -> torch.Tensor:
        """image_loader (PIL decode, host) -> uint8 HWC -> a device kernel doing expand2square(mean colour) + PIL-exact bicubic
        resize + centre crop + /255 + normalise (engine.clip_preprocess_u8; bit-identical to the CPU path `clip_preprocess`, which
        is what the reference runs per image on the host: mm_utils.py:128-139 + CLIPImageProcessor). fp32 [n,3,S,S] on the device.
        A video file becomes the canvas of `num_frames` frames side by side that the reference scores for it (mm_utils.video_canvas).
        One launch per slice of engine.CLIP_SLICE_BYTES of pixels (a call of still images of ordinary size is one launch)."""
        import numpy as np
        from ...engine import clip_preprocess_u8_sliced
        raw = [torch.from_numpy(video_canvas(p, num_frames) if p[-4:].lower() in VIDEO_EXTENSIONS else
                                np.ascontiguousarray(np.asarray(self.image_loader(p).convert("RGB"), dtype=np.uint8))) for p in image]
        return clip_preprocess_u8_sliced(raw, self.cfg.image_size, self.engine.device, pad=self.image_aspect_ratio == "pad")

    def _prompt_ids(self, questions: List[str]) -> List[List[int]]:
        cache = self.__dict__.setdefault("_chunk_cache", {})
        if len(cache) > 65536:
            cache.clear()
        return prompt_token_ids(self.tokenizer, questions, self.context_len, self.cfg.vocab, cache)

    def _tokenize(self, questions: List[str], answers: List[str]):
        cache = self.__dict__.setdefault("_chunk_cache", {})
        if len(cache) > 65536:
            cache.clear()
        ids = prompt_token_ids(self.tokenizer, questions, self.context_len, self.cfg.vocab, cache)
        labs = [t5_tokenizer_image_token(a, self.tokenizer, chunk_cache=cache)[: self.context_len] for a in answers]
        pad = getattr(self.tokenizer, "pad_token_id", 0) or 0
        for row in labs:
            if any(t < 0 or t >= self.cfg.vocab for t in row):
                raise ValueError(f"answer token id outside [0, vocab) (answers must not contain {DEFAULT_IMAGE_TOKEN!r})")
        L, T = max(map(len, ids)), max(map(len, labs))
        if 0 < len(ids) <= getattr(self, "cuda_graph_max_pairs", 0):
            L = (L + 15) // 16 * 16          # few distinct shapes -> few graphs; padded columns are masked by `lens` in the engine
        input_ids = torch.full((len(ids), L), pad, dtype=torch.int32)
        labels = torch.full((len(labs), T), IGNORE_INDEX, dtype=torch.int32)
        lens = torch.zeros(len(ids), dtype=torch.int32)
        for i, (a, b) in enumerate(zip(ids, labs)):
            input_ids[i, : len(a)] = torch.tensor(a, dtype=torch.int32)
            labels[i, : len(b)] = torch.tensor(b, dtype=torch.int32)
            lens[i] = len(a)
        return input_ids, lens, labels

    # ---- generation ----------------------------------------------------------------------------------------------
    GENERATE_MAX_PAIRS = 64

    def _eos_ids(self) -> List[int]:
        """generation_config.json's eos_token_id beside the checkpoint (an id or a list), else the tokenizer's."""
        from ...checkpoint import generation_config_value
        spec = CLIP_T5_MODELS[self.model_name]
        eos = generation_config_value(self._checkpoint or spec["model"]["path"], "eos_token_id", None)
        if eos is None:
            eos = getattr(self.tokenizer, "eos_token_id", None)
        if eos is None:
            return []
        return [int(e) for e in eos] if isinstance(eos, (list, tuple)) else [int(eos)]

    @torch.no_grad()
    def generate(self, images: List[str], texts: List[str], max_new_tokens: int = 256, temperature: float = 0.0,
                 do_sample: Optional[bool] = None, top_p: float = 0.9, eos_token_ids: Optional[List[int]] = None,
                 generator: Optional[torch.Generator] = None) -> List[str]:
        """Text generation with CLIP-FlanT5 (V_3.0_README.md:316-325: `model.generate(images=..., texts=...) -> List[str]`).

        Per sample the prompt is format_question(text) -- the raw text, no question template -- through t5_tokenizer_image_token,
        truncated to context_len, i.e. the scoring path's prompt; identical image paths are encoded once. Decoding is HF
        T5ForConditionalGeneration.generate(inputs_embeds=<spliced prompt>, attention_mask=<its mask>, num_beams=1) from decoder_start_id;
        a sample stops on an EOS id (kept, then dropped by the decode) or after max_new_tokens tokens. EOS ids come from
        generation_config.json beside the checkpoint, else the tokenizer; `eos_token_ids=` overrides both. Output:
        tokenizer.decode(ids, skip_special_tokens=True).strip().

        With the default temperature 0 decoding is greedy (do_sample=False): each token is the arg-max of the fp32-cast bf16 logits over
        the whole vocabulary (ties to the lowest id), with no logits processors (FlanT5's generation config has no repetition penalty).
        With do_sample (None: temperature > 0) and temperature > 0 it samples as generate(do_sample=True, temperature, top_p) does, with
        generation_config.json's top_k (default 50): see sampling_params; a generation_config.json with a repetition penalty is refused,
        since the sampled T5 step applies none. Each pair's draws come from a 63-bit seed taken, in the caller's order, from `generator`
        (None: torch's default generator, so torch.manual_seed(s) before the call reproduces it). Identical (image, text) pairs of a sampled
        call run the vision tower and the encoder once and draw their samples from that one encoding.

        The v3.0 wrapper's own generate signature is not recoverable from the reference (SURVEY App. A): the sampling keywords and their
        defaults (top_p=0.9) are those of the reference's Qwen2VLModel.generate. Its default length is not recoverable either; 256 is this
        implementation's choice and sizes the K/V cache (393 KB per sample per token at xxl width). The batch runs as one encoder pass and
        one decode loop on the device, in calls of at most GENERATE_MAX_PAIRS pairs."""
        assert len(images) == len(texts), "Number of images and texts must match"
        if any(p[-4:].lower() in VIDEO_EXTENSIONS for p in images):
            raise NotImplementedError("generate takes image files; video files are scored by forward only")
        sampling = None
        if do_sample or temperature > 0:
            # the engine's capability is looked up on its class, so nothing of the instance is touched before the refusal
            if not callable(getattr(type(getattr(self, "engine", None)), "sample_tensors", None)):
                raise NotImplementedError("this engine has only greedy decoding (temperature=0.0, do_sample=False): it has no "
                                          "sample_tensors for top-k / top-p sampling")
            from ...checkpoint import generation_config_value
            ckpt = self._checkpoint or CLIP_T5_MODELS[self.model_name]["model"]["path"]
            sampling = sampling_params(ckpt, do_sample, temperature, top_p)
            penalty = generation_config_value(ckpt, "repetition_penalty", 1.0)
            if sampling is not None and penalty != 1.0:
                raise NotImplementedError(f"generation_config.json sets repetition_penalty = {penalty!r}: the sampled CLIP-FlanT5 step applies "
                                          "no repetition penalty")
        prompts = self._prompt_ids([format_question(t, self.conversational_style) for t in texts])
        eos = self._eos_ids() if eos_token_ids is None else [int(e) for e in eos_token_ids]
        if sampling is not None:
            seeds = torch.randint(0, 2 ** 63 - 1, (len(prompts),), dtype=torch.int64, generator=generator).tolist()
            return self._sample(images, texts, prompts, seeds, sampling, max_new_tokens, eos)
        out: List[str] = []
        for lo in range(0, len(images), self.GENERATE_MAX_PAIRS):
            chunk_images, chunk_prompts = images[lo:lo + self.GENERATE_MAX_PAIRS], prompts[lo:lo + self.GENERATE_MAX_PAIRS]
            pixels, input_ids, lens, image_index = self._generate_inputs(chunk_images, chunk_prompts)
            ids = self.engine.generate_tensors(pixels, input_ids, lens, max_new_tokens, eos, image_index=image_index)
            out.extend(self.tokenizer.decode(x, skip_special_tokens=True).strip() for x in ids)
        return out

    def _generate_inputs(self, images: List[str], prompts: List[List[int]]):
        """Device inputs of one engine generation call: pixels of the distinct image paths, padded input_ids, text_lens and image_index
        (None when every path differs)."""
        uniq: Dict[str, int] = {}
        index = [uniq.setdefault(p, len(uniq)) for p in images]
        pixels = self.load_images(list(uniq.keys()))
        dev = self.engine.device
        L = max(map(len, prompts))
        pad = getattr(self.tokenizer, "pad_token_id", 0) or 0
        input_ids = torch.full((len(prompts), L), pad, dtype=torch.int32)
        for i, row in enumerate(prompts):
            input_ids[i, :len(row)] = torch.tensor(row, dtype=torch.int32)
        lens = torch.tensor([len(r) for r in prompts], dtype=torch.int32)
        image_index = torch.tensor(index, dtype=torch.int32).to(dev) if len(uniq) != len(images) else None
        return pixels, input_ids.to(dev), lens.to(dev), image_index

    def _sample(self, images, texts, prompts, seeds, sampling, max_new_tokens: int, eos) -> List[str]:
        """The sampled generate: identical (image, text) pairs form a group whose samples share one encoding; groups are packed into engine
        calls of at most GENERATE_MAX_PAIRS samples, a group kept whole where it fits; strings come back in the caller's order."""
        groups: Dict[tuple, List[int]] = {}
        for i, pair in enumerate(zip(images, texts)):
            groups.setdefault(pair, []).append(i)
        cap = self.GENERATE_MAX_PAIRS
        chunks: List[List[int]] = [[]]
        for members in groups.values():
            while members:
                if len(chunks[-1]) + len(members) > cap and chunks[-1] and len(members) <= cap:
                    chunks.append([])          # a group that fits in a call of its own is not split
                room = cap - len(chunks[-1])
                chunks[-1] += members[:room]
                members = members[room:]
                if len(chunks[-1]) == cap:
                    chunks.append([])
        out: List[Optional[str]] = [None] * len(images)
        T, k, p = sampling
        for chunk in (c for c in chunks if c):
            firsts: Dict[tuple, int] = {}
            prompt_of_sample = [firsts.setdefault((images[i], texts[i]), len(firsts)) for i in chunk]
            distinct = list(firsts)
            rep = {pair: next(i for i in chunk if (images[i], texts[i]) == pair) for pair in distinct}
            pixels, input_ids, lens, image_index = self._generate_inputs([pair[0] for pair in distinct], [prompts[rep[pair]] for pair in distinct])
            ids = self.engine.sample_tensors(pixels, input_ids, lens, max_new_tokens, eos, [seeds[i] for i in chunk], T, k, p,
                                             image_index=image_index, prompt_of_sample=prompt_of_sample)
            for i, x in zip(chunk, ids):
                out[i] = self.tokenizer.decode(x, skip_special_tokens=True).strip()
        return out

    # ---- scoring -------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, images: List[str], texts: List[str], question_template: str = default_question_template,
                answer_template: str = default_answer_template, num_frames: int = 8) -> torch.Tensor:
        """One score per (images[i], texts[i]) pair. An image path ending in .mp4 / .avi / .mov / .mkv is a video: it is scored as the
        horizontal concatenation of `num_frames` equally spaced frames, as the reference's Score.forward does for this model."""
        assert len(images) == len(texts), "Number of images and texts must match"
        if num_frames < 1:
            raise ValueError(f"num_frames must be >= 1, got {num_frames}")
        questions = [format_question(question_template.format(t), self.conversational_style) for t in texts]
        answers = [format_answer(answer_template.format(t), self.conversational_style) for t in texts]
        input_ids, lens, labels = self._tokenize(questions, answers)
        # identical paths are encoded once (Score.forward repeats one image N times, score.py:104-106)
        uniq: Dict[str, int] = {}
        index = []
        for p in images:
            index.append(uniq.setdefault(p, len(uniq)))
        pixels = self.load_images(list(uniq.keys()), num_frames)
        dev = self.engine.device
        image_index = torch.tensor(index, dtype=torch.int32).to(dev, non_blocking=True)
        args = (pixels, input_ids.to(dev, non_blocking=True), lens.to(dev, non_blocking=True), labels.to(dev, non_blocking=True))
        kw = dict(image_index=image_index if len(uniq) != len(images) else None)
        if 0 < len(images) <= self.cuda_graph_max_pairs:
            try:
                return self.engine.score_tensors_graphed(*args, **kw).float().cpu()
            except RuntimeError as e:        # stream capture refused (e.g. another thread is issuing CUDA calls): same kernels, launched directly
                import warnings
                warnings.warn(f"CUDA-graph capture failed ({e}); small calls will be launched directly from now on")
                self.cuda_graph_max_pairs = 0
                torch.cuda.synchronize(dev)
        return self.engine.score_tensors(*args, **kw).float().cpu()

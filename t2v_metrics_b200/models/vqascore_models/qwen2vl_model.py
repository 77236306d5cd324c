"""Qwen2.5-VL VQAScore plugin backed by the H100 engine (image and video inputs).

Same plugin contract as the reference's `Qwen2VLModel` (t2v_metrics/models/vqascore_models/qwen2vl_model.py:93-301): class
attributes, `forward(images, texts, question_template, answer_template, temperature) -> CPU fp32 Tensor[n]` with
score = softmax(last-position logits / temperature)[first answer token]. The reference loops over samples and calls
`generate(max_new_tokens=1)`; here the whole batch is ONE prefill in libvqa_b200.so and identical images are encoded once.
With `max_new_tokens = k > 1`, `forward` and `forward_with_trace` score the answer tokens on a greedy rollout of k tokens, as the
reference does with one `generate(max_new_tokens=k, output_scores=True)` per sample (qwen2vl_model.py:239-289, :381-487): here the
pairs run as batched rollouts on the GPU decode loop, with the answer probabilities of every step computed on the device.
Videos arrive as decoded frame stacks: a 4-D `.npy` [n, h, w, 3] is scored as a video, as the reference's decoder-free path does
(qwen2vl_model.py:145-153, a list of frames as `{"type": "video"}`), with its frames pre-processed on the device in the same launch as the
still images of the call, video tokens in the prompt and the processor's `second_per_grid_ts`. Stills and videos mix freely in one call.
Video files (.mp4, .avi, .mov, .mkv) are scored when the plugin has a decoder (`video_reader=`, opt-in), as the reference's file path does
(qwen2vl_model.py:135-144): qwen_vl_utils' frame sampling at `fps` and pixel budget on the host, torchvision's antialiased bicubic resize
of the sampled frames on the device. Without a decoder they raise, before anything is launched.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from ...config import QWEN25VL_MODELS as _TABLE, Qwen25VLConfig
from ...constants import HF_CACHE_DIR
from .qwen_utils import qwen_image_to_patches, build_prompt_ids, default_question_template, default_answer_template
from .sampling import _UNSUPPORTED_WARPERS, HF_DEFAULT_TOP_K, sampling_params  # noqa: F401  (importable from here as before)
from .vqa_model import VQAScoreModel

QWEN2_VL_MODELS: Dict[str, dict] = {name: dict(model=dict(path=spec["weights"]), config=spec["config"], listed=spec["listed"])
                                    for name, spec in _TABLE.items()}


# Pixel bounds of the resize the reference applies BEFORE the HF processor: `process_vision_info` (qwen_vl_utils.vision_process.fetch_image)
# calls smart_resize(h, w, factor=28, min_pixels=MIN_PIXELS, max_pixels=MAX_PIXELS) with MIN_PIXELS = 4 * 28 * 28 and
# MAX_PIXELS = 16384 * 28 * 28, and the processor then runs with do_resize=False (reference qwen2vl_model.py:201-216), so the processor's own
# 14*14*4*1280 ceiling never applies. qwen_vl_utils is an unpinned dependency that is not installed here: the two values are restated from
# its source and exposed as constructor arguments (`min_pixels=`, `max_pixels=`) for other versions.
QWEN_VL_UTILS_MIN_PIXELS = 4 * 28 * 28
QWEN_VL_UTILS_MAX_PIXELS = 16384 * 28 * 28

# A frame stack reaches the processor as a list of frames, whose VideoMetadata has fps None, and `VideoMetadata.sampled_fps` is then
# `self.fps or 24` (transformers 5.5.0 video_utils.py:108-111). Qwen2_5_VLProcessor divides temporal_patch_size by it
# (processing_qwen2_5_vl.py:103-113), so a stack's second_per_grid_ts is temporal_patch_size / 24 whatever `fps` the caller passes, and
# the temporal rope step tokens_per_second * int(2 / 24) is 0 (modeling_qwen2_5_vl.py:1019, :1120).
HF_FRAME_LIST_FPS = 24

_VIDEO_FILES = (".mp4", ".avi", ".mov", ".mkv")

# The reference's video element for a file (qwen2vl_model.py:135-144): {"type": "video", "video": path, "max_pixels": 360*420, "fps": fps},
# with fps None -> the model table's 8.0, and fps "dynamic" -> no "fps" key, so qwen_vl_utils' FPS = 2.0 applies.
VIDEO_FILE_MAX_PIXELS = 360 * 420
VIDEO_FILE_DEFAULT_FPS = 8.0


def _is_video_file(path: str) -> bool:
    return path[-4:].lower() in _VIDEO_FILES


def _is_frame_stack(path: str) -> bool:
    """A 4-D .npy is a decoded video; only its header is read."""
    import numpy as np
    return path.lower().endswith(".npy") and np.load(path, mmap_mode="r").ndim == 4


def _chunks(n_pairs: int, max_pairs: int, budget: int, workspace_bytes, seq_len: int, sizes: List[int]) -> List[List[int]]:
    """Pairs in order, in chunks of at most max_pairs, halved while one chunk's workspace_bytes(pairs, seq_len, patch rows) exceeds the
    budget (a chunk's patch rows are bounded by all of them and by pairs x the largest item)."""
    chunk = min(max_pairs, n_pairs)
    while chunk > 1 and workspace_bytes(chunk, seq_len, min(sum(sizes), chunk * max(sizes))) > budget:
        chunk = (chunk + 1) // 2
    return [list(range(c0, min(n_pairs, c0 + chunk))) for c0 in range(0, n_pairs, chunk)]


def _subset(patches: torch.Tensor, grids, index: List[int], sel: List[int]):
    """The patch rows and grids of the items the pairs `sel` use, each once, and each pair's item in that subset."""
    items = sorted({index[i] for i in sel})
    local = {g: j for j, g in enumerate(items)}
    if len(items) == len(grids):
        pix = patches
    else:
        offs = [0]
        for t, h, w in grids:
            offs.append(offs[-1] + t * h * w)
        pix = torch.cat([patches[offs[g]:offs[g + 1]] for g in items])
    return pix, items, [local[index[i]] for i in sel]


def _require_rollout_engine(plugin) -> None:
    """max_new_tokens > 1 is scored on a greedy rollout, which only the device engine's scored decode loop (QwenVLEngine.rollout_scores)
    runs. A plugin without such an engine (none loaded, or an engine object without scored rollouts) refuses before any image is read or
    any kernel launched."""
    if not callable(getattr(getattr(plugin, "engine", None), "rollout_scores", None)):
        raise NotImplementedError("max_new_tokens > 1 needs an engine with scored greedy rollouts (QwenVLEngine.rollout_scores), and this "
                                  "plugin has none; without it only the single-prefill scoring of max_new_tokens=1 exists")


def _generation_config_penalty(checkpoint_path: str) -> float:
    """repetition_penalty of the generation_config.json stored beside the checkpoint (what `from_pretrained` would attach to
    `model.generation_config` in the reference, qwen2vl_model.py:116-130); 1.0 when there is none."""
    from ...checkpoint import generation_config_value
    return float(generation_config_value(checkpoint_path, "repetition_penalty", 1.0) or 1.0)


def _checkpoint_config(checkpoint_path: str, expected: Qwen25VLConfig, model_name: str) -> Qwen25VLConfig:
    """The architecture of the config.json in a checkpoint directory, which must agree with `expected` (the model table's entry or the
    caller's `config=`) on every field: a checkpoint of another size, or a fine-tune that changed a dimension, raises here before any
    weight is converted or bound. Without a config.json (a single weights file, or a directory without one) `expected` stands."""
    import os
    f = os.path.join(checkpoint_path, "config.json")
    if not (os.path.isdir(checkpoint_path) and os.path.isfile(f)):
        return expected
    found = Qwen25VLConfig.from_hf_config(f)
    diff = expected.mismatches(found)
    if diff:
        raise ValueError(f"{f} does not describe {model_name}: " + ", ".join(f"{k} = {b!r} (expected {a!r})" for k, (a, b) in diff.items()))
    return found


class Qwen2VLModel(VQAScoreModel):
    video_mode = "direct"
    allows_image = True
    supports_trace = True
    # Scoring with max_new_tokens > 1 runs batched rollouts of at most this many pairs, halved until one chunk's generation workspace
    # (prefill activations of the padded prompts + K/V cache of prompt and rollout, vqa_qwen25vl_generate_workspace_bytes) fits the
    # budget: large `max_pixels` images make prompts of thousands of tokens.
    ROLLOUT_MAX_PAIRS = 32
    ROLLOUT_WORKSPACE_BUDGET = 8 << 30
    # A video makes a prompt of thousands of tokens: a single-prefill scoring or `generate` call with a video is split, by the same halving
    # rule, into engine calls whose workspace (score_workspace_bytes / generate_workspace_bytes) fits this budget. Calls with still images
    # only run as one engine call, as they always have.
    VIDEO_WORKSPACE_BUDGET = 8 << 30

    def __init__(self, model_name="qwen2.5-vl-7b", device="cuda", cache_dir=HF_CACHE_DIR, tokenizer=None,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, config: Optional[Qwen25VLConfig] = None,
                 checkpoint: Optional[str] = None, repetition_penalty: Optional[float] = None,
                 min_pixels: int = QWEN_VL_UTILS_MIN_PIXELS, max_pixels: int = QWEN_VL_UTILS_MAX_PIXELS, video_reader=None, **kwargs):
        """`video_reader` decodes video files: "opencv" (qwen_utils.OpenCVVideoReader) or any object with
        open(path) -> (num_frames, avg_fps, get(indices) -> uint8 [k, h, w, 3] RGB). None (the default): video files raise, and videos
        are given as decoded frame stacks (4-D .npy). It is opt-in because two decoders need not return the same pixels for one file,
        and every parity guarantee of this engine starts from identical decoded pixels: the reference decodes with decord, so a reader
        wrapping decord reproduces its frames, and OpenCV's may differ."""
        assert model_name in QWEN2_VL_MODELS
        self.min_pixels, self.max_pixels = int(min_pixels), int(max_pixels)
        if video_reader == "opencv":
            from .qwen_utils import OpenCVVideoReader
            video_reader = OpenCVVideoReader()
        elif video_reader is not None and not callable(getattr(video_reader, "open", None)):
            raise ValueError("video_reader must be None, 'opencv' or an object with open(path) -> (num_frames, avg_fps, get)")
        self.video_reader = video_reader
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
        if self._state_dict is None:
            self.cfg = _checkpoint_config(self._checkpoint or spec["model"]["path"], self.cfg, self.model_name)
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

    def load_images(self, image: List[str], fps=None):
        """-> (patches fp32 [sum P, 1176] on the device, [(t, gh, gw), ...]): t = 1 for a still image, ceil(n / 2) for a 4-D .npy stack
        of n frames or for n frames sampled from a video file at `fps` (a video)."""
        files = [p for p in image if _is_video_file(p)]
        if files and getattr(self, "video_reader", None) is None:
            raise NotImplementedError("video files need a decoder: construct the model with video_reader='opencv' (or a reader object), "
                                      "or pass the decoded frames as a 4-D .npy [n, h, w, 3]")
        if files:
            rest = [p for p in image if not _is_video_file(p)]
            loaded = dict(zip(files, (self._load_video_file(p, fps) for p in files)))
            if rest:
                patches, grids = self.load_images(rest)
                o = 0
                for p, g in zip(rest, grids):
                    n = g[0] * g[1] * g[2]
                    loaded[p] = (patches[o:o + n], g)
                    o += n
            parts = [loaded[p] for p in image]
            return torch.cat([x for x, _ in parts]), [g for _, g in parts]
        # PIL decode on the host, everything else (smart_resize, PIL-exact bicubic, normalise, frame duplication or pairing, merge-order
        # patch rows) in ONE device kernel -- bit-identical to qwen_utils.qwen_image_to_patches / qwen_video_to_patches, the CPU paths
        # the reference runs per image / per video
        import numpy as np
        from PIL import Image
        from ...engine import qwen_preprocess_video_u8
        raw = []
        for p in image:
            if p.lower().endswith(".npy"):
                # the reference's Qwen path takes the array as RGB, no channel flip (qwen2vl_model.py:146-153); a 4-D array is a frame
                # stack, each frame Image.fromarray(frame.astype('uint8'), 'RGB'), scored as a video
                arr = np.load(p)
                if arr.ndim == 4:
                    arr = np.stack([np.asarray(Image.fromarray(f.astype("uint8"), "RGB"), dtype=np.uint8) for f in arr])
                elif arr.ndim == 3:
                    arr = np.asarray(Image.fromarray(arr.astype("uint8"), "RGB"), dtype=np.uint8)
                else:
                    raise ValueError(f"Unexpected shape for NumPy array in {p}")
            else:
                with Image.open(p) as im:
                    arr = np.asarray(im.convert("RGB"), dtype=np.uint8)
            raw.append(torch.from_numpy(np.ascontiguousarray(arr)))
        return qwen_preprocess_video_u8(raw, self.engine.device, self.cfg.patch_size, self.cfg.temporal_patch_size, self.cfg.spatial_merge_size,
                   min_pixels=self.min_pixels, max_pixels=self.max_pixels)

    def _load_video_file(self, path: str, fps):
        """One video file -> (patches on the device, (t, gh, gw)): the reader's frames at qwen_vl_utils' sampled indices, sent to the
        device in slices of engine.VIDEO_SLICE_BYTES and resized there (engine.qwen_preprocess_video_file_u8)."""
        import numpy as np
        from ...engine import VIDEO_SLICE_BYTES, qwen_preprocess_video_file_u8
        from .qwen_utils import qwen_video_file_plan
        fps = VIDEO_FILE_DEFAULT_FPS if fps is None else fps
        total, avg_fps, get = self.video_reader.open(path)
        first = np.asarray(get([0]))             # every sampling starts at frame 0, and its size is the video's
        idx, _, size = qwen_video_file_plan(total, avg_fps, first.shape[1], first.shape[2], fps=None if fps == "dynamic" else float(fps),
                                            max_pixels=VIDEO_FILE_MAX_PIXELS)
        per = max(1, VIDEO_SLICE_BYTES // first[0].size)
        slices = (torch.from_numpy(np.ascontiguousarray(get(idx[i:i + per]), dtype=np.uint8)) for i in range(0, len(idx), per))
        return qwen_preprocess_video_file_u8(slices, size, self.engine.device, n_frames=len(idx), patch=self.cfg.patch_size,
                                             temporal_patch=self.cfg.temporal_patch_size, merge=self.cfg.spatial_merge_size)

    def _vision(self, images: List[str], fps=None):
        """Identical paths encoded once: -> (item of every pair, patches, grids, per-item prompt token id, per-item second_per_grid_ts
        or None when there is no video). A video file gets the 2/24 of a frame stack: the reference hands its frames to the processor as
        a tensor without metadata, whose sampled_fps is 24 whatever `fps` sampled them (see HF_FRAME_LIST_FPS)."""
        uniq: Dict[str, int] = {}
        index = [uniq.setdefault(p, len(uniq)) for p in images]
        paths = list(uniq.keys())
        files = [_is_video_file(p) for p in paths]
        patches, grids = self.load_images(paths, fps) if any(files) else self.load_images(paths)
        video = [f or _is_frame_stack(p) for p, f in zip(paths, files)]
        tokens = [self.cfg.video_token_id if v else self.cfg.image_token_id for v in video]
        spg = [self.cfg.temporal_patch_size / HF_FRAME_LIST_FPS if v else 1.0 for v in video] if any(video) else None
        return index, patches, grids, tokens, spg

    def _memo(self) -> dict:
        cache = self.__dict__.setdefault("_prompt_cache", {})
        if len(cache) > 65536:
            cache.clear()
        return cache

    def _answer_ids(self, answer: str, cache: dict) -> tuple:
        ids = cache.get(("answer", answer))
        if ids is None:
            ids = cache[("answer", answer)] = tuple(self.tokenizer.encode(answer, add_special_tokens=False))
        if not ids:
            raise ValueError("empty answer")
        return ids

    @torch.no_grad()
    def forward_with_trace(self, images: List[str], texts: List[str], fps=None, question_template: str = default_question_template,
                           answer_template: str = default_answer_template, max_new_tokens: int = 1, temperature: float = 1.0,
                           score_position: str = "end", debug: bool = False, repetition_penalty: Optional[float] = None):
        """Scores plus the per-sample trace dictionaries of the reference's forward_with_trace (qwen2vl_model.py:303-493; schema at
        :469-487): the greedy token, the answer token's probability and the five most probable alternatives. With one generated position
        `score_position` "start" and "end" coincide. The alternatives come from a top-k pass over the last position's logits
        (engine.topk_last) under the same temperature / repetition penalty as the score."""
        assert score_position in ("start", "end"), f"score_position must be 'start' or 'end', got '{score_position}'"
        if max_new_tokens != 1:
            _require_rollout_engine(self)
            return self._trace_rollout(images, texts, question_template, answer_template, max_new_tokens, temperature, score_position, debug,
                                       repetition_penalty, fps)
        assert len(images) == len(texts), "Number of images/videos and texts must match"
        probs, answer_ids, ids, top_p = self._score(images, texts, question_template, answer_template, temperature, repetition_penalty, 5,
                                                    fps)
        dec = lambda t: self.tokenizer.decode([t]) if hasattr(self.tokenizer, "decode") else str(t)
        special = {getattr(self.tokenizer, n, None) for n in ("eos_token_id", "bos_token_id", "pad_token_id")} - {None}
        traces = []
        for b, (p, answer_id) in enumerate(zip(probs.tolist(), answer_ids)):
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

    def _rollout(self, images: List[str], texts: List[str], question_template: str, answer_template: str, max_new_tokens: int,
                 temperature: float, repetition_penalty: float, mode: str, top_k: int, fps=None) -> List[dict]:
        """Scored greedy rollouts of max_new_tokens for every (image, text) pair: the scoring prompt, generate(do_sample=False) under the
        repetition penalty and the EOS ids of generation, and per step the log-probability of every answer token
        (engine.rollout_scores), then the reference's step selection (qwen_host.rollout_answer_score, `mode` "forward", "start" or "end").
        Identical images are encoded once per chunk; a chunk holds at most ROLLOUT_MAX_PAIRS pairs and fewer when its generation workspace
        would exceed ROLLOUT_WORKSPACE_BUDGET. Returns one rollout_answer_score dict per pair, with `tokens`, `answer_ids` and, with
        top_k > 0, the per-step `topk_ids` / `topk_probs` [max_new_tokens, top_k] added."""
        from ... import qwen_host
        if max_new_tokens < 1:
            raise ValueError("max_new_tokens must be at least 1")
        questions = [question_template.format(t) for t in texts]
        answers = [answer_template.format(t) for t in texts]
        index, patches, grids, tokens, spg = self._vision(images, fps)
        unit = self.cfg.spatial_merge_size ** 2
        cache = self._memo()
        prompts, answer_ids = [], []
        for q, a, img in zip(questions, answers, index):
            t, gh, gw = grids[img]
            prompts.append(build_prompt_ids(self.tokenizer, q, t * gh * gw // unit, tokens[img], cache))
            answer_ids.append(list(self._answer_ids(a, cache)))
        eos = self._eos_ids()
        special = {getattr(self.tokenizer, n, None) for n in ("eos_token_id", "bos_token_id", "pad_token_id")} - {None}
        ws = lambda b, s, p: self.engine.generate_workspace_bytes(b, s, p, max_new_tokens)
        results = []
        for sel in _chunks(len(prompts), self.ROLLOUT_MAX_PAIRS, self.ROLLOUT_WORKSPACE_BUDGET, ws, max(len(p) for p in prompts),
                           [t * h * w for t, h, w in grids]):
            pix, items, local = _subset(patches, grids, index, sel)
            video = {} if spg is None else dict(second_per_grid_ts=[spg[g] for g in items])
            out = self.engine.rollout_scores(pix, [grids[g] for g in items], [prompts[i] for i in sel], [answer_ids[i] for i in sel],
                                             max_new_tokens, eos, temperature=temperature, repetition_penalty=repetition_penalty,
                                             top_k=top_k, image_of_sample=local, **video)
            for b, i in enumerate(sel):
                r = qwen_host.rollout_answer_score(out["tokens"][b], out["logp"][b], answer_ids[i], special, mode)
                r.update(tokens=out["tokens"][b], answer_ids=answer_ids[i])
                if top_k > 0:
                    r.update(topk_ids=out["topk_ids"][b], topk_probs=out["topk_probs"][b])
                results.append(r)
        return results

    def _trace_rollout(self, images, texts, question_template, answer_template, max_new_tokens, temperature, score_position, debug,
                       repetition_penalty, fps=None):
        """forward_with_trace for max_new_tokens > 1 (reference qwen2vl_model.py:381-487): scored rollouts, answer tokens placed at the
        start or the end of the generation, and the reference's trace dictionary per sample."""
        pen = self.repetition_penalty if repetition_penalty is None else repetition_penalty
        results = self._rollout(images, texts, question_template, answer_template, max_new_tokens, temperature, pen, score_position, 5, fps)
        one = lambda t: self.tokenizer.decode([int(t)])
        traces = []
        for b, r in enumerate(results):
            toks, start, n = r["tokens"], r["start"], r["n"]
            details = []
            for i, s in enumerate(r["steps"]):
                alts = [dict(token_id=int(t), token_text=one(t), probability=float(p))
                        for t, p in zip(r["topk_ids"][s].tolist(), r["topk_probs"][s].tolist())]
                details.append(dict(position=s, expected_token_id=r["answer_ids"][i], expected_token_text=one(r["answer_ids"][i]),
                                    probability=r["probs"][i], top_alternatives=alts))
            traces.append(dict(generated_text=self.tokenizer.decode(toks, skip_special_tokens=True), generated_length=len(toks),
                               score_position=score_position, score_start_idx=start, scored_indices=list(r["steps"]),
                               scored_tokens_text=self.tokenizer.decode(toks[start:start + n], skip_special_tokens=True),
                               probability=r["score"], token_details=details))
            if debug:
                print(f"sample {b}: generated {traces[-1]['generated_text']!r} ({len(toks)} tokens); scored steps {r['steps']}; "
                      f"probabilities {[round(p, 6) for p in r['probs']]}; geometric mean {r['score']:.6f}")
        return torch.tensor([r["score"] for r in results], dtype=torch.float32), traces

    @torch.no_grad()
    def generate(self, images: List[str], texts: List[str], fps=None, max_new_tokens: int = 2048, temperature: float = 0.0,
                 do_sample: Optional[bool] = None, top_p: float = 0.9, eos_token_ids: Optional[List[int]] = None,
                 generator: Optional[torch.Generator] = None) -> List[str]:
        """Text generation, the reference's Qwen2VLModel.generate (qwen2vl_model.py:495-563): per sample, the chat prompt of the raw
        text and the image, generate() under the checkpoint's repetition penalty, the prompt cut off, decoded with skip_special_tokens and
        stripped. With the default temperature 0 it is greedy (do_sample=False). With do_sample (None: temperature > 0) and temperature > 0
        it samples as generate(do_sample=True, temperature, top_p) does, with generation_config.json's top_k (default 50): see
        sampling_params. Each prompt's draws come from a 63-bit seed taken from `generator` (None: torch's default generator, so
        torch.manual_seed(s) before the call reproduces it). Here the whole batch is one prefill and one decode loop on the device (a call
        with a video: as few as fit VIDEO_WORKSPACE_BUDGET); identical paths are encoded once. `fps` samples the frames of a video file and
        does not change the output for a .npy frame stack (see HF_FRAME_LIST_FPS)."""
        assert len(images) == len(texts), "Number of images/videos and texts must match"
        sampling = None
        if do_sample or temperature > 0:
            # the engine's capability is looked up on its class, so nothing of the instance is touched before the refusal
            if not callable(getattr(type(getattr(self, "engine", None)), "sample_prompts", None)):
                raise NotImplementedError("this engine has only greedy decoding (temperature=0.0, do_sample=False): it has no "
                                          "sample_prompts for top-k / top-p sampling")
            sampling = sampling_params(self._checkpoint or QWEN2_VL_MODELS[self.model_name]["model"]["path"], do_sample, temperature, top_p)
        index, patches, grids, tokens, spg = self._vision(images, fps)
        unit = self.cfg.spatial_merge_size ** 2
        cache = self._memo()
        prompts = []
        for text, img in zip(texts, index):
            t, gh, gw = grids[img]
            prompts.append(build_prompt_ids(self.tokenizer, text, t * gh * gw // unit, tokens[img], cache))
        eos = self._eos_ids() if eos_token_ids is None else [int(e) for e in eos_token_ids]
        ws = lambda b, s, p: self.engine.generate_workspace_bytes(b, s, p, max_new_tokens)
        if sampling is not None:
            seeds = torch.randint(0, 2 ** 63 - 1, (len(prompts),), dtype=torch.int64, generator=generator).tolist()
        ids = []
        for sel in self._prefill_chunks(prompts, grids, spg, ws):
            pix, items, local = _subset(patches, grids, index, sel)
            video = {} if spg is None else dict(second_per_grid_ts=[spg[g] for g in items])
            args = (pix, [grids[g] for g in items], [prompts[i] for i in sel], max_new_tokens, eos)
            if sampling is None:
                ids += self.engine.generate_prompts(*args, image_of_sample=local, repetition_penalty=self.repetition_penalty, **video)
            else:
                t, k, p = sampling
                ids += self.engine.sample_prompts(*args, [seeds[i] for i in sel], t, k, p, image_of_sample=local,
                                                  repetition_penalty=self.repetition_penalty, **video)
        return [self.tokenizer.decode(x, skip_special_tokens=True, clean_up_tokenization_spaces=False).strip() for x in ids]

    def _prefill_chunks(self, prompts, grids, spg, workspace_bytes) -> List[List[int]]:
        """All pairs in one engine call without a video (spg None); with one, chunks under VIDEO_WORKSPACE_BUDGET."""
        if spg is None:
            return [list(range(len(prompts)))]
        return _chunks(len(prompts), len(prompts), self.VIDEO_WORKSPACE_BUDGET, workspace_bytes, max(len(p) for p in prompts),
                       [t * h * w for t, h, w in grids])

    def _score(self, images, texts, question_template, answer_template, temperature, repetition_penalty, top_k, fps=None):
        """Single-prefill scores of the first answer token -> (probs fp32 CPU [n], answer ids, and with top_k > 0 the top-k ids / probs of
        the last position as lists, else None, None)."""
        questions = [question_template.format(t) for t in texts]
        answers = [answer_template.format(t) for t in texts]
        index, patches, grids, tokens, spg = self._vision(images, fps)
        unit = self.cfg.spatial_merge_size ** 2
        prompts, answer_ids = [], []
        cache = self._memo()
        for q, a, img in zip(questions, answers, index):
            t, gh, gw = grids[img]
            prompts.append(build_prompt_ids(self.tokenizer, q, t * gh * gw // unit, tokens[img], cache))
            # one generated position => the reference truncates a multi-token answer to its first token ("Generated 1 tokens but need n,
            # adjusting", qwen2vl_model.py:259-263) and the geometric mean over one token is that token's probability
            answer_ids.append(self._answer_ids(a, cache)[0])
        pen = self.repetition_penalty if repetition_penalty is None else repetition_penalty
        probs, top_ids, top_p = [], [], []
        for sel in self._prefill_chunks(prompts, grids, spg, lambda b, s, p: self.engine.score_workspace_bytes(b, s, p)):
            pix, items, local = _subset(patches, grids, index, sel)
            video = {} if spg is None else dict(second_per_grid_ts=[spg[g] for g in items])
            probs.append(self.engine.score_prompts(pix, [grids[g] for g in items], [prompts[i] for i in sel], [answer_ids[i] for i in sel],
                                                   image_of_sample=local, temperature=temperature, repetition_penalty=pen, **video).float().cpu())
            if top_k:
                ids, p = self.engine.topk_last(top_k, temperature=temperature, repetition_penalty=pen)
                top_ids += ids.cpu().tolist()
                top_p += p.cpu().tolist()
        return torch.cat(probs), answer_ids, (top_ids if top_k else None), (top_p if top_k else None)

    @torch.no_grad()
    def forward(self, images: List[str], texts: List[str], fps=None, question_template: str = default_question_template,
                answer_template: str = default_answer_template, max_new_tokens: int = 1, temperature: float = 1.0,
                debug: bool = False, repetition_penalty: Optional[float] = None) -> torch.Tensor:
        """Scores of (image or video, text) pairs. A 4-D .npy is a video; `fps` is accepted and does not change its score, as in the
        reference on transformers 5.5.0, whose processor takes a frame list's rate to be 24 fps whatever is passed (HF_FRAME_LIST_FPS).
        A video file (with a `video_reader`) is a video whose frames are sampled at `fps` (None: 8.0; "dynamic": qwen_vl_utils' 2.0).
        A call with a video runs as few single-prefill engine calls as fit VIDEO_WORKSPACE_BUDGET; one with still images only, as one."""
        assert len(images) == len(texts), "Number of images/videos and texts must match"
        if max_new_tokens != 1:
            # the reference scores answer token i on the scores of step len(scores) - n + i (- 1 after a trailing special token) of its own
            # greedy continuation (qwen2vl_model.py:239-289): a scored rollout on the decode loop
            _require_rollout_engine(self)
            pen = self.repetition_penalty if repetition_penalty is None else repetition_penalty
            return torch.tensor([r["score"] for r in self._rollout(images, texts, question_template, answer_template, max_new_tokens,
                                                                    temperature, pen, "forward", 0, fps)], dtype=torch.float32)
        return self._score(images, texts, question_template, answer_template, temperature, repetition_penalty, 0, fps)[0]

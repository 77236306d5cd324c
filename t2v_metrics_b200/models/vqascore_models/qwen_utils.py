"""Host-side image / prompt preparation of the Qwen2.5-VL path.

* `smart_resize` + `qwen_image_to_patches`: what `qwen_vl_utils.process_vision_info` (PIL resize to multiples of 28) and
  `Qwen2VLImageProcessor._preprocess` with do_resize=False (transformers/models/qwen2_vl/image_processing_qwen2_vl.py:62-87,
  :191-220) do to one still image: rescale, CLIP-normalise, duplicate the frame along the temporal axis, cut 14x14 patches and
  emit them in 2x2 merge-block order as rows of 3*2*14*14 = 1176 values.
* `qwen_video_to_patches`: the same for one decoded frame stack, as the reference's decoder-free video path hands it to
  `Qwen2VLVideoProcessor` (consecutive frames fill the temporal slots of a patch row).
* `build_prompt_ids`: the chat template the reference applies (qwen2vl_model.py:197-200) with the image pad expanded to one
  token per merged patch group (processing_qwen2_5_vl.py:119-137).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from PIL import Image

OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)

default_question_template = 'Does this figure show "{}"? Please answer Yes or No.'   # qwen2vl_model.py:173
default_answer_template = "Yes"                                                        # qwen2vl_model.py:174

CHAT_PREFIX = "<|im_start|>system\nYou are a helpful assistant.<|im_end|>\n<|im_start|>user\n<|vision_start|>"
CHAT_SUFFIX = "<|vision_end|>{question}<|im_end|>\n<|im_start|>assistant\n"


def smart_resize(height: int, width: int, factor: int = 28, min_pixels: int = 56 * 56, max_pixels: int = 14 * 14 * 4 * 1280) -> Tuple[int, int]:
    """Both sides divisible by `factor`, pixel count within [min_pixels, max_pixels], aspect ratio kept as closely as possible."""
    if max(height, width) / min(height, width) > 200:
        raise ValueError("absolute aspect ratio must be smaller than 200")
    h_bar = round(height / factor) * factor
    w_bar = round(width / factor) * factor
    if h_bar * w_bar > max_pixels:
        beta = math.sqrt((height * width) / max_pixels)
        h_bar = max(factor, math.floor(height / beta / factor) * factor)
        w_bar = max(factor, math.floor(width / beta / factor) * factor)
    elif h_bar * w_bar < min_pixels:
        beta = math.sqrt(min_pixels / (height * width))
        h_bar = math.ceil(height * beta / factor) * factor
        w_bar = math.ceil(width * beta / factor) * factor
    return h_bar, w_bar


def qwen_image_to_patches(img: Image.Image, patch_size: int = 14, temporal_patch_size: int = 2, merge_size: int = 2,
                          min_pixels: int = 56 * 56, max_pixels: int = 14 * 14 * 4 * 1280):
    """One RGB image -> (patches fp32 [gh*gw, 3*temporal*ps*ps], (1, gh, gw))."""
    img = img.convert("RGB")
    w, h = img.size
    rh, rw = smart_resize(h, w, patch_size * merge_size, min_pixels, max_pixels)
    if (rw, rh) != (w, h):
        img = img.resize((rw, rh), resample=Image.BICUBIC)
    x = torch.from_numpy(np.asarray(img, dtype=np.float32)).permute(2, 0, 1) / 255.0
    x = (x - torch.tensor(OPENAI_CLIP_MEAN)[:, None, None]) / torch.tensor(OPENAI_CLIP_STD)[:, None, None]
    x = x[None].repeat(temporal_patch_size, 1, 1, 1)                      # still image: the frame is duplicated
    gh, gw = rh // patch_size, rw // patch_size
    x = x.view(1, temporal_patch_size, 3, gh // merge_size, merge_size, patch_size, gw // merge_size, merge_size, patch_size)
    x = x.permute(0, 3, 6, 4, 7, 2, 1, 5, 8)                             # (t, h/m, w/m, m, m, c, tp, ps, ps)
    return x.reshape(gh * gw, 3 * temporal_patch_size * patch_size * patch_size).contiguous(), (1, gh, gw)


def qwen_video_to_patches(frames, patch_size: int = 14, temporal_patch_size: int = 2, merge_size: int = 2, min_pixels: int = 56 * 56,
                          max_pixels: int = 14 * 14 * 4 * 1280):
    """One decoded frame stack (uint8 [n, h, w, 3] RGB, or a list of PIL images of one size) -> (patches fp32 [t*gh*gw, 1176], (t, gh, gw)),
    what the reference's decoder-free video path computes: qwen_vl_utils 0.0.8 `fetch_video` on a list of frames runs `fetch_image`
    (smart_resize(factor 28, min_pixels, max_pixels) + PIL BICUBIC resize) on each and pads the count to a multiple of FRAME_FACTOR = 2 with
    the last frame; `Qwen2VLVideoProcessor._preprocess` with do_resize=False (transformers 5.5.0, video_processing_qwen2_vl.py:228-275)
    then rescales and normalises, pads to a multiple of temporal_patch_size with the last frame, and emits frames k*tp .. k*tp + tp - 1 as
    the temporal slots of group k's patch rows, in the merge-block order of still images."""
    imgs = [f.convert("RGB") if isinstance(f, Image.Image) else Image.fromarray(np.asarray(f, dtype=np.uint8), "RGB") for f in frames]
    w, h = imgs[0].size
    rh, rw = smart_resize(h, w, patch_size * merge_size, min_pixels, max_pixels)
    x = torch.stack([torch.from_numpy(np.asarray(im if (rw, rh) == (w, h) else im.resize((rw, rh), resample=Image.BICUBIC), dtype=np.float32))
                     for im in imgs]).permute(0, 3, 1, 2) / 255.0
    x = (x - torch.tensor(OPENAI_CLIP_MEAN)[:, None, None]) / torch.tensor(OPENAI_CLIP_STD)[:, None, None]
    if pad := -x.shape[0] % temporal_patch_size:
        x = torch.cat([x, x[-1:].expand(pad, -1, -1, -1)])
    gt, gh, gw = x.shape[0] // temporal_patch_size, rh // patch_size, rw // patch_size
    x = x.reshape(gt, temporal_patch_size, 3, gh // merge_size, merge_size, patch_size, gw // merge_size, merge_size, patch_size)
    x = x.permute(0, 3, 6, 4, 7, 2, 1, 5, 8)
    return x.reshape(gt * gh * gw, 3 * temporal_patch_size * patch_size * patch_size).contiguous(), (gt, gh, gw)


def build_prompt_ids(tokenizer, question: str, n_image_tokens: int, image_token_id: int, cache: Optional[dict] = None) -> List[int]:
    """`cache` (SURVEY 8(f)3): exact memo string -> ids; the chat prefix is constant and M x N scoring repeats each question M times."""
    def enc(s: str):
        if cache is None:
            return list(tokenizer.encode(s, add_special_tokens=False))
        ids = cache.get(s)
        if ids is None:
            ids = cache[s] = tuple(tokenizer.encode(s, add_special_tokens=False))
        return list(ids)
    return enc(CHAT_PREFIX) + [image_token_id] * n_image_tokens + enc(CHAT_SUFFIX.format(question=question))

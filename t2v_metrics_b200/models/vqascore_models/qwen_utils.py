"""Host-side image / prompt preparation of the Qwen2.5-VL path.

* `smart_resize` + `qwen_image_to_patches`: what `qwen_vl_utils.process_vision_info` (PIL resize to multiples of 28) and
  `Qwen2VLImageProcessor._preprocess` with do_resize=False (transformers/models/qwen2_vl/image_processing_qwen2_vl.py:62-87,
  :191-220) do to one still image: rescale, CLIP-normalise, duplicate the frame along the temporal axis, cut 14x14 patches and
  emit them in 2x2 merge-block order as rows of 3*2*14*14 = 1176 values.
* `qwen_video_to_patches`: the same for one decoded frame stack, as the reference's decoder-free video path hands it to
  `Qwen2VLVideoProcessor` (consecutive frames fill the temporal slots of a patch row).
* `qwen_video_file_plan`, `qwen_video_file_to_patches`, `OpenCVVideoReader`: the same for a video FILE, which qwen_vl_utils samples at
  `fps` and resizes as one tensor with torchvision's antialiased bicubic (a different filter from PIL's).
* `build_prompt_ids`: the chat template the reference applies (qwen2vl_model.py:197-200) with the image pad expanded to one
  token per merged patch group (processing_qwen2_5_vl.py:119-137).
"""
from __future__ import annotations

import math
import os
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
                     for im in imgs]).permute(0, 3, 1, 2)
    return _video_patch_rows(x, patch_size, temporal_patch_size, merge_size)


def _video_patch_rows(x: torch.Tensor, patch_size: int, temporal_patch_size: int, merge_size: int):
    """Resized frames as fp32 uint8 levels [n, 3, rh, rw] -> (patches fp32 [t*gh*gw, 1176], (t, gh, gw)): `Qwen2VLVideoProcessor._preprocess`
    with do_resize=False (transformers 5.5.0, video_processing_qwen2_vl.py:228-275) -- rescale and normalise, pad to a multiple of
    temporal_patch_size with the last frame, frames k*tp .. k*tp + tp - 1 as the temporal slots of group k's patch rows, merge-block order."""
    x = (x / 255.0 - torch.tensor(OPENAI_CLIP_MEAN)[:, None, None]) / torch.tensor(OPENAI_CLIP_STD)[:, None, None]
    if pad := -x.shape[0] % temporal_patch_size:
        x = torch.cat([x, x[-1:].expand(pad, -1, -1, -1)])
    gt, gh, gw = x.shape[0] // temporal_patch_size, x.shape[2] // patch_size, x.shape[3] // patch_size
    x = x.reshape(gt, temporal_patch_size, 3, gh // merge_size, merge_size, patch_size, gw // merge_size, merge_size, patch_size)
    x = x.permute(0, 3, 6, 4, 7, 2, 1, 5, 8)
    return x.reshape(gt * gh * gw, 3 * temporal_patch_size * patch_size * patch_size).contiguous(), (gt, gh, gw)


# qwen_vl_utils 0.0.8 (vision_process.py, the version qwen_video_to_patches restates), what `fetch_video` does with a video FILE: these
# constants, `smart_nframes`, frame indices torch.linspace(0, total - 1, nframes).round(), and the pixel budget of the resize.
# VIDEO_TOTAL_PIXELS is read from the environment variable VIDEO_MAX_PIXELS at import, as qwen_vl_utils reads it.
VIDEO_MIN_PIXELS = 128 * 28 * 28
VIDEO_MAX_PIXELS = 768 * 28 * 28
VIDEO_TOTAL_PIXELS = int(float(os.environ.get("VIDEO_MAX_PIXELS", 128000 * 28 * 28 * 0.9)))
FRAME_FACTOR = 2
FPS = 2.0
FPS_MIN_FRAMES = 4
FPS_MAX_FRAMES = 768


def qwen_video_file_plan(total_frames: int, video_fps: float, height: int, width: int, fps: Optional[float] = None,
                         max_pixels: Optional[float] = None, min_pixels: int = VIDEO_MIN_PIXELS, total_pixels: int = VIDEO_TOTAL_PIXELS,
                         factor: int = 28) -> Tuple[List[int], float, Tuple[int, int]]:
    """qwen_vl_utils 0.0.8 fetch_video's sampling and size for a file of `total_frames` frames at `video_fps` -> (frame indices,
    sample_fps, (rh, rw)). `fps` / `max_pixels` are the video element's keys (None: absent, so FPS = 2.0 / no per-element cap).
    smart_nframes: nframes = floor_by_factor(min(min(max(total / video_fps * fps, ceil_by_factor(FPS_MIN_FRAMES, 2)),
    floor_by_factor(min(FPS_MAX_FRAMES, total), 2)), total), 2), refused unless 2 <= nframes <= total. Pixel bounds: min_pixels, and
    min(max_pixels, max(min(VIDEO_MAX_PIXELS, total_pixels / nframes * 2), int(min_pixels * 1.05))). smart_resize is the one still images
    use; it agrees with qwen_vl_utils' own wherever both sides of the result are at least `factor`."""
    fps = FPS if fps is None else float(fps)
    min_frames = math.ceil(FPS_MIN_FRAMES / FRAME_FACTOR) * FRAME_FACTOR
    max_frames = math.floor(min(FPS_MAX_FRAMES, total_frames) / FRAME_FACTOR) * FRAME_FACTOR
    nframes = total_frames / video_fps * fps
    nframes = math.floor(min(min(max(nframes, min_frames), max_frames), total_frames) / FRAME_FACTOR) * FRAME_FACTOR
    if not FRAME_FACTOR <= nframes <= total_frames:
        raise ValueError(f"nframes should in interval [{FRAME_FACTOR}, {total_frames}], but got {nframes}.")
    indices = torch.linspace(0, total_frames - 1, nframes).round().long().tolist()
    sample_fps = nframes / max(total_frames, 1e-6) * video_fps
    bound = max(min(VIDEO_MAX_PIXELS, total_pixels / nframes * FRAME_FACTOR), int(min_pixels * 1.05))
    if max_pixels is not None:
        bound = min(max_pixels, bound)
    return indices, sample_fps, smart_resize(height, width, factor, min_pixels, bound)


def qwen_video_file_to_patches(frames_u8, size: Tuple[int, int], patch_size: int = 14, temporal_patch_size: int = 2, merge_size: int = 2):
    """Frames sampled from a video file (uint8 [n, h, w, 3] RGB) -> (resized uint8 frames [n, rh, rw, 3], patches fp32 [t*gh*gw, 1176],
    (t, gh, gw)): fetch_video's torchvision resize(BICUBIC, antialias=True) of the whole stack to `size` = (rh, rw) (uint8 -> fp32 ->
    _upsample_bicubic2d_aa -> clamp -> round half to even -> uint8; then `.float()`), and Qwen2VLVideoProcessor with do_resize=False.
    The resize runs on this host's CPU, whose SIMD path may move a value at a rounding tie by one level."""
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms import functional as TF
    x = torch.as_tensor(np.asarray(frames_u8, dtype=np.uint8)).permute(0, 3, 1, 2)
    x = TF.resize(x, list(size), interpolation=InterpolationMode.BICUBIC, antialias=True)
    rows, grid = _video_patch_rows(x.float(), patch_size, temporal_patch_size, merge_size)
    return x.permute(0, 2, 3, 1).contiguous(), rows, grid


class OpenCVVideoReader:
    """`video_reader="opencv"`: frames decoded by OpenCV's FFMPEG backend. open(path) -> (frames, average fps, get), where the frame
    count comes from decoding the whole stream (container headers can be wrong) and get(indices) decodes forward to the (non-decreasing)
    indices and returns them as uint8 [k, h, w, 3] RGB; successive calls continue where the last one stopped."""

    def open(self, path: str):
        try:
            import cv2
        except ImportError as e:
            raise ImportError("video_reader='opencv' needs OpenCV (cv2); without it, decode the frames yourself and pass them as a 4-D "
                              ".npy [n, h, w, 3]") from e
        cap = cv2.VideoCapture(path)
        if not cap.isOpened():
            raise ValueError(f"OpenCV cannot open the video {path}")
        avg_fps, total = float(cap.get(cv2.CAP_PROP_FPS)), 0
        while cap.grab():
            total += 1
        cap.release()
        if total == 0 or not avg_fps > 0:
            raise ValueError(f"OpenCV decodes no frames or no frame rate from {path}")
        state = dict(cap=None, pos=0, last=None)      # pos: frames decoded so far; last: frame pos - 1, RGB

        def get(indices):
            if state["cap"] is None or (len(indices) and indices[0] < state["pos"] - 1):
                state.update(cap=cv2.VideoCapture(path), pos=0, last=None)
            cap, out = state["cap"], []
            for i in indices:
                if i >= state["pos"]:
                    while state["pos"] < i:
                        if not cap.grab():
                            raise ValueError(f"{path}: frame {i} is past the end of the stream")
                        state["pos"] += 1
                    ok, bgr = cap.read()
                    if not ok:
                        raise ValueError(f"{path}: frame {i} is past the end of the stream")
                    state["pos"] += 1
                    state["last"] = cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)
                elif i != state["pos"] - 1:
                    raise ValueError("frame indices must not decrease")
                out.append(state["last"])
            return np.stack(out)

        return total, avg_fps, get


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

"""Host-side pieces of the CLIP-FlanT5 path that survive in the reference's mm_utils.py, rebuilt for this engine."""
import io
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch
from PIL import Image

from ...constants import IMAGE_TOKEN_INDEX, DEFAULT_IMAGE_TOKEN

CLIP_IMAGE_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_IMAGE_STD = (0.26862954, 0.26130258, 0.27577711)


def expand2square(pil_img: Image.Image, background_color) -> Image.Image:
    """Centre the image on a square canvas of `background_color` (reference mm_utils.py:128-139)."""
    w, h = pil_img.size
    if w == h:
        return pil_img
    side = max(w, h)
    canvas = Image.new(pil_img.mode, (side, side), background_color)
    canvas.paste(pil_img, ((side - w) // 2, (side - h) // 2))
    return canvas


def t5_tokenizer_image_token(prompt: str, tokenizer, image_token_index: int = IMAGE_TOKEN_INDEX, return_tensors=None,
                             chunk_cache: Optional[dict] = None):
    """Tokenise every text chunk around '<image>' separately (each keeps its own trailing </s>) and join the chunks
    with `image_token_index` (reference mm_utils.py:164-179).
    `chunk_cache` (SURVEY 8(f)3): an exact memo chunk-string -> ids. The chunk before '<image>' is the constant system prompt and
    M x N scoring repeats every caption M times, so the slow SentencePiece tokenizer (`use_fast=False`, mm_utils.py:198) runs once
    per distinct chunk; whole chunks are the cache unit because sub-word tokenisation is not prefix-stable."""
    input_ids: List[int] = []
    for i, chunk in enumerate(prompt.split(DEFAULT_IMAGE_TOKEN)):
        if i > 0:
            input_ids.append(image_token_index)
        if chunk_cache is None:
            input_ids.extend(tokenizer(chunk).input_ids)
        else:
            ids = chunk_cache.get(chunk)
            if ids is None:
                ids = chunk_cache[chunk] = tuple(tokenizer(chunk).input_ids)
            input_ids.extend(ids)
    if return_tensors is not None:
        if return_tensors == 'pt':
            return torch.tensor(input_ids, dtype=torch.long)
        raise ValueError(f'Unsupported tensor type: {return_tensors}')
    return input_ids


def clip_preprocess(pil_img: Image.Image, image_size: int, pad: bool = True) -> torch.Tensor:
    """'pad' aspect mode of the v3.0 wrapper + CLIPImageProcessor (transformers image_processing_clip.py:23-34):
    expand2square(mean colour) -> bicubic resize (shortest edge) -> centre crop -> /255 -> normalise. fp32 [3,S,S]."""
    img = pil_img.convert("RGB")
    if pad:
        img = expand2square(img, tuple(int(x * 255) for x in CLIP_IMAGE_MEAN))
    w, h = img.size
    if w <= h:
        nw, nh = image_size, int(h * image_size / w)
    else:
        nw, nh = int(w * image_size / h), image_size
    if (nw, nh) != (w, h):
        img = img.resize((nw, nh), resample=Image.BICUBIC)
    w, h = img.size
    left, top = (w - image_size) // 2, (h - image_size) // 2
    img = img.crop((left, top, left + image_size, top + image_size))
    arr = np.asarray(img, dtype=np.float32) / 255.0
    arr = (arr - np.asarray(CLIP_IMAGE_MEAN, dtype=np.float32)) / np.asarray(CLIP_IMAGE_STD, dtype=np.float32)
    return torch.from_numpy(arr).permute(2, 0, 1).contiguous()


# ------------------------------------------------------------------------------------------------ videos for single-image models
CONCAT_GAP = 10                 # black columns between two frames of the canvas (the reference's dist_images)
JPEG_MAX_SIDE = 65500           # libjpeg's largest dimension: a wider canvas cannot be stored as the JPEG the reference reads back


def _jpeg_round_trip(bgr: np.ndarray):
    import cv2
    ok, buf = cv2.imencode(".jpg", bgr)
    if not ok:
        raise ValueError(f"cannot encode a {bgr.shape[1]}x{bgr.shape[0]} image as JPEG")
    return buf


def video_frames_bgr(path: str, num_frames: int) -> List[np.ndarray]:
    """`num_frames` frames of a video file as the reference's extract_frames + cv2.imread leave them (BGR uint8 [h, w, 3]), in temporal
    order: the container's frame count, step = count // num_frames, a seek to frame i * step before each read (every read seeks to frame
    0 when the clip has fewer frames than num_frames), a failed read skipped, and each frame through one JPEG encode / decode at OpenCV's
    default quality -- in memory instead of through frame files."""
    import cv2
    if num_frames < 1:
        raise ValueError(f"num_frames must be >= 1, got {num_frames}")
    cap = cv2.VideoCapture(path)
    try:
        step = int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) // num_frames
        frames = []
        for i in range(num_frames):
            cap.set(cv2.CAP_PROP_POS_FRAMES, i * step)
            ok, frame = cap.read()
            if ok:
                frames.append(cv2.imdecode(_jpeg_round_trip(frame), cv2.IMREAD_COLOR))
    finally:
        cap.release()
    if not frames:
        raise ValueError(f"no frame could be read from {path!r}")
    return frames


def concat_frames_rgb(frames_bgr: Sequence[np.ndarray], gap: int = CONCAT_GAP) -> np.ndarray:
    """Frames side by side, top-aligned, `gap` black columns apart, on a canvas as tall as the tallest frame (the reference's
    concatenate_images_horizontal), then through the JPEG the reference writes and PIL's decode of it -> RGB uint8 [h, W, 3]."""
    width = sum(f.shape[1] for f in frames_bgr) + gap * (len(frames_bgr) - 1)
    height = max(f.shape[0] for f in frames_bgr)
    if width > JPEG_MAX_SIDE or height > JPEG_MAX_SIDE:
        raise ValueError(f"the concatenated canvas is {width}x{height} px; JPEG allows at most {JPEG_MAX_SIDE} px a side")
    canvas = np.zeros((height, width, 3), dtype=np.uint8)
    x = 0
    for f in frames_bgr:
        canvas[:f.shape[0], x:x + f.shape[1]] = f
        x += f.shape[1] + gap
    buf = _jpeg_round_trip(canvas)
    return np.array(Image.open(io.BytesIO(buf.tobytes())).convert("RGB"), dtype=np.uint8)


def video_canvas(path: str, num_frames: int = 8) -> np.ndarray:
    """What a single-image model of the reference scores for a video file: `num_frames` frames concatenated into one image, RGB uint8
    [h, W, 3] (reference score.py:78-98 with mm_utils.extract_frames and concatenate_images_horizontal), bit for bit, with the frames in
    temporal order."""
    return concat_frames_rgb(video_frames_bgr(path, num_frames))

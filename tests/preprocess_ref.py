"""Shared by the pre-processing tests: image content that changes at every row and column, CPU references of the device resize (Pillow's
integer resampling, then the fp32 normalisation), a restatement of the planner's shared-memory arithmetic, and the production geometries
the GPU tests run with the automatic tile plan."""
import ctypes as C

import numpy as np
import torch
from PIL import Image

from t2v_metrics_b200 import _lib
from t2v_metrics_b200.models.vqascore_models.mm_utils import CLIP_IMAGE_MEAN, CLIP_IMAGE_STD
from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import QWEN_VL_UTILS_MAX_PIXELS, QWEN_VL_UTILS_MIN_PIXELS
from t2v_metrics_b200.models.vqascore_models.qwen_utils import OPENAI_CLIP_MEAN, OPENAI_CLIP_STD, smart_resize

PRE_MAX_SMEM = 200 * 1024          # preprocess.cuh: shared-memory budget of image_preprocess_kernel
PLUGIN_PIXELS = (QWEN_VL_UTILS_MIN_PIXELS, QWEN_VL_UTILS_MAX_PIXELS)     # Qwen2VLModel's default smart_resize bounds
PATCH, TEMPORAL, MERGE = 14, 2, 2

# Production geometries, run on the device with the automatic plan (tests/test_gpu_preprocess_tiles.py); tests/test_preprocess_host.py
# checks that they reach column tiles, chunk 1 and small row tiles in each layout.
# Qwen: (h, w, frames, (min_pixels, max_pixels)); frames 0 = a still image, else a frame stack of that many frames.
QWEN_PRODUCTION = [(2160, 3840, 0, PLUGIN_PIXELS), (3024, 4032, 0, PLUGIN_PIXELS), (6000, 4000, 0, PLUGIN_PIXELS),
                   (4000, 6000, 0, PLUGIN_PIXELS), (3000, 9000, 0, PLUGIN_PIXELS), (720, 1280, 0, PLUGIN_PIXELS),
                   (1080, 1920, 0, PLUGIN_PIXELS), (1999, 2997, 0, PLUGIN_PIXELS), (1, 150, 0, PLUGIN_PIXELS), (150, 1, 0, PLUGIN_PIXELS),
                   (1000, 8000, 0, (QWEN_VL_UTILS_MIN_PIXELS, 1003520)), (2160, 3840, 3, PLUGIN_PIXELS)]
# CLIP: (h, w, out_size, pad_to_square)
CLIP_PRODUCTION = [(h, w, s, pad) for s in (336, 224) for h, w, pad in
                   ((1, 900, False), (2000, 3, False), (1, 900, True), (2000, 3, True), (360, 5190, True), (720, 10310, True))]


def canvas(w, h, seed):
    """Frames-like content: a smooth gradient with noise and saturated blocks (exercises the clip8 over/undershoot). A tall image is
    built from 97 distinct rows so that pil_reference stays cheap for it."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:(97 if h > w else h), 0:w]
    a = np.stack([(x * 7 + y) % 256, (y * 3 + x // 5) % 256, ((x // 37 + y // 23) % 2) * 255], -1).astype(np.int32)
    a = np.clip(a + rng.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)
    return a[(np.arange(h) * 31) % 97] if h > w else a


def photo(h, w, seed):
    """The content of canvas() with every row distinct, built channel by channel so that a 24-megapixel image stays cheap."""
    rng = np.random.default_rng(seed)
    y, x = np.arange(h, dtype=np.int32)[:, None], np.arange(w, dtype=np.int32)[None, :]
    a = np.empty((h, w, 3), np.uint8)
    for c, base in enumerate(((x * 7 + y) % 256, (y * 3 + x // 5) % 256, ((x // 37 + y // 23) % 2) * 255)):
        a[..., c] = np.clip(base + rng.integers(-20, 21, (h, w), dtype=np.int16), 0, 255)
    return a


def pil_reference(a, size=336):
    """mm_utils.clip_preprocess (pad on) without materialising the padded square: Pillow resizes the canvas horizontally into a uint8
    image and then vertically (Resample.c), and skips an axis whose size does not change, so resizing each distinct canvas row on its
    own (width only) and then the stacked rows (height only) runs Pillow's own two passes on the same pixels."""
    h, w = a.shape[:2]
    side = max(h, w)
    bg = tuple(int(v * 255) for v in CLIP_IMAGE_MEAN)
    py, px = (side - h) // 2, (side - w) // 2
    uniq, inv = np.unique(a.reshape(h, -1), axis=0, return_inverse=True)
    rows = np.empty((len(uniq) + 1, side, 3), np.uint8)
    rows[:] = bg
    rows[:-1, px:px + w] = uniq.reshape(-1, w, 3)
    hz = np.asarray(Image.fromarray(rows).resize((size, len(rows)), Image.BICUBIC))
    inter = np.repeat(hz[-1:], side, 0)
    inter[py:py + h] = hz[inv.reshape(-1)]
    out = np.asarray(Image.fromarray(inter).resize((size, size), Image.BICUBIC), dtype=np.float32) / 255.0
    out = (out - np.asarray(CLIP_IMAGE_MEAN, dtype=np.float32)) / np.asarray(CLIP_IMAGE_STD, dtype=np.float32)
    return torch.from_numpy(out).permute(2, 0, 1).contiguous()


def qwen_lut():
    """[3, 256] fp32: every uint8 level through the Qwen plugin's normalisation, (u8 / 255 - mean) / std, with the same torch ops."""
    x = torch.arange(256, dtype=torch.float32)[None, :] / 255.0
    return (x - torch.tensor(OPENAI_CLIP_MEAN)[:, None]) / torch.tensor(OPENAI_CLIP_STD)[:, None]


def qwen_reference(item, min_pixels, max_pixels, device="cpu"):
    """The Qwen patch rows of one still image (uint8 [h, w, 3]) or frame stack ([n, h, w, 3]): Pillow's uint8 bicubic resize of every frame
    to its smart_resize size, the normalisation through qwen_lut(), and the patch-row layout of qwen_utils (a still fills every temporal
    slot; a stack is padded to a multiple of the temporal patch with its last frame) by reshape and permute on `device`.
    -> (fp32 [t * gh * gw, 3 * TEMPORAL * PATCH^2], (t, gh, gw))."""
    frames = item[None] if item.ndim == 3 else item
    h, w = frames.shape[1:3]
    rh, rw = smart_resize(h, w, PATCH * MERGE, min_pixels, max_pixels)
    u8 = np.stack([f if (rh, rw) == (h, w) else np.asarray(Image.fromarray(f).resize((rw, rh), Image.BICUBIC)) for f in frames])
    u8 = torch.from_numpy(u8).to(device).long()
    lut = qwen_lut().to(device)
    x = torch.stack([lut[c][u8[..., c]] for c in range(3)], 1)                   # [n, 3, rh, rw]
    x = x.repeat(TEMPORAL, 1, 1, 1) if item.ndim == 3 else torch.cat([x, x[-1:].expand(-len(x) % TEMPORAL, -1, -1, -1)])
    gt, gh, gw = len(x) // TEMPORAL, rh // PATCH, rw // PATCH
    x = x.reshape(gt, TEMPORAL, 3, gh // MERGE, MERGE, PATCH, gw // MERGE, MERGE, PATCH).permute(0, 3, 6, 4, 7, 2, 1, 5, 8)
    return x.reshape(gt * gh * gw, 3 * TEMPORAL * PATCH * PATCH), (gt, gh, gw)


# ---------------------------------------------------------------------------------------------- the planner's arithmetic, restated
def axis_words(in_size, out_size, first, count):
    """One resize axis as image_preprocess_kernel reads it: per output, the group of 4 source pixels that holds its first tap, and the
    most 4-pixel tap words any output needs (preprocess.cuh pre_pack_table), from the library's Pillow tap table."""
    b = (C.c_int32 * (2 * count))()
    assert _lib.load().vqa_resample_table(in_size, out_size, first, count, b, None) > 0
    b = np.frombuffer(b, dtype=np.int32).reshape(count, 2).astype(np.int64)
    x0, n = b[:, 0], b[:, 1]
    start4 = x0 // 4
    last4 = np.where(n > 0, (x0 + n - 1) // 4, start4)
    return start4, int(max(1, (last4 - start4 + 1).max()))


def clip_axes(h, w, size, pad):
    """(horizontal, vertical) axis_words of a CLIP image: shortest edge -> size with int() truncation, centre crop, on the padded square."""
    ch, cw = (max(h, w),) * 2 if pad else (h, w)
    nw = size if cw <= ch else int(size * cw / ch)
    nh = int(size * ch / cw) if cw <= ch else size
    return axis_words(cw, nw, (nw - size) // 2, size), axis_words(ch, nh, (nh - size) // 2, size)


def qwen_axes(h, w, min_pixels, max_pixels):
    rh, rw = smart_resize(h, w, PATCH * MERGE, min_pixels, max_pixels)
    return axis_words(w, rw, 0, rw), axis_words(h, rh, 0, rh)


def plan_needs(axes, tile_rows, tile_cols, chunk_groups):
    """(shared-memory bytes, band groups) a tile plan needs: the band holds the 4-row groups of the tallest row tile's windows for
    min(tile_cols, out_w) columns, the stage chunk_groups * 4 canvas rows of the widest column tile's 4-column groups."""
    (hs, hnp), (vs, vnp) = axes
    oh, ow = len(vs), len(hs)
    tw = min(tile_cols, ow)
    y0 = np.arange(0, oh, tile_rows)
    band = int((vs[np.minimum(y0 + tile_rows, oh) - 1] + vnp - vs[y0]).max())
    x0 = np.arange(0, ow, tw)
    span = int((hs[np.minimum(x0 + tw, ow) - 1] + hnp - hs[x0]).max())
    return 768 * 4 + 4 * (3 * band * tw + 3 * chunk_groups * 4 * span), band


def geometry(layout, sizes, out_size=336, pad=True, pixels=PLUGIN_PIXELS, frames=None):
    """vqa_debug_preprocess_geometry: [(tile_rows, tile_cols, col_tiles, chunk_groups, band_groups)] per item (layout 0 CLIP, 1 Qwen);
    raises RuntimeError with the library's message when the planner refuses."""
    lib, i32 = _lib.load(), C.c_int32
    n = len(sizes)
    arr = lambda v: (i32 * n)(*v)
    nf = arr([max(f, 1) for f in frames]) if frames else None
    vid = arr([int(f > 0) for f in frames]) if frames else None
    g = (i32 * (5 * n))()
    rc = lib.vqa_debug_preprocess_geometry(layout, nf, arr([s[0] for s in sizes]), arr([s[1] for s in sizes]), vid, n, out_size, int(pad),
                                           PATCH, TEMPORAL, MERGE, pixels[0], pixels[1], g)
    if rc != 0:
        raise RuntimeError(_lib.last_error(None))
    return [tuple(g[5 * i:5 * i + 5]) for i in range(n)]

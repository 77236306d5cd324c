"""image_preprocess_kernel (csrc/preprocess.cuh) bit-exact against Pillow under every tile plan, and at the geometries the plugins run.

The planner picks, per image, the output rows per CTA (32 ... 1), the canvas rows staged per pass (8 or 4) and one or several column
tiles; each choice moves which canvas rows and columns a CTA stages and where its buffers sit in shared memory. The plan sweep forces
every (rows, chunk) pair with several column-tile widths through vqa_debug_set_preprocess_tiles on images small enough for all of
them to fit, and the
production tests run the automatic plans of ordinary photos at the Qwen plugin's pixel bounds and of CLIP's extreme and wide canvases.
The pipeline is integer up to the normalisation table, so every comparison is torch.equal; every output sits between sentinel-filled
guard bands that must come back untouched."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import clipt5_oracle as orc
from preprocess_ref import (CLIP_PRODUCTION, MERGE, PATCH, PLUGIN_PIXELS, PRE_MAX_SMEM, QWEN_PRODUCTION, TEMPORAL, clip_axes, geometry,
                            photo, pil_reference, plan_needs, qwen_axes, qwen_reference)
from t2v_metrics_b200 import _lib
from t2v_metrics_b200.engine import CLIP_MEAN, CLIP_STD, clip_preprocess_u8

pytestmark = pytest.mark.gpu

GUARD = 4096
SENTINEL = -1232.0                  # exact in fp32 and bf16, and no normalised pixel value
TILE_ROWS, CHUNKS = (32, 16, 8, 4, 2, 1), (2, 1)
WHOLE = 1 << 16                     # a tile_cols no output is as wide as: one column tile


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda", 0)


@pytest.fixture
def force_tiles():
    lib = _lib.load()

    def force(tile_rows, tile_cols, chunk_groups):
        assert lib.vqa_debug_set_preprocess_tiles(tile_rows, tile_cols, chunk_groups) == 0
    yield force
    assert lib.vqa_debug_set_preprocess_tiles(0, 0, 0) == 0


def guarded(n, dtype, dev):
    """n output elements between two sentinel-filled guard bands -> (whole buffer, output view)."""
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=dtype, device=dev)
    return buf, buf[GUARD:GUARD + n]


def assert_guards(buf):
    torch.cuda.synchronize()
    assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all()), "write outside the output"


def run_clip(images, size, pad, dtype, dev):
    """vqa_clip_preprocess on host uint8 images, packed back to back (engine.clip_preprocess_u8) -> [n, 3, size, size]."""
    n = len(images)
    buf, out = guarded(n * 3 * size * size, dtype, dev)
    out = out.view(n, 3, size, size)
    clip_preprocess_u8([torch.from_numpy(a) for a in images], size, dev, pad=pad, out=out)
    assert_guards(buf)
    return out


def run_qwen(items, dtype, dev, pixels):
    """Still images (uint8 [h, w, 3]) and frame stacks ([n, h, w, 3]) through vqa_qwen_preprocess_video, packed back to back on the
    device -> (patch rows, [(t, gh, gw)])."""
    lib, i32, i64 = _lib.load(), C.c_int32, C.c_int64
    n = len(items)
    arr = lambda t, v: (t * len(v))(*v)
    nf = [it.shape[0] if it.ndim == 4 else 1 for it in items]
    vid = [int(it.ndim == 4) for it in items]
    hs, ws = [it.shape[-3] for it in items], [it.shape[-2] for it in items]
    offs, total = [], 0
    for it, f, h, w in zip(items, nf, hs, ws):
        offs += [total + k * h * w * 3 for k in range(f)]
        total += it.size
    src = torch.from_numpy(np.concatenate([it.reshape(-1) for it in items])).to(dev)
    grid, rows, need = (i32 * (3 * n))(), C.c_int64(0), C.c_size_t(0)
    if lib.vqa_qwen_preprocess_video_plan(arr(i32, nf), arr(i32, hs), arr(i32, ws), arr(i32, vid), n, PATCH, TEMPORAL, MERGE, pixels[0],
                                          pixels[1], grid, C.byref(rows), C.byref(need)):
        raise RuntimeError(_lib.last_error(None))
    width = 3 * TEMPORAL * PATCH * PATCH
    buf, out = guarded(rows.value * width, dtype, dev)
    wsb = torch.empty(max(need.value, 16), dtype=torch.uint8, device=dev)
    mean, std = (C.c_float * 3)(*CLIP_MEAN), (C.c_float * 3)(*CLIP_STD)
    dt = _lib.VQA_DTYPE_F32 if dtype == torch.float32 else _lib.VQA_DTYPE_BF16
    stream = torch.cuda.current_stream(dev).cuda_stream
    rc = lib.vqa_qwen_preprocess_video(src.data_ptr(), arr(i64, offs), arr(i32, nf), arr(i32, hs), arr(i32, ws), arr(i32, vid), n, PATCH,
                                       TEMPORAL, MERGE, pixels[0], pixels[1], mean, std, out.data_ptr(), dt, wsb.data_ptr(), wsb.numel(),
                                       None, stream)
    if rc:
        raise RuntimeError(_lib.last_error(None))
    assert_guards(buf)
    return out.view(rows.value, width), [tuple(grid[3 * i:3 * i + 3]) for i in range(n)]


def first_mismatch(got, want, bounds):
    """Index of the first item (row ranges `bounds`) where got != want, with its largest difference, for the failure message."""
    for i, (lo, hi) in enumerate(bounds):
        if not torch.equal(got[lo:hi], want[lo:hi]):
            return f"item {i}: max diff {float((got[lo:hi].float() - want[lo:hi].float()).abs().max())}"
    return "shapes differ"


def sweep(force_tiles, axes, tile_cols, run, layout_geometry, auto):
    """Force every (tile_rows, chunk_groups, tile_cols) plan on images small enough for all of them to fit: each must be the geometry
    the planner reports and reproduce `auto` bit for bit."""
    widths = [len(ax[0][0]) for ax in axes]
    for tr, cg, tc in itertools.product(TILE_ROWS, CHUNKS, tile_cols):
        assert all(plan_needs(ax, tr, tc, cg)[0] <= PRE_MAX_SMEM for ax in axes)
        force_tiles(tr, tc, cg)
        assert [g[:4] for g in layout_geometry()] == [(tr, min(tc, w), -(-w // min(tc, w)), cg) for w in widths]
        got, bounds = run()
        assert torch.equal(got, auto), f"plan ({tr} rows, chunk {cg}, {tc} cols): {first_mismatch(got, auto, bounds)}"


# (h, w): 333 * 517 is odd, so every later image starts at a byte offset that is not a multiple of 4 and its rows alternate between the
# aligned 12-byte staging loads and the byte gather; 40 x 70 is upscaled, the rest downscaled by up to 2.7.
CLIP_SWEEP = [(333, 517), (40, 70), (901, 600), (480, 853), (700, 700), (305, 899)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("pad", [True, False])
def test_clip_every_tile_plan_bit_exact(dev, force_tiles, pad, dtype):
    S = 336
    imgs = [photo(h, w, i) for i, (h, w) in enumerate(CLIP_SWEEP)]
    ref = torch.stack([orc.clip_preprocess(Image.fromarray(a), S, pad=pad) for a in imgs]).to(dev, dtype)
    bounds = [(i, i + 1) for i in range(len(imgs))]
    auto = run_clip(imgs, S, pad, dtype, dev)
    assert torch.equal(auto, ref), first_mismatch(auto, ref, bounds)
    axes = [clip_axes(h, w, S, pad) for h, w in CLIP_SWEEP]
    # one column tile; a multiple of 128; under PRE_XL (128 lanes); odd; S - 1 (a last tile of one column)
    sweep(force_tiles, axes, (WHOLE, 256, 100, 173, S - 1), lambda: (run_clip(imgs, S, pad, dtype, dev), bounds),
          lambda: geometry(0, CLIP_SWEEP, S, pad), auto)


# (h, w, frames) at (min_pixels, 512 * 28 * 28): 333 x 517 -> 336 x 504 (odd byte size, as above; up in height, down in width),
# 40 x 70 -> 56 x 84 (min_pixels upscale), a 3-frame stack 610 x 590 -> 616 x 588 (up / down; its last frame fills both temporal
# slots), 901 x 600 -> 756 x 504 and 700 x 700 -> 616 x 616 (max_pixels downscale), 305 x 899 -> 308 x 896 (up / down).
QWEN_SWEEP = [(333, 517, 0), (40, 70, 0), (610, 590, 3), (901, 600, 0), (480, 853, 0), (305, 899, 0), (700, 700, 0)]
QWEN_SWEEP_PIXELS = (PLUGIN_PIXELS[0], 512 * 28 * 28)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_qwen_every_tile_plan_bit_exact(dev, force_tiles, dtype):
    items = [photo(h, w, i) if not f else np.stack([photo(h, w, 10 * i + k) for k in range(f)]) for i, (h, w, f) in enumerate(QWEN_SWEEP)]
    refs = [qwen_reference(it, *QWEN_SWEEP_PIXELS, device=dev) for it in items]
    ref = torch.cat([r for r, _ in refs]).to(dtype)
    ends = np.cumsum([len(r) for r, _ in refs]).tolist()
    bounds = list(zip([0] + ends[:-1], ends))
    auto, grids = run_qwen(items, dtype, dev, QWEN_SWEEP_PIXELS)
    assert grids == [g for _, g in refs]
    assert torch.equal(auto, ref), first_mismatch(auto, ref, bounds)
    axes = [qwen_axes(h, w, *QWEN_SWEEP_PIXELS) for h, w, _ in QWEN_SWEEP]
    first_w = len(axes[0][0][0])
    frames = [f for _, _, f in QWEN_SWEEP]
    sweep(force_tiles, axes, (WHOLE, 256, 100, 173, first_w - 1), lambda: (run_qwen(items, dtype, dev, QWEN_SWEEP_PIXELS)[0], bounds),
          lambda: geometry(1, [(h, w) for h, w, _ in QWEN_SWEEP], pixels=QWEN_SWEEP_PIXELS, frames=frames), auto)


@pytest.mark.parametrize("h,w,frames,pixels", QWEN_PRODUCTION, ids=[f"{h}x{w}{f'x{f}f' if f else ''}-{p[1]}" for h, w, f, p in QWEN_PRODUCTION])
def test_qwen_production_geometry_bit_exact(dev, h, w, frames, pixels):
    item = photo(h, w, h + w) if not frames else np.stack([photo(h, w, h + w + k) for k in range(frames)])
    got, grids = run_qwen([item], torch.float32, dev, pixels)
    ref, grid = qwen_reference(item, *pixels, device=dev)
    assert grids == [grid]
    assert torch.equal(got, ref), first_mismatch(got, ref, [(0, len(ref))])


@pytest.mark.parametrize("h,w,size,pad", CLIP_PRODUCTION)
def test_clip_production_geometry_bit_exact(dev, h, w, size, pad):
    a = photo(h, w, h * 7 + w)
    ref = orc.clip_preprocess(Image.fromarray(a), size, pad=pad) if max(h, w) <= 2000 else pil_reference(a, size)
    got = run_clip([a], size, pad, torch.float32, dev)
    assert torch.equal(got[0].cpu(), ref), f"max diff {float((got[0].cpu() - ref).abs().max())}"

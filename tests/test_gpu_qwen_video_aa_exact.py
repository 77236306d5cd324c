"""video_resize_aa_kernel (csrc/preprocess.cuh), the antialiased bicubic resize of Qwen2.5-VL video files, bit for bit against its host
restatement (tests/aa_resize_ref.py) under every row-tile plan and at qwen_vl_utils' own frame budgets.

The planner gives each CTA 32, 16, 8, 4, 2 or 1 output rows, the most whose band of input rows fits 96 KB of shared memory; a plan
moves which input rows a CTA stages and where each output's window starts in the band. Every test runs the device path of
engine.qwen_preprocess_video_file_u8, recovers the uint8 frames from the patch rows and asserts with torch.equal that they are the
restatement's and that the patch rows, in fp32 and bf16, are the processor layout of the restated frames. A mismatch is reported with
its frame, pixel, row tile and 64-column tile."""
import ctypes as C

import numpy as np
import pytest
import torch

import aa_resize_ref as ar
from t2v_metrics_b200 import _lib, engine
from t2v_metrics_b200.models.vqascore_models import qwen_utils as qu
from test_gpu_qwen_video_file import device_levels

pytestmark = pytest.mark.gpu

SENTINEL = -1232.0                  # exact in fp32, and no normalised pixel value


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda", 0)


@pytest.fixture
def aa_rows():
    """Forces vqa_debug_set_preprocess_aa_rows, and leaves it automatic whatever the test did."""
    lib = _lib.load()

    def force(tile_rows):
        assert lib.vqa_debug_set_preprocess_aa_rows(tile_rows) == 0
    try:
        yield force
    finally:
        assert lib.vqa_debug_set_preprocess_aa_rows(0) == 0


def random_frames(n, src, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, *src, 3), dtype=np.uint8)


def smooth_like(n, h, w, seed):
    """The moving gradients of test_qwen_video_file_host.smooth_frames with +-3 levels of noise, built by broadcasting so that 8K
    frames stay cheap."""
    rng = np.random.default_rng(seed)
    y, x = np.arange(h, dtype=np.float32)[:, None], np.arange(w, dtype=np.float32)[None, :]
    out = np.empty((n, h, w, 3), np.uint8)
    for f in range(n):
        for c, v in enumerate((128 + 100 * np.sin(x / 9 + f / 2 + seed), 128 + 100 * np.cos(y / 7 - f / 3),
                               128 + 90 * np.sin((x + y) / 13 + f))):
            out[f, ..., c] = np.clip(v + rng.integers(-3, 4, (h, w), dtype=np.int8), 0, 255)
    return out


def locate(got, want, value, tile_rows, rows=None):
    """The first mismatching element: frame, output pixel and channel, its row tile and 64-column tile, both levels and the fp32 value."""
    f, i, x, c = (int(v) for v in np.argwhere(got != want)[0])
    y = int(rows[i]) if rows is not None else i
    return (f"{int((got != want).sum())} levels differ; first at frame {f} pixel (y {y}, x {x}) channel {c}: row tile {y // tile_rows} "
            f"of {tile_rows} rows, column tile {x // ar.AA_TX}; device {got[f, i, x, c]} restatement {want[f, i, x, c]} "
            f"(fp32 {value[f, i, x, c]!r})")


def device_rows(frames, size, dev, dtype=torch.float32):
    rows, grid = engine.qwen_preprocess_video_file_u8(torch.from_numpy(frames), size, dev, out_dtype=dtype)
    n = len(frames)
    assert grid == (-(-n // 2), size[0] // 14, size[1] // 14)
    return rows.cpu(), grid


def assert_exact(frames, size, dev, want, value, tile_rows, bf16=True):
    """The device's levels are `want` (the restated uint8 frames) and its patch rows the processor layout of them, in fp32 (and bf16)."""
    got, grid = device_rows(frames, size, dev)
    lv = device_levels(got, grid)[:len(frames)].numpy()
    assert np.array_equal(lv, want), locate(lv, want, value, tile_rows)
    ref, g = qu._video_patch_rows(torch.from_numpy(want).permute(0, 3, 1, 2).float(), 14, 2, 2)
    assert g == grid and torch.equal(got, ref)
    if bf16:
        assert torch.equal(device_rows(frames, size, dev, torch.bfloat16)[0], ref.to(torch.bfloat16))


def assert_refused_before_launch(frames, size, dev, match):
    """vqa_qwen_preprocess_video_aa_plan refuses the resize, and vqa_qwen_preprocess_video_aa refuses it without writing a byte."""
    lib = _lib.load()
    (fh, wh, th), (fv, wv, tv) = engine._aa_bicubic_taps(frames.shape[2], size[1]), engine._aa_bicubic_taps(frames.shape[1], size[0])
    ip = lambda t: C.cast(t.data_ptr(), C.POINTER(C.c_int32))
    fp = lambda t: C.cast(t.data_ptr(), C.POINTER(C.c_float))
    n, h, w = frames.shape[:3]
    with pytest.raises(RuntimeError, match=match):
        engine.qwen_preprocess_video_file_u8(torch.from_numpy(frames), size, dev)
    rows, need = C.c_int64(0), C.c_size_t(0)
    assert lib.vqa_qwen_preprocess_video_aa_plan(h, w, *size, ip(fh), th, ip(fv), tv, 14, 2, 2, n, C.byref(rows), C.byref(need)) != 0
    assert match in _lib.last_error(None)
    src = torch.from_numpy(frames).to(dev)
    out = torch.full((-(-n // 2) * (size[0] // 14) * (size[1] // 14), 1176), SENTINEL, device=dev)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    rc = lib.vqa_qwen_preprocess_video_aa(src.data_ptr(), n, 0, n, h, w, *size, ip(fh), fp(wh), th, ip(fv), fp(wv), tv, 14, 2, 2,
                                          (C.c_float * 3)(*engine.CLIP_MEAN), (C.c_float * 3)(*engine.CLIP_STD), out.data_ptr(),
                                          _lib.VQA_DTYPE_F32, ws.data_ptr(), ws.numel(), None, engine._stream_ptr(dev))
    assert rc != 0 and match in _lib.last_error(None)
    torch.cuda.synchronize(dev)
    assert bool((out == SENTINEL).all()), "a refused resize wrote to its output"


# ---------------------------------------------------------------------------------------------- every automatic plan
@pytest.mark.parametrize("src,size,tile", ar.AUTO_PLANS, ids=[f"{s[0]}x{s[1]}-{z[0]}x{z[1]}-plan{t}" for s, z, t in ar.AUTO_PLANS])
def test_every_automatic_plan_bit_exact(dev, src, size, tile):
    g = ar.aa_geometry(src, size)
    print(f"\n[aa plan] {src} -> {size}: tile_rows {g[0]}, band_rows {g[1]}, tiles_x {g[2]}")
    assert g[0] == tile
    frames = random_frames(3, src, src[0] * 3 + src[1])
    want, value = ar.aa_resize_u8(frames, size)
    assert_exact(frames, size, dev, want, value, tile)


# ---------------------------------------------------------------------------------------------- every forced plan
def test_every_forced_plan_bit_exact(dev, aa_rows):
    """Row counts 1 ... 32 (powers of two or not, most ending on a partial row tile) at a geometry where all fit, and at a steep one
    where 1 ... 29 fit and the rest are refused before any launch."""
    forced = {}
    for (src, size) in (ar.FORCED, ar.STEEP):
        frames = random_frames(3, src, 11 * src[0] + src[1])
        want, value = ar.aa_resize_u8(frames, size)
        for t in range(1, 33):
            aa_rows(t)
            plan = ar.plan_aa(src[0], size[0], t)
            if plan is None:
                assert_refused_before_launch(frames, size, dev, "vqa_debug_set_preprocess_aa_rows")
                continue
            assert ar.aa_geometry(src, size)[:2] == plan
            assert_exact(frames, size, dev, want, value, t, bf16=t in (1, 7, 32))
            forced.setdefault((src, size), []).append(t)
        aa_rows(0)
    print(f"\n[aa forced plans] {forced}")
    assert forced[ar.FORCED] == list(range(1, 33)) and {7, 11, 13} <= set(forced[ar.STEEP])


# ---------------------------------------------------------------------------------------------- the refusal boundary
def test_refusal_boundary(dev):
    """123 vertical taps (1736 -> 56) run with one output row per CTA, bit-exact; 128 taps (1792 -> 56) have no plan and are refused."""
    src, size, tile = ar.AUTO_PLANS[-1]
    assert src[0] == 1736 and ar.aa_geometry(src, size)[:2] == (1, 123) == (tile, ar.taps(src[0], size[0])[2])
    frames = random_frames(2, src, 1736)
    want, value = ar.aa_resize_u8(frames, size)
    assert_exact(frames, size, dev, want, value, 1, bf16=False)
    assert ar.taps(ar.REFUSED[0][0], ar.REFUSED[1][0])[2] == 128
    assert_refused_before_launch(random_frames(2, *ar.REFUSED[:1], 1792), ar.REFUSED[1], dev, "downscale too steep")


# ---------------------------------------------------------------------------------------------- qwen_vl_utils' own frame budgets
@pytest.mark.parametrize("name,size", ar.PRODUCTION, ids=[f"{n}-{s[0]}x{s[1]}" for n, s in ar.PRODUCTION])
def test_production_budgets_bit_exact(dev, name, size):
    """Two frames at full source size resized to what qwen_video_file_plan gives a 4-frame and a 3000-frame clip. 1080p is restated
    whole; 4K and 8K at every row tile's first and last output row plus 64 random rows. The whole output is also checked against
    torchvision on the host within the +-1-at-ties rule of test_gpu_qwen_video_file.py."""
    src = ar.SOURCES[name]
    tile, band, tiles_x = ar.aa_geometry(src, size)
    print(f"\n[aa production] {name} {src} -> {size} ({'; '.join(ar.production_sizes(name)[size])}): tile_rows {tile}, band_rows {band}")
    frames = smooth_like(2, *src, seed=src[0] + src[1])
    got, grid = device_rows(frames, size, dev)
    lv = device_levels(got, grid)[:2]
    rows = None
    if name != "1080p":
        starts = np.arange(0, size[0], tile)
        rng = np.random.default_rng(size[0] * 7 + src[1])
        rows = np.unique(np.concatenate([starts, np.minimum(starts + tile, size[0]) - 1, rng.choice(size[0], 64, replace=False)]))
    want, value = ar.aa_resize_u8(frames, size, rows=rows)
    sel = lv.numpy() if rows is None else lv.numpy()[:, rows]
    assert np.array_equal(sel, want), locate(sel, want, value, tile, rows)
    ref, g = qu._video_patch_rows(lv.permute(0, 3, 1, 2).float(), 14, 2, 2)
    assert g == grid and torch.equal(got, ref)
    assert torch.equal(device_rows(frames, size, dev, torch.bfloat16)[0], ref.to(torch.bfloat16))
    tv, _, _ = qu.qwen_video_file_to_patches(frames, size)
    diff = lv.int() - tv.int()
    bad = diff != 0
    exact = ar.torch_fp32(frames, size)[bad]
    print(f"[aa production] {int(bad.sum())} of {bad.numel()} levels differ from torchvision")
    assert int(diff.abs().max()) <= 1
    assert bool(((exact - exact.floor() - 0.5).abs() <= 1e-3).all())


# ---------------------------------------------------------------------------------------------- slices
@pytest.mark.parametrize("slice_frames", [1, 2, 3])
def test_slices_equal_the_restated_stack(dev, monkeypatch, slice_frames):
    """7 frames sent in slices of 1, 2 or 3 frames at a plan-8 geometry: later slices start at frame0 > 0 and the odd last frame fills
    both temporal slots of its patch rows."""
    src, size = ar.SLICED
    assert ar.aa_geometry(src, size)[0] == 8
    frames = random_frames(7, src, 4320 + slice_frames)
    want, value = ar.aa_resize_u8(frames, size)
    monkeypatch.setattr(engine, "VIDEO_SLICE_BYTES", slice_frames * src[0] * src[1] * 3)
    assert_exact(frames, size, dev, want, value, 8)


# ---------------------------------------------------------------------------------------------- the fixtures discriminate
def test_fixtures_catch_the_mistaken_restatements():
    """Over the frames of the automatic-plan and forced-plan tests, the mistaken restatements change this many uint8 outputs: taps
    summed last to first, product and sum rounded separately, every vertical window one input row lower. A kernel making one of these
    mistakes fails those tests."""
    counts, total = {"reversed": 0, "no fma": 0, "window + 1": 0}, 0
    fixtures = [(random_frames(3, s, s[0] * 3 + s[1]), z) for s, z, _ in ar.AUTO_PLANS]
    fixtures += [(random_frames(3, s, 11 * s[0] + s[1]), z) for s, z in (ar.FORCED, ar.STEEP)]
    for frames, size in fixtures:
        want, _ = ar.aa_resize_u8(frames, size)
        total += want.size
        for name, kw in (("reversed", dict(order="reversed")), ("no fma", dict(fma=False)), ("window + 1", dict(vshift=1))):
            counts[name] += int((ar.aa_resize_u8(frames, size, **kw)[0] != want).sum())
    print(f"\n[aa mistakes] of {total} outputs changed: {counts}")
    assert counts["reversed"] > 0 and counts["no fma"] > 0 and counts["window + 1"] > 0.01 * total

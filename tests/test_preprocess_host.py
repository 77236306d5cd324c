"""Host logic of the device pre-processing (SURVEY 8(f)2), no GPU: the fixed-point bicubic tap tables libvqa_b200.so builds
(vqa_resample_table, the same code vqa_clip_preprocess uploads to the device) must reproduce Pillow's resize bit for bit when the
two integer passes are replayed in numpy, and the geometry must match the reference's CLIP processor (shortest edge -> S, centre crop)."""
import ctypes as C

import numpy as np
import pytest
import torch
from PIL import Image

import preprocess_ref as pr
from oracle import clipt5_oracle as orc
from t2v_metrics_b200 import _lib

PREC = 22


def table(in_size, out_size, first=0, count=None):
    lib = _lib.load()
    count = out_size - first if count is None else count
    ks = lib.vqa_resample_table(in_size, out_size, first, count, None, None)
    assert ks > 0
    b = (C.c_int32 * (2 * count))()
    k = (C.c_int32 * (ks * count))()
    assert lib.vqa_resample_table(in_size, out_size, first, count, b, k) == ks
    return np.array(b, dtype=np.int64).reshape(count, 2), np.array(k, dtype=np.int64).reshape(count, ks)


def resample_axis(img, bounds, kk):
    """One pass along axis 1 of [rows, n, 3] uint8 with Resample.c's rounding: (sum + 2^21) >> 22 clipped to uint8."""
    out = np.empty((img.shape[0], bounds.shape[0], 3), dtype=np.uint8)
    src = img.astype(np.int64)
    for xx, (x0, n) in enumerate(bounds):
        acc = (src[:, x0:x0 + n, :] * kk[xx, :n][None, :, None]).sum(axis=1) + (1 << (PREC - 1))
        out[:, xx, :] = np.clip(acc >> PREC, 0, 255).astype(np.uint8)
    return out


def replay_resize(arr, nw, nh):
    h, w = arr.shape[:2]
    hb, hk = table(w, nw)
    vb, vk = table(h, nh)
    tmp = resample_axis(arr, hb, hk)                                        # horizontal first, rounded to uint8
    return resample_axis(tmp.transpose(1, 0, 2), vb, vk).transpose(1, 0, 2)  # then vertical


@pytest.mark.parametrize("w,h,nw,nh", [(512, 512, 336, 336), (640, 400, 537, 336), (300, 500, 336, 560), (200, 150, 448, 336),
                                       (336, 336, 336, 336), (1000, 37, 336, 12), (97, 1301, 25, 336)])
def test_tables_reproduce_pillow_resize(w, h, nw, nh):
    rng = np.random.RandomState(w * 7 + h)
    arr = rng.randint(0, 256, (h, w, 3), dtype=np.uint8)
    ref = np.asarray(Image.fromarray(arr).resize((nw, nh), resample=Image.BICUBIC))
    got = replay_resize(arr, nw, nh)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), f"max diff {np.abs(got.astype(int) - ref.astype(int)).max()}"


def test_table_slices_and_identity():
    b, k = table(512, 336)
    b2, k2 = table(512, 336, 100, 50)
    assert np.array_equal(b[100:150], b2) and np.array_equal(k[100:150], k2)
    bi, ki = table(336, 336)
    for xx in range(336):                       # same size: a single tap of exactly 1.0 on the pixel itself
        x0, n = bi[xx]
        taps = {int(x0 + j): int(ki[xx, j]) for j in range(n) if ki[xx, j] != 0}
        assert taps == {xx: 1 << PREC}
    assert _lib.load().vqa_resample_table(0, 336, 0, 336, None, None) == 0
    assert "bad resample" in _lib.last_error(None)


@pytest.mark.parametrize("w,h", [(512, 512), (640, 400), (300, 500), (123, 77)])
def test_replayed_pipeline_equals_oracle_preprocess(w, h):
    """expand2square + resize + crop + normalise replayed with the library's tables == oracle.clip_preprocess (PIL path)."""
    rng = np.random.RandomState(w + h)
    arr = rng.randint(0, 256, (h, w, 3), dtype=np.uint8)
    ref = orc.clip_preprocess(Image.fromarray(arr), 336)
    side = max(w, h)
    canvas = np.empty((side, side, 3), dtype=np.uint8)
    canvas[:] = np.array([int(x * 255) for x in orc.CLIP_MEAN], dtype=np.uint8)
    canvas[(side - h) // 2:(side - h) // 2 + h, (side - w) // 2:(side - w) // 2 + w] = arr
    u8 = replay_resize(canvas, 336, 336)
    x = u8.astype(np.float32) / np.float32(255.0)
    x = (x - np.asarray(orc.CLIP_MEAN, dtype=np.float32)) / np.asarray(orc.CLIP_STD, dtype=np.float32)
    assert torch.equal(torch.from_numpy(x).permute(2, 0, 1), ref)


def test_workspace_sizing_and_errors():
    lib = _lib.load()
    H, W = (C.c_int32 * 3)(512, 400, 512), (C.c_int32 * 3)(512, 640, 512)
    n = lib.vqa_clip_preprocess_workspace_bytes(H, W, 3, 336, 1)
    assert n > 0
    one = lib.vqa_clip_preprocess_workspace_bytes((C.c_int32 * 1)(512), (C.c_int32 * 1)(512), 1, 336, 1)
    assert 0 < one < n                                              # tables are shared between images of the same canvas size
    assert lib.vqa_clip_preprocess_workspace_bytes((C.c_int32 * 1)(0), (C.c_int32 * 1)(5), 1, 336, 1) == 0
    # a 200000-pixel-high strip cannot keep its vertical window in shared memory: refused, not mangled
    assert lib.vqa_clip_preprocess_workspace_bytes((C.c_int32 * 1)(200000), (C.c_int32 * 1)(200000), 1, 336, 1) == 0
    assert "too large" in _lib.last_error(None)


def test_qwen_plan_matches_python_smart_resize():
    """vqa_qwen_preprocess_video_plan (C++ smart_resize incl. Python's round-half-even) == qwen_utils.smart_resize on a sweep of sizes,
    including the min-pixel and max-pixel branches and exact .5 ties (h / 28 = k + 0.5)."""
    from t2v_metrics_b200.engine import qwen_preprocess_plan
    from t2v_metrics_b200.models.vqascore_models.qwen_utils import smart_resize
    rng = np.random.RandomState(0)
    sizes = [(448, 448), (14, 14), (42, 70), (126, 98), (30, 30), (40, 2000), (3000, 4000), (1003, 1003), (2047, 777), (98, 154)]
    sizes += [(int(a), int(b)) for a, b in rng.randint(20, 2500, (60, 2))]
    grids, total, wsb = qwen_preprocess_plan(sizes)
    ref = [smart_resize(h, w) for h, w in sizes]
    assert [(g[1] * 14, g[2] * 14) for g in grids] == ref
    assert total == sum(h // 14 * (w // 14) for h, w in ref) and wsb > 0
    with pytest.raises(RuntimeError, match="aspect ratio"):
        qwen_preprocess_plan([(10, 2500)])


# ---------------------------------------------------------------------------------------------- tile plans of image_preprocess_kernel
@pytest.fixture
def automatic_plans():
    """Leaves the process-wide tile-plan override at automatic whatever the test did."""
    yield _lib.load()
    assert _lib.load().vqa_debug_set_preprocess_tiles(0, 0, 0) == 0


@pytest.mark.parametrize("layout", ["clip", "qwen"])
def test_production_geometries_reach_every_plan_branch(layout):
    """The automatic plans of the GPU production list (tests/test_gpu_preprocess_tiles.py) include, in each output layout, column tiles,
    one 4-row group staged per pass, and at most 4 output rows per CTA over a single column tile -- so that list keeps running those
    kernel paths bit-exactly against Pillow if the planner's cost model changes."""
    if layout == "clip":
        plans = [pr.geometry(0, [(h, w)], size, pad)[0] for h, w, size, pad in pr.CLIP_PRODUCTION]
    else:
        plans = [pr.geometry(1, [(h, w)], pixels=px, frames=[f])[0] for h, w, f, px in pr.QWEN_PRODUCTION]
    assert any(g[2] > 1 for g in plans), plans
    assert any(g[3] == 1 for g in plans), plans
    assert any(g[0] <= 4 and g[2] == 1 for g in plans), plans


def random_items(n, seed):
    """n seeded (layout, axes, geometry call) triples over the CLIP (pad on / off, S 224 / 336) and Qwen (plugin bounds and
    max_pixels 1003520) planners, sizes log-uniform from 1 to 40000 px a side."""
    rng = np.random.default_rng(seed)
    items = []
    while len(items) < n:
        h, w = (int(v) for v in np.exp(rng.uniform(0, np.log(40000), 2)))
        if rng.random() < 0.5:
            size, pad = int(rng.choice([224, 336])), bool(rng.random() < 0.5)
            if pad and max(h, w) > 65500:
                continue
            items.append(("clip", pr.clip_axes(h, w, size, pad), lambda h=h, w=w, s=size, p=pad: pr.geometry(0, [(h, w)], s, p)[0]))
        else:
            if max(h, w) / min(h, w) > 200:
                continue
            px = pr.PLUGIN_PIXELS if rng.random() < 0.5 else (pr.PLUGIN_PIXELS[0], 1003520)
            items.append(("qwen", pr.qwen_axes(h, w, *px), lambda h=h, w=w, px=px: pr.geometry(1, [(h, w)], pixels=px)[0]))
    return items


def test_automatic_plans_fit_and_cover_their_windows():
    """For seeded random geometries, the automatic plan fits the shared-memory budget (restated from the tap tables), its column tiles
    cover the output width with no empty tile, and its band holds the 4-row groups of every row tile's vertical windows."""
    for layout, axes, plan in random_items(300, 0):
        tr, tc, ct, cg, band = plan()
        ow = len(axes[0][0])
        need, need_band = pr.plan_needs(axes, tr, tc, cg)
        assert 1 <= tr <= 32 and cg in (1, 2), (layout, tr, cg)
        assert tc * ct >= ow and (ct - 1) * tc < ow and (ct > 1 or tc == ow), (layout, ow, tc, ct)
        assert band >= need_band, (layout, band, need_band)
        assert need <= pr.PRE_MAX_SMEM, (layout, need)


def test_forced_plans_are_used_or_refused(automatic_plans):
    """A forced tile plan is used exactly when it fits shared memory and is refused with an error naming the override otherwise; bad
    override values are rejected and leave the override as it was; zeros restore every automatic plan."""
    lib = automatic_plans
    rng = np.random.default_rng(1)
    items = random_items(120, 2)
    auto = [plan() for _, _, plan in items]
    used = refused = 0
    for layout, axes, plan in items:
        tr, tc, cg = int(rng.choice([1, 2, 4, 8, 16, 32])), int(rng.integers(1, 2000)), int(rng.integers(1, 3))
        assert lib.vqa_debug_set_preprocess_tiles(tr, tc, cg) == 0
        ow = len(axes[0][0])
        try:
            g = plan()
        except RuntimeError as e:
            assert "vqa_debug_set_preprocess_tiles" in str(e)
            assert pr.plan_needs(axes, tr, tc, cg)[0] > pr.PRE_MAX_SMEM, (layout, tr, tc, cg)
            refused += 1
            continue
        assert pr.plan_needs(axes, tr, tc, cg)[0] <= pr.PRE_MAX_SMEM
        assert g[:4] == (tr, min(tc, ow), -(-ow // min(tc, ow)), cg) and g[4] == pr.plan_needs(axes, tr, tc, cg)[1]
        used += 1
    assert used >= 40 and refused >= 10, (used, refused)
    # a 4000 x 6000 photo at the Qwen plugin's bounds needs column tiles: one 32-row tile over all 4368 columns does not fit
    assert lib.vqa_debug_set_preprocess_tiles(32, 1 << 16, 2) == 0
    with pytest.raises(RuntimeError, match="vqa_debug_set_preprocess_tiles"):
        pr.geometry(1, [(4000, 6000)])
    # out-of-range values are rejected and keep the override in force
    assert lib.vqa_debug_set_preprocess_tiles(4, 100, 1) == 0
    for bad in [(0, 100, 1), (4, 0, 1), (4, 100, 0), (33, 100, 1), (4, 100, 3), (-1, 100, 1), (4, -5, 1)]:
        assert lib.vqa_debug_set_preprocess_tiles(*bad) != 0, bad
    assert pr.geometry(0, [(512, 512)])[0][:4] == (4, 100, 4, 1)
    assert lib.vqa_debug_set_preprocess_tiles(0, 0, 0) == 0
    assert [plan() for _, _, plan in items] == auto


def test_qwen_restatement_equals_the_plugin_path():
    """tests/preprocess_ref.qwen_reference (Pillow's uint8 resize, a 768-entry normalisation table, patch rows by reshape) equals the
    plugin's CPU path at its pixel bounds: noise that smart_resize leaves at its size (84 x 140), so that every level of every channel
    goes through the table, a resized photo, and a 3-frame stack."""
    from t2v_metrics_b200.models.vqascore_models.qwen_utils import qwen_image_to_patches, qwen_video_to_patches
    mn, mx = pr.PLUGIN_PIXELS
    noise = np.random.default_rng(3).integers(0, 256, (84, 140, 3), dtype=np.uint8)
    assert all(len(np.unique(noise[..., c])) == 256 for c in range(3))
    for a in (noise, pr.photo(333, 517, 4)):
        got, grid = pr.qwen_reference(a, mn, mx)
        ref, gref = qwen_image_to_patches(Image.fromarray(a), min_pixels=mn, max_pixels=mx)
        assert grid == gref and torch.equal(got, ref)
    stack = np.stack([pr.photo(61, 95, k) for k in range(3)])
    got, grid = pr.qwen_reference(stack, mn, mx)
    ref, gref = qwen_video_to_patches(stack, min_pixels=mn, max_pixels=mx)
    assert grid == gref and torch.equal(got, ref)

"""Host restatement of video_resize_aa_kernel (csrc/preprocess.cuh), the antialiased bicubic resize of Qwen2.5-VL video files, and of its
row-tile planner (pre_plan_aa).

The kernel's arithmetic is fully specified: for every output, a horizontal fp32 pass over torch's own fp32 weights, then a vertical
fp32 pass over those rows, each a chain of single-rounding fused multiply-adds in tap order starting from +0, then round half to even
and a clamp to [0, 255]. aa_resize_u8 computes exactly that on the host, so the device's uint8 frames can be compared bit for bit.
Python has no math.fma and numpy has none, so fmaf builds one from fp64 arithmetic."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from t2v_metrics_b200 import _lib
from t2v_metrics_b200.engine import _aa_bicubic_taps

AA_TX = 64                          # preprocess.cuh PRE_AA_TX: output columns per CTA
AA_MAX_SMEM = 96 * 1024             # preprocess.cuh PRE_AA_MAX_SMEM: the band's shared-memory budget


def fmaf(a, b, c):
    """fp32 fused multiply-add a * b + c, rounded once to nearest even, over numpy arrays of fp32 values (uint8 levels count as fp32).

    The product of two fp32 values has at most 48 significant bits, so it is exact in fp64. s = fl64(p + c) is then rounded to fp32.
    That second rounding is wrong only when s lies exactly on an fp32 midpoint while p + c does not: the tie must then go toward the
    remainder of the fp64 sum (TwoSum), not to the even neighbour. Everywhere else fp32(s) is already the correctly rounded result."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    p, c = np.broadcast_arrays(p, c)
    s = p + c
    r = s.astype(np.float32)
    # Candidates: an fp32-normal midpoint has 25 significant bits, the last one set, so its low 29 fp64 mantissa bits are 1 << 28.
    # Below fp32's normal range the spacing is fixed and every element is checked in full.
    cand = ((s.view(np.int64) & 0x1FFFFFFF) == 0x10000000) | (np.abs(s) < 2.0 ** -126)
    if cand.any():
        st, rt = s[cand], r[cand].astype(np.float64)
        d = st - rt                                 # exact: s and its fp32 rounding differ in at most 29 bits
        other = rt + 2.0 * d                        # s's mirror image past r; an fp32 exactly when s is a midpoint
        tie = (d != 0) & (other.astype(np.float32) == other)
        pt, ct = p[cand], c[cand]
        bb = st - pt
        err = (pt - (st - bb)) + (ct - bb)          # TwoSum: p + c == s + err exactly
        r[cand] = np.where(tie & (err * d > 0), other, rt).astype(np.float32)
    return r


def mul_add_f32(a, b, c):
    """a * b rounded to fp32, then + c rounded to fp32: the kernel's arithmetic without the fused multiply-add."""
    return np.asarray(a, np.float32) * np.asarray(b, np.float32) + np.asarray(c, np.float32)


def taps(in_size, out_size):
    """engine._aa_bicubic_taps as numpy: (first input of each window int64 [out], fp32 weights [out, taps], taps)."""
    first, w, t = _aa_bicubic_taps(in_size, out_size)
    return first.numpy().astype(np.int64), w.numpy(), t


def aa_resize_u8(frames, size, rows=None, order="forward", fma=True, vshift=0):
    """uint8 frames [n, h, w, 3] -> (uint8 [n, len(rows), rw, 3], fp32 values before rounding), the two passes of video_resize_aa_kernel
    to size = (rh, rw).

    rows: the output rows to restate (all by default); the horizontal pass then runs only for the input rows their windows read.
    order="reversed", fma=False and vshift=k are mistaken variants (taps summed last to first; product and sum rounded separately;
    every vertical window moved k input rows down, kept inside the frame) for checking that a fixture can tell them apart."""
    frames = np.asarray(frames, np.uint8)
    n, h, w, _ = frames.shape
    rh, rw = (int(v) for v in size)
    fh, wh, th = taps(w, rw)
    fv, wv, tv = taps(h, rh)
    fv = np.clip(fv + vshift, 0, h - tv)
    rows = np.arange(rh) if rows is None else np.asarray(rows, np.int64)
    step = fmaf if fma else mul_add_f32
    tap_order = (lambda k: range(k)) if order == "forward" else (lambda k: range(k - 1, -1, -1))
    need = np.unique((fv[rows][:, None] + np.arange(tv)).ravel())          # input rows the windows read; each window is contiguous
    band = np.empty((n, len(need), rw, 3), np.float32)

    def horizontal(k):                      # 32 input rows as [input column, (frame, row, channel)], so that each tap is a row gather
        x = frames[:, need[k:k + 32]]
        cols = x.transpose(2, 0, 1, 3).reshape(w, -1)
        acc = np.zeros((rw, cols.shape[1]), np.float32)
        for j in tap_order(th):
            acc = step(cols[fh + j], wh[:, j, None], acc)
        band[:, k:k + 32] = acc.reshape(rw, n, x.shape[1], 3).transpose(1, 2, 0, 3)
    with ThreadPoolExecutor(os.cpu_count()) as pool:        # numpy releases the GIL inside each operation
        list(pool.map(horizontal, range(0, len(need), 32)))
    pos = np.searchsorted(need, fv[rows])
    acc = np.zeros((n, len(rows), rw, 3), np.float32)
    for j in tap_order(tv):
        acc = step(band[:, pos + j], wv[rows, j][None, :, None, None], acc)
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8), acc


def torch_fp32(frames, size):
    """torch's own fp32 antialiased bicubic resize on this host's CPU, before rounding: [n, rh, rw, 3]."""
    x = torch.from_numpy(np.asarray(frames, np.uint8)).permute(0, 3, 1, 2).float()
    return torch.nn.functional.interpolate(x, size=list(size), mode="bicubic", antialias=True, align_corners=False).permute(0, 2, 3, 1)


# ---------------------------------------------------------------------------------------------- pre_plan_aa's row-tile choice, restated
def aa_smem_bytes(band_rows):
    """preprocess.cuh pre_aa_smem_bytes: the normalisation table and the fp32 band [3][band_rows][AA_TX]."""
    return (768 + 3 * band_rows * AA_TX) * 4


def band_rows(first_v, vtaps, tile_rows):
    """Input rows of the tallest band of tile_rows output rows (windows monotonic: first row of the first window .. end of the last)."""
    first_v = np.asarray(first_v, np.int64)
    y0 = np.arange(0, len(first_v), tile_rows)
    y1 = np.minimum(y0 + tile_rows, len(first_v)) - 1
    return int((first_v[y1] + vtaps - first_v[y0]).max())


def plan_aa(in_h, out_h, tile_rows=0):
    """(tile_rows, band_rows) of an in_h -> out_h resize: the forced tile_rows, or the most output rows in 32, 16, ..., 1 whose band fits
    AA_MAX_SMEM; None where the plan is refused."""
    fv, _, tv = taps(in_h, out_h)
    for tile in ([tile_rows] if tile_rows else [32, 16, 8, 4, 2, 1]):
        band = band_rows(fv, tv, tile)
        if aa_smem_bytes(band) <= AA_MAX_SMEM:
            return tile, band
    return None


def aa_geometry(src, size, patch=14, merge=2):
    """vqa_debug_preprocess_aa_geometry for an (in_h, in_w) -> size = (out_h, out_w) resize with engine._aa_bicubic_taps' windows:
    (tile_rows, band_rows, tiles_x) as vqa_qwen_preprocess_video_aa launches it; RuntimeError with the library's message if refused."""
    (fh, _, th), (fv, _, tv) = _aa_bicubic_taps(src[1], size[1]), _aa_bicubic_taps(src[0], size[0])
    ip = lambda t: C.cast(t.data_ptr(), C.POINTER(C.c_int32))
    g = (C.c_int32 * 3)()
    if _lib.load().vqa_debug_preprocess_aa_geometry(src[0], src[1], size[0], size[1], ip(fh), th, ip(fv), tv, patch, merge, g):
        raise RuntimeError(_lib.last_error(None))
    return tuple(g)


# ---------------------------------------------------------------------------------------------- geometries of the device tests
# ((in_h, in_w), (out_h, out_w), automatic tile_rows). The vertical axes reach every plan: an upscale (4 taps), 1080p's and 4K's
# vertical at qwen_vl_utils' budget of 560 rows (8 and 16 taps), then 31, 67, 96, 120 and 123 taps. Output heights are multiples of 28,
# so only plans of 8 rows and more can end on a partial row tile; these do. The widths 56 < 64 and 84, 140, 252 leave a partial
# 64-column tile, 252 from an upscale.
AUTO_PLANS = [((97, 61), (392, 252), 32), ((1080, 200), (560, 140), 32), ((2160, 300), (532, 84), 16), ((4320, 250), (588, 56), 8),
              ((952, 500), (56, 140), 4), ((1344, 61), (56, 252), 2), ((1680, 300), (56, 84), 1), ((1736, 200), (56, 56), 1)]
FORCED = ((168, 250), (112, 140))             # automatic plan 32; every forced row count 1 ... 32 fits
STEEP = ((2160, 300), (560, 84))              # automatic plan 16; forced 1 ... 29 fit, 30 ... 32 are refused
SLICED = ((4320, 160), (588, 56))             # plan 8
REFUSED = ((1792, 200), (56, 56))             # 128 vertical taps: no plan fits
SOURCES = {"1080p": (1080, 1920), "4K": (2160, 3840), "4K-portrait": (3840, 2160), "8K": (4320, 7680)}


def production_sizes(source):
    """{(out_h, out_w): [labels]} for one SOURCES entry: the sizes qwen_video_file_plan gives it at 30 fps for a 60-frame clip (4
    sampled frames) and a 3000-frame one (200 sampled frames, where the per-frame pixel budget applies), under qwen_vl_utils' own
    budget and under the Qwen plugin's per-element max_pixels."""
    from t2v_metrics_b200.models.vqascore_models import qwen_utils as qu
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import VIDEO_FILE_MAX_PIXELS
    h, w = SOURCES[source]
    out = {}
    for budget, max_pixels in (("qwen_vl_utils", None), ("plugin", VIDEO_FILE_MAX_PIXELS)):
        for total in (60, 3000):
            idx, _, size = qu.qwen_video_file_plan(total, 30.0, h, w, max_pixels=max_pixels)
            out.setdefault(tuple(size), []).append(f"{budget} {total} frames -> {len(idx)}")
    return out


PRODUCTION = [(name, size) for name in SOURCES for size in production_sizes(name)]

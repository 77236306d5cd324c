"""The host restatement of the antialiased video-file resize (tests/aa_resize_ref.py), no GPU: its fused multiply-add against glibc's
fmaf bit for bit, including at constructed fp32 midpoints where double rounding goes wrong; the whole resize against torch's own CPU
resize except at rounding ties; and its copy of the row-tile planner against the library's launch geometry
(vqa_debug_preprocess_aa_geometry) on every geometry the device tests run, with and without a forced row count."""
import ctypes as C

import numpy as np
import pytest

import aa_resize_ref as ar
from t2v_metrics_b200 import _lib
from test_gpu_qwen_video_file import CASES


def glibc_fmaf(a, b, c):
    libm = C.CDLL("libm.so.6")
    f = libm.fmaf
    f.restype, f.argtypes = C.c_float, [C.c_float] * 3
    return np.array([f(x, y, z) for x, y, z in zip(np.asarray(a, np.float32).tolist(), np.asarray(b, np.float32).tolist(),
                                                  np.asarray(c, np.float32).tolist())], np.float32)


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def weights(rng, n):
    """n weights drawn from torch's own antialiased bicubic tap tables, downscales and upscales (negative lobes included)."""
    w = np.concatenate([ar.taps(i, o)[1].ravel() for i, o in ((1080, 560), (4320, 560), (952, 56), (61, 252), (640, 504), (333, 308))])
    return rng.choice(w[w != 0], n)


def test_fmaf_equals_glibc_on_kernel_shaped_operands():
    """10^6 triples shaped like the kernel's two passes: uint8 level x weight + accumulator, and fp32 band value x weight + accumulator."""
    rng = np.random.default_rng(0)
    n = 500_000
    levels = rng.integers(0, 256, n).astype(np.float32)
    band = rng.uniform(-40, 300, n).astype(np.float32)
    for a in (levels, band):
        b = weights(rng, n)
        c = rng.uniform(-60, 320, n).astype(np.float32) * (rng.random(n) < 0.95)     # 5 % start from +0
        got, want = ar.fmaf(a, b, c), glibc_fmaf(a, b, c)
        assert np.array_equal(bits(got), bits(want)), int((bits(got) != bits(want)).sum())


def midpoint_triples(rng, n, shape):
    """n triples whose fp64 sum s = fl64(a*b + c) lies exactly on an fp32 midpoint while a*b + c does not. c is drawn in [2^e, 2^(e+1))
    and b is the fp32 nearest to t / a for t = +-2^(e-24), half an fp32 ulp of c; a*b then misses t by a relative 2^-24 at most, and
    the candidates kept are those where s has exactly 25 significant bits, the last one set, and TwoSum leaves a non-zero remainder."""
    out = []
    while sum(len(x[0]) for x in out) < n:
        m = 400_000
        e = rng.integers(-2, 9, m)
        a = rng.integers(1, 256, m).astype(np.float32) if shape == "level" else rng.uniform(1, 256, m).astype(np.float32)
        t = np.ldexp(np.where(rng.random(m) < 0.5, 1.0, -1.0), e - 24)
        b = (t / a.astype(np.float64)).astype(np.float32)
        c = np.ldexp(rng.uniform(1, 2, m), e).astype(np.float32)
        p = a.astype(np.float64) * b
        s = p + c
        scaled = np.ldexp(np.frexp(s)[0], 25)
        bb = s - p
        keep = (scaled == np.floor(scaled)) & (scaled % 2 == 1) & ((p - (s - bb)) + (c - bb) != 0)
        out.append((a[keep], b[keep], c[keep]))
    return tuple(np.concatenate(x)[:n] for x in zip(*out))


@pytest.mark.parametrize("shape", ["level", "band"])
def test_fmaf_at_fp32_midpoints_where_double_rounding_fails(shape):
    a, b, c = midpoint_triples(np.random.default_rng(1 if shape == "level" else 2), 10_000, shape)
    p = a.astype(np.float64) * b
    want = glibc_fmaf(a, b, c)
    naive = (p + c).astype(np.float32)
    wrong_naive = int((bits(naive) != bits(want)).sum())
    wrong = int((bits(ar.fmaf(a, b, c)) != bits(want)).sum())
    print(f"\n[fmaf midpoints, {shape} x weight] {len(a)} triples: double rounding wrong on {wrong_naive}, fmaf wrong on {wrong}")
    assert wrong_naive > 0 and wrong == 0


@pytest.mark.parametrize("src,size", CASES + [(s, z) for s, z, _ in ar.AUTO_PLANS] + [ar.STEEP[:2]],
                         ids=lambda v: "x".join(map(str, v)))
def test_restatement_equals_torch_except_at_rounding_ties(src, size):
    """aa_resize_u8 against torch's CPU interpolate(bicubic, antialias=True) + round half to even: equal except by one level where
    torch's own fp32 value is within 1e-3 of a tie, which a different summation order on this host's CPU may put on the other side."""
    frames = np.random.default_rng(src[0] * 7 + src[1]).integers(0, 256, (2, *src, 3), dtype=np.uint8)
    got, value = ar.aa_resize_u8(frames, size)
    exact = ar.torch_fp32(frames, size).numpy()
    want = np.clip(np.rint(exact), 0, 255).astype(np.uint8)
    bad = got != want
    print(f"\n[aa restatement {src} -> {size}] {int(bad.sum())} of {bad.size} differ from torch; max |fp32 - torch| "
          f"{float(np.abs(value - exact).max()):.2e}")
    assert int(np.abs(got.astype(int) - want).max()) <= 1
    assert np.all(np.abs(exact[bad] - np.floor(exact[bad]) - 0.5) <= 1e-3)
    assert float(np.abs(value - exact).max()) <= 1e-3


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


def test_plan_copy_equals_the_library_geometry(aa_rows):
    """On every geometry of tests/test_gpu_qwen_video_aa_exact.py the library's launch geometry is the Python copy's, the automatic
    plans are the ones that module aims at, and a forced row count is used exactly when its band fits, else refused naming the override."""
    plans = []
    for src, size, tile in ar.AUTO_PLANS:
        g = ar.aa_geometry(src, size)
        assert g == (*ar.plan_aa(src[0], size[0]), -(-size[1] // ar.AA_TX)) and g[0] == tile, (src, size, g)
        plans.append(g[0])
    for name, size in ar.PRODUCTION:
        src = ar.SOURCES[name]
        assert ar.aa_geometry(src, size) == (*ar.plan_aa(src[0], size[0]), -(-size[1] // ar.AA_TX)), (name, size)
    assert ar.aa_geometry(*ar.SLICED)[0] == 8
    print(f"\n[aa plans] automatic {plans}; production " +
          ", ".join(f"{n} {s}: {ar.aa_geometry(ar.SOURCES[n], s)[0]}" for n, s in ar.PRODUCTION))
    assert sorted(set(plans)) == [1, 2, 4, 8, 16, 32]
    with pytest.raises(RuntimeError, match="downscale too steep"):
        ar.aa_geometry(*ar.REFUSED)
    for src, size in (ar.FORCED, ar.STEEP):
        fitted = []
        for t in range(1, 33):
            aa_rows(t)
            want = ar.plan_aa(src[0], size[0], t)
            if want is None:
                with pytest.raises(RuntimeError, match="vqa_debug_set_preprocess_aa_rows"):
                    ar.aa_geometry(src, size)
            else:
                assert ar.aa_geometry(src, size) == (*want, -(-size[1] // ar.AA_TX))
                fitted.append(t)
        aa_rows(0)
        assert ar.aa_geometry(src, size)[0] == ar.plan_aa(src[0], size[0])[0]
        assert fitted == (list(range(1, 33)) if (src, size) == ar.FORCED else list(range(1, 30))), (src, size, fitted)


def test_debug_entry_point_arguments(aa_rows):
    lib = _lib.load()
    aa_rows(5)
    for bad in (-1, 33, 1 << 20):
        assert lib.vqa_debug_set_preprocess_aa_rows(bad) != 0
        assert "tile_rows" in _lib.last_error(None)
    assert ar.aa_geometry(*ar.FORCED)[0] == 5                       # a rejected value leaves the override in force
    aa_rows(0)
    (fh, _, th), (fv, _, tv) = ar._aa_bicubic_taps(250, 140), ar._aa_bicubic_taps(168, 112)
    ip = lambda t: C.cast(t.data_ptr(), C.POINTER(C.c_int32))
    g = (C.c_int32 * 3)()
    assert lib.vqa_debug_preprocess_aa_geometry(168, 250, 112, 140, ip(fh), th, ip(fv), tv, 14, 2, g) == 0
    assert tuple(g) == ar.aa_geometry(*ar.FORCED)
    calls = [((168, 250, 112, 140, ip(fh), th, ip(fv), tv, 14, 2, None), "bad argument"),
             ((168, 250, 112, 140, None, th, ip(fv), tv, 14, 2, g), "bad argument"),
             ((168, 250, 112, 140, ip(fh), th, None, tv, 14, 2, g), "bad argument"),
             ((168, 250, 112, 140, ip(fh), th, ip(fv), tv, 0, 2, g), "bad argument"),
             ((168, 250, 112, 140, ip(fh), th, ip(fv), tv, 14, 0, g), "bad argument"),
             ((168, 250, 112, 140, ip(fh), th, ip(fv), tv, 14, 3, g), "multiple of patch"),
             ((168, 250, 112, 140, ip(fh), 251, ip(fv), tv, 14, 2, g), "bad sizes"),
             ((168, 250, 112, 140, ip(fh), th, ip(fv), 0, 14, 2, g), "bad sizes"),
             ((100, 250, 112, 140, ip(fh), th, ip(fv), tv, 14, 2, g), "vertical windows")]
    for args, msg in calls:
        assert lib.vqa_debug_preprocess_aa_geometry(*args) != 0, args
        assert msg in _lib.last_error(None), (args, _lib.last_error(None))

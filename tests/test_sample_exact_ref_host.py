"""The exact restatement of the sampled selection (tests/sample_exact_ref.py) on the CPU: it agrees with the fp64 warpers of
tests/sample_ref.py outside a band derived from the mass arithmetic, it gives the known answers of hand-built rows at the top-p cut, and its
top-p threshold is HF's fp32(1 - top_p) of the caller's double."""
import numpy as np
import pytest
import torch

import sample_exact_ref as ex
import sample_ref as sr

EXPF_ULPS = 2                     # CUDA C Programming Guide: expf's maximum error, full range


def fp64_masses(x: np.ndarray) -> np.ndarray:
    """The masses the kernel forms, with the fp32 expf replaced by fp64 exp rounded to fp32: mass_of_exp(fp32(exp(fp32(x - max))))."""
    with np.errstate(over="ignore"):         # -FLT_MAX - FLT_MAX is -inf, as on the device
        d = (x - x.max()).astype(np.float32).astype(np.float64)
    return ex.mass_of_exp(np.exp(d).astype(np.float32))


def mass_band(V: int) -> float:
    """How far a kept-set boundary may sit from 1 - top_p in fp64 cumulative probability and still differ between the restatement and the
    fp64 warpers. Each mass carries a relative error of at most 2^-24 (the fp32 product, rounded once) plus expf's 2 ulp (2 * 2^-23); a
    ratio of two sums of such terms is off by twice that. Quantising to 2^-40 units moves each term by at most half a unit, and a term
    below 2^-41 becomes 0: V * 2^-41 of probability in all (the maximum's mass is 2^40 units, so the total is at least that). Truncating
    the double product to tg moves the cut by less than one unit, 2^-40."""
    rel = 2.0 ** -24 + EXPF_ULPS * 2.0 ** -23
    return 2 * rel + V * 2.0 ** -41 + 2.0 ** -40


def rows(V: int, gen: torch.Generator) -> torch.Tensor:
    """bf16 rows: Gaussian, heavy-tailed, flat on a 1/8 grid (huge tie groups), all negative, and saturating +-inf / NaN logits."""
    g = torch.randn(V, generator=gen) * 3
    h = torch.randn(V, generator=gen) * 1.5
    h[torch.randint(0, V, (min(V, 40),), generator=gen)] += torch.rand(min(V, 40), generator=gen) * 12
    f = torch.randint(-16, 9, (V,), generator=gen).float() / 8
    n = -(torch.rand(V, generator=gen) * 6 + 0.5)
    s = torch.randn(V, generator=gen)
    s[torch.randint(0, V, (8,), generator=gen)] = float("inf")
    s[torch.randint(0, V, (8,), generator=gen)] = -float("inf")
    s[torch.randint(0, V, (8,), generator=gen)] = float("nan")
    return torch.stack([g, h, f, n, s]).bfloat16()


@pytest.mark.parametrize("V", [1000, 32128, 152064])
def test_restatement_agrees_with_fp64_warpers_outside_the_mass_band(V):
    gen = torch.Generator().manual_seed(V + 1)
    band = mass_band(V)
    outside = 0
    for T in (0.7, 1.0):
        x = sr.processed_scores(rows(V, gen), None, 1.0, T)
        for b in range(x.shape[0]):
            m = fp64_masses(x[b])
            v = np.zeros(V, np.float32)
            for k in (0, 1, 50, V - 1, V + 5):
                for p in (1e-8, 0.3, 0.9, 0.95, 0.99, 1.0):
                    got = ex.select_row(x[b], m, v, k, p)
                    want, cum, thr = sr.warp_row(x[b], k, p)
                    assert thr == float(ex.threshold(p))
                    diff = np.nonzero(got.kept != want)[0]
                    assert np.all(np.abs(cum[diff] - thr) <= band), (V, T, b, k, p, diff[:5], cum[diff][:5] - thr, band)
                    outside += V - len(diff)
    assert outside > 0


def hand_row(x, mass):
    return np.asarray(x, np.float32), np.asarray(mass, np.uint64)


def top_p_for(thr: float) -> float:
    """The double top_p whose fp32(1 - top_p) is the fp32 value thr (1 - thr is exact in double for thr >= 2^-29)."""
    t = np.float32(thr)
    p = 1.0 - float(t)
    assert ex.threshold(p) == t
    return p


# ids:                0    1    2    3    4    5       (ascending (score, id): 5, 4, 3, 1, 2, 0; running sums 1, 2, 4, 8, 12, 20)
HAND_X = [0.0, -1.0, -1.0, -2.0, -3.0, -3.5]
HAND_M = [8, 4, 4, 2, 1, 1]


@pytest.mark.parametrize("tg,kept,drop", [
    (4, [0, 1, 2], 0),                 # tg equals the running sum through id 3: ids 5, 4, 3 go
    (3, [0, 1, 2, 3], 0),              # tg one below it: id 3 completes the sum past tg and stays
    (5, [0, 1, 2], 0),                 # one above: the cut moves into the group of ids 1 and 2, rest 1 < q 4
    (8, [0, 2], 1),                    # a running sum inside the group (ids 1, 2 at q 4): the lower id goes
    (7, [0, 1, 2], 0),                 # one below it
    (9, [0, 2], 1),                    # one above it
    (12, [0], 0),                      # the running sum through the whole group
])
def test_hand_built_cut(tg, kept, drop):
    x, m = hand_row(HAND_X, HAND_M)
    sel = ex.select_row(x, m, np.zeros(6, np.float32), 0, top_p_for((tg + 0.5) / 20))
    assert (sel.total, sel.tg, sel.drop) == (20, tg, drop)
    assert np.nonzero(sel.kept)[0].tolist() == kept
    assert sel.tg_equals_cumsum == (tg in (1, 2, 4, 8, 12, 20))


def test_hand_built_clamp_and_max_tie_group():
    # fp32(1 - 1e-8) is 1: tg = total is clamped to total - 1, and only the last unit's id stays -- the highest id of the maximum's group
    x, m = hand_row([0.0, 0.0, 0.0, -1.0], [8, 8, 8, 1])
    assert ex.threshold(1e-8) == np.float32(1.0)
    sel = ex.select_row(x, m, np.zeros(4, np.float32), 0, 1e-8)
    assert sel.clamped and sel.tg == 24 and sel.drop == 2 and np.nonzero(sel.kept)[0].tolist() == [2]
    # a cut inside the maximum's own group: tg 9 = id 3's 1 + one member of 8 -> the group's lowest id goes
    sel = ex.select_row(x, m, np.zeros(4, np.float32), 0, top_p_for(9 / 25 + 1e-6))
    assert sel.tg == 9 and sel.drop == 1 and np.nonzero(sel.kept)[0].tolist() == [1, 2]
    # top-k first: k = 2 inside the group of three keeps all three (ties included), and the total is theirs alone
    sel = ex.select_row(x, m, np.zeros(4, np.float32), 2, top_p_for(0.5))
    assert sel.total == 24 and sel.tg == 12 and sel.drop == 1 and np.nonzero(sel.kept)[0].tolist() == [1, 2]


def test_hand_built_zero_mass_ids_go_at_any_cut():
    # ids 1 and 3 have mass 0: their running sum 0 is <= any tg, so they go even at tg = 0 (fp32(1 - top_p) * total < 1)
    x, m = hand_row([0.0, -40.0, -1.0, -45.0], [2 ** 40, 0, 2 ** 38, 0])
    sel = ex.select_row(x, m, np.zeros(4, np.float32), 0, 1.0 - 2.0 ** -50)
    assert sel.tg == 0 and sel.zero_mass_kept == 2 and np.nonzero(sel.kept)[0].tolist() == [0, 2]
    sel = ex.select_row(x, m, np.zeros(4, np.float32), 0, 1.0)
    assert np.nonzero(sel.kept)[0].tolist() == [0, 1, 2, 3]


def test_hand_built_draw_ties_to_the_lowest_id():
    x, m = hand_row([0.0, 0.0, 0.0, -1.0], [8, 8, 8, 1])
    v = np.array([1.0, 3.0, 3.0, 5.0], np.float32)
    assert ex.select_row(x, m, v, 0, 1.0).token == 3
    assert ex.select_row(x, m, v, 3, 1.0).token == 1
    assert ex.select_row(x, m, v, 3, 1.0, mutation="argmax_ties_high").token == 2
    v = np.array([-np.inf, -np.inf, 0.0, -np.inf], np.float32)
    assert ex.select_row(x, m, v, 0, 1.0).token == 2


@pytest.mark.parametrize("p,ulps", [(0.9, 3), (0.95, 3), (0.99, -10), (0.8, -1), (0.6, -1)])
def test_threshold_is_hf_fp32_of_the_double(p, ulps):
    """HF's TopPLogitsWarper compares its fp32 cumulative probabilities with the Python float 1 - top_p, which torch rounds to fp32 once.
    Rounding top_p to fp32 first (a float struct field) moves the threshold by these many fp32 ulps."""
    thr = ex.threshold(p)
    assert thr == np.float32(1.0 - p)
    old = ex.threshold(p, mutation="float_top_p")
    assert int(old.view(np.int32)) - int(thr.view(np.int32)) == ulps
    # HF's TopPLogitsWarper drops an id when its fp32 cumulative probability is <= 1 - top_p, a Python float against an fp32 tensor:
    # torch compares in fp32, so of thr and the next fp32 value up, the first goes and the second stays
    up = np.nextafter(thr, np.float32(1))
    assert (torch.tensor([thr, up]) <= (1 - p)).tolist() == [True, False]


def test_order_key_and_mass_quantisation():
    xs = np.array([-np.finfo(np.float32).max, -1.5, -1e-45, 0.0, 1e-45, 2.0, np.finfo(np.float32).max], np.float32)
    k = ex.order_key(xs)
    assert np.all(np.diff(k.astype(np.int64)) > 0)
    assert ex.order_key(np.float32(0.0)) == np.uint32(0x80000000)
    assert ex.mass_of_exp(np.float32(1.0)) == 2 ** 40
    assert ex.mass_of_exp(np.float32(2.0 ** -41)) == 1 and ex.mass_of_exp(np.float32(2.0 ** -42)) == 0
    # above 2^24 units the + 0.5 rounds away in fp32: the mass is the fp32 product itself
    y = np.float32(1.0 + 2.0 ** -23) * np.float32(2.0 ** -10)
    assert ex.mass_of_exp(y) == int(float(y) * 2 ** 40)


def test_philox_mutations_change_the_bits():
    b = ex.philox_bits(2 ** 63 - 1, 3, 4099)
    assert np.array_equal(b[:8], sr.philox4x32_10(np.array([[0, 3, 0, 0], [1, 3, 0, 0]], np.uint32), (2 ** 32 - 1, 2 ** 31 - 1)).reshape(-1))
    for mut in ("philox_id_step_swapped", "lanes_reversed"):
        assert not np.array_equal(b, ex.philox_bits(2 ** 63 - 1, 3, 4099, mut))
    e = ex.gumbel_e_f64(b)
    assert np.allclose(-np.log(e), sr.gumbel(2 ** 63 - 1, 3, 4099), rtol=0, atol=1e-12)

"""Sampled token selection (sample_select_kernel) bit for bit on a real H100: the kept set and the drawn token of every fixture row equal
the exact restatement of tests/sample_exact_ref.py, built from the per-id terms vqa_debug_sample_terms computes with the kernel's own
device functions, with no band and no near-tie exception; the state after each launch is SelectState's. The terms themselves are checked
against independent references, within the CUDA C Programming Guide's documented maximum errors of expf (2 ulp), logf and log1pf (1 ulp),
the only tolerances here. The fixtures reach every branch (radix passes, drop values, clamp, exact cut, thread-range boundaries,
threshold window), which the host asserts, and each deliberately wrong variant of the restatement disagrees with the kernel somewhere."""
from collections import defaultdict

import numpy as np
import pytest
import torch

import sample_exact_ref as ex
import sample_ref as sr
from test_gpu_decode_kernels import SelectState, assert_same_state

pytestmark = pytest.mark.gpu

PEN = 1.3
SEEDS = [0, 2 ** 32 - 1, 2 ** 32, 2 ** 63 - 1]
SENT = 0x5A5A5A5A                 # kept words of a finished row must come back as this
DEV = "cuda"


def ulp(a) -> np.ndarray:
    """fp32 spacing at |a| (a rounded to fp32 first)."""
    return np.spacing(np.abs(np.asarray(a, np.float64)).astype(np.float32)).astype(np.float64)


def within_ulps(got, ref, n) -> np.ndarray:
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    same_inf = np.isinf(ref) & (got == ref)
    return same_inf | (np.abs(got - ref) <= n * np.maximum(ulp(got), ulp(ref)))


def check_terms(t, logits, bitmap, penalty, T, seeds, lengths):
    """The debug terms against independent references: scores and maxima exact; expf within 2 ulp of fp64 exp of the exact fp32
    x - max and each mass exactly mass_of_exp of it; the Philox bits exact; e within 1 ulp of fp64 -log u; v within 1 ulp of log e plus
    one rounding of its fp64 value."""
    with np.errstate(over="ignore", invalid="ignore"):     # -FLT_MAX - FLT_MAX is -inf and -inf - log e stays -inf, as on the device
        x = sr.processed_scores(logits, bitmap if penalty != 1.0 else None, penalty, T)
        assert np.array_equal(t["score"].view(np.uint32), x.view(np.uint32))
        mx = x.max(1)
        assert np.array_equal(t["row_max"].view(np.uint32), mx.view(np.uint32))
        d = (x - mx[:, None]).astype(np.float32)
        assert within_ulps(t["ex"], np.exp(d.astype(np.float64)), 2).all()
        assert np.array_equal(t["mass"], ex.mass_of_exp(t["ex"]))
        for b in range(x.shape[0]):
            assert np.array_equal(t["bits"][b], ex.philox_bits(int(seeds[b]), int(lengths[b]), x.shape[1]))
        e_ref = ex.gumbel_e_f64(t["bits"])
        assert within_ulps(t["e"], e_ref, 1).all()
        loge = np.log(t["e"].astype(np.float64))
        v_ref = d.astype(np.float64) - loge
        v = t["v"].astype(np.float64)
        ok = (np.isinf(v_ref) & (v == v_ref)) | (np.abs(v - v_ref) <= ulp(loge) + 0.5 * np.maximum(ulp(v), ulp(v_ref)))
        assert ok.all()
    return x, mx


class Recorder:
    """Per fixture group: the rows checked and their Selections; per row what the mutation check needs."""

    def __init__(self):
        self.sel = defaultdict(list)
        self.rows = []

    def report(self, group):
        s = self.sel[group]
        kp = sorted({x.k_pass for x in s if x.k_pass is not None})
        drops = sorted({x.drop for x in s if x.key_p})
        print(f"\n[sample exact {group}] {len(s)} rows; top-k passes {kp}; drops {drops[:12]}{' ...' if len(drops) > 12 else ''}")


def run(ops, rec, group, logits, T, k, p, bitmap=None, penalty=1.0, seeds=None, lengths=None, done=None, eos=(), first_pos=None,
        max_new=64):
    """One vqa_debug_sample_terms and one vqa_op_sample_select launch on the same inputs; the kernel's kept bitmap, token and state
    must equal the restatement's. Returns the Selections of the unfinished rows."""
    B, V = logits.shape
    seeds = [SEEDS[b % 4] for b in range(B)] if seeds is None else seeds
    lengths = torch.zeros(B, dtype=torch.int32) if lengths is None else torch.as_tensor(lengths, dtype=torch.int32)
    done = torch.zeros(B, dtype=torch.int32) if done is None else torch.as_tensor(done, dtype=torch.int32)
    t = ex.device_terms(logits, bitmap, penalty, seeds, T, lengths, k, p)
    x, mx = check_terms(t, logits, bitmap, penalty, T, seeds, lengths)
    ref = SelectState(B, V, max_new, bitmap, first_pos, lengths, done)
    dev = ref.to_device()
    words = (V + 31) // 32
    kept = torch.full((B, words), SENT, dtype=torch.int32, device=DEV)
    eos_dev = torch.tensor(list(eos), dtype=torch.int32, device=DEV) if eos else None
    ops.sample_select(logits.cuda(), torch.tensor(seeds, dtype=torch.int64, device=DEV), T, k, p, dev.tokens, dev.lengths, dev.done,
                      dev.n_done, dev.all_done, dev.next_ids, eos_ids=eos_dev, pen_bitmap=dev.bitmap, repetition_penalty=penalty,
                      first_pos=dev.first_pos, pos3=dev.pos3, kept=kept)
    torch.cuda.synchronize()
    got_kept = kept.cpu().numpy().view(np.uint32)
    toks, sels = [], []
    for b in range(B):
        if done[b]:
            assert (got_kept[b] == np.uint32(SENT)).all(), (group, b)        # a finished row's kept row is not written
            toks.append(-1)
            continue
        s = ex.select_row(x[b], t["mass"][b], t["v"][b], k, p)
        want = ex.pack_bits(s.kept[None])[0]
        assert np.array_equal(got_kept[b], want), (group, b, V, T, k, p, np.nonzero(got_kept[b] != want)[0][:8])
        toks.append(s.token)
        sels.append(s)
        rec.sel[group].append(s)
        rec.rows.append(dict(x=x[b], mass=t["mass"][b], v=t["v"][b], mx=mx[b], bits=t["bits"][b], k=k, p=p, seed=int(seeds[b]),
                             step=int(lengths[b]), kept=s.kept, token=s.token))
    ex.expected_state(ref, toks, eos)
    assert_same_state(dev, ref, (group, V, T, k, p))
    return sels, t


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def rec():
    return Recorder()


def bitmap_of(bits: torch.Tensor) -> torch.Tensor:
    """bool [B, V] -> int32 words [B, ceil(V / 32)]."""
    B, V = bits.shape
    words = -(-V // 32)
    pad = torch.zeros(B, words * 32, dtype=torch.bool)
    pad[:, :V] = bits
    packed = (pad.view(B, words, 32).long() << torch.arange(32)).sum(-1)
    return torch.where(packed >= 1 << 31, packed - (1 << 32), packed).to(torch.int32)


def mixed_rows(V, gen):
    """Gaussian, flat on a 1/8 grid (tie groups), heavy-tailed, all negative."""
    g = torch.randn(V, generator=gen) * 3
    f = torch.randint(-16, 9, (V,), generator=gen).float() / 8
    h = torch.randn(V, generator=gen) * 1.5
    h[torch.randint(0, V, (min(V, 40),), generator=gen)] += torch.rand(min(V, 40), generator=gen) * 12
    n = -(torch.rand(V, generator=gen) * 6 + 0.5)
    return torch.stack([g, f, h, n]).bfloat16()


# ------------------------------------------------------------------------------------------------ vocabularies
@pytest.mark.parametrize("V", [1, 3, 5, 1000, 1001, 8191, 8192, 8193, 32128, 151936, 152064])
def test_vocabularies(ops, rec, V):
    """Below one Philox group and below one thread per id, around the 1024 x 8 stride of the scan, the T5 and Qwen2.5-VL-3B / 7B
    vocabularies, and V % 32 != 0 (kept bits past V stay zero); a penalty on two rows, steps > 0."""
    gen = torch.Generator().manual_seed(V)
    logits = mixed_rows(V, gen)
    bitmap = bitmap_of(torch.rand(4, V, generator=gen) < 0.3)
    for T, k, p in ((0.7, 50, 0.9), (1.0, 0, 0.95), (1.0, 3, 0.5)):
        run(ops, rec, "vocab", logits, T, k, p, bitmap, PEN, lengths=[0, 1, 5, 9])
    rec.report("vocab")


# ------------------------------------------------------------------------------------------------ radix passes
def pass2_pair():
    """A bf16 logit a whose penalised fp32 score s = a / PEN shares the top 22 bits of its key with the bf16 value b of s's top 16 bits,
    b != s: an unpenalised id at b and a penalised one at a differ only in the 10-bit pass. (A negative logit is multiplied by the
    penalty, and no bf16 product with fp32(1.3) has those six bits clear.)"""
    pen = np.float32(PEN)
    for i in range(0x3F80, 0x4200):          # bf16 1.0 ... 32.0
        a = np.array([i << 16], np.uint32).view(np.float32)[0]
        u = np.array([np.float32(a / pen)], np.float32).view(np.uint32)[0]
        if (u >> 10) & 0x3F == 0 and u & 0x3FF:
            return float(a), float(np.array([u & 0xFFFF0000], np.uint32).view(np.float32)[0])
    raise AssertionError("no pair")


def radix_rows(V, gen):
    """Rows whose top-k thresholds the three radix passes decide: 0 a unique maximum far above the rest (pass 0 at k = 1); 1 two maxima
    one bf16 ulp apart (pass 1); 2 a penalised-unpenalised pair sharing its top 22 key bits (pass 2); 3 all negative (complemented keys)
    with two maxima one ulp apart; 4 mixed signs; 5 -0 next to +0 above negatives; 6 +-inf and NaN logits that saturate; 7 flat (k
    inside tie groups). Returns (logits, penalty bits)."""
    r = torch.randn(8, V, generator=gen).clamp(-3, 3)
    bits = torch.rand(8, V, generator=gen) < 0.2
    r[0, 17] = 10.0
    r[1, 40], r[1, 41] = 4.0, 4.03125
    bits[1, 40:42] = False
    a, b = pass2_pair()
    r[2] = r[2].clamp(max=min(a / PEN, b) - 1)
    r[2, 100], r[2, V - 3] = a, b
    bits[2, 100], bits[2, V - 3] = True, False
    r[3] = -(r[3].abs() + 5)
    r[3, 7], r[3, 900] = -4.0, -4.03125
    bits[3, 7], bits[3, 900] = False, False
    r[4] = torch.randn(V, generator=gen) * 4
    r[5] = -(r[5].abs() + 0.5)
    r[5, 3], r[5, 600] = -0.0, 0.0
    bits[5, 3] = True
    r[6, 5], r[6, 6], r[6, 9] = float("inf"), float("inf"), float("nan")
    r[6, 11], r[6, 12] = -float("inf"), float("nan")
    r[7] = torch.randint(-8, 5, (V,), generator=gen).float() / 4
    return r.bfloat16(), bits


@pytest.mark.parametrize("V", [1001, 32128])
def test_radix_passes_and_top_k_edges(ops, rec, V):
    """k = 1, 2, inside a tie group, V - 1, V and V + 5 on rows built so the 11-, 11- and 10-bit passes each decide a threshold; at
    T 1e-38 nearly every score saturates to +-FLT_MAX."""
    gen = torch.Generator().manual_seed(V + 7)
    logits, bits = radix_rows(V, gen)
    bitmap = bitmap_of(bits)
    flat = sr.processed_scores(logits, bitmap, PEN, 1.0)[7]
    k_tie = int((flat >= np.float32(0.25)).sum()) - 3          # lands inside the group at 0.25 (or the next below)
    for T in (1.0, 1e-38):
        for k in (1, 2, k_tie, V - 1, V, V + 5):
            for p in (1.0, 0.9):
                run(ops, rec, "radix", logits, T, k, p, bitmap, PEN, lengths=[3] * 8)
    passes = {s.k_pass for s in rec.sel["radix"] if s.k_pass is not None}
    assert passes == {0, 1, 2}, passes
    rec.report("radix")


# ------------------------------------------------------------------------------------------------ top-p cut
def top_p_for_target(total: int, lo: int, hi: int) -> float:
    """A double top_p whose cut target tg = floor(fp32(1 - top_p) * total) lies in [lo, hi): the fp32 threshold nearest the middle, then
    1 - it, which is exact in double and rounds back to it."""
    t = np.float32((lo + hi) / 2 / total)
    for _ in range(64):
        tg = ex.cut_target(t, total)
        if lo <= tg < hi:
            p = 1.0 - float(t)
            assert ex.threshold(p) == t
            return p
        t = np.nextafter(t, np.float32(1 if tg < lo else 0))
    raise AssertionError((total, lo, hi))


def group_row(V, gen, G, stride):
    """One maximum at 2.0; a tie group of G ids at 0.0 every `stride` ids from id 11 (over many threads' id ranges); V / 30 ids at -2.0;
    V / 10 ids at -20.0, whose masses of some 300 units make running sums fine enough for an exact cut target; the rest at -40.0 (mass 0)."""
    r = torch.full((V,), -40.0)
    r[torch.randint(0, V, (V // 10,), generator=gen)] = -20.0
    r[torch.randint(0, V, (V // 30,), generator=gen)] = -2.0
    r[11:11 + G * stride:stride] = 0.0
    r[V - 2] = 2.0
    return r.bfloat16()


def exact_target_top_p(total: int, want: int):
    """A double top_p with floor(fp32(1 - top_p) * total) == want exactly, or None. Needs fp32 thresholds spaced by less than one unit
    of total and 1 - threshold exact in double (threshold >= 2^-29)."""
    t = np.float32(want / total)
    for _ in range(64):
        tg = ex.cut_target(t, total)
        if tg == want:
            p = 1.0 - float(t)
            return p if ex.threshold(p) == t else None
        t = np.nextafter(t, np.float32(1 if tg < want else 0))
    return None


def test_top_p_cut_drop_values_clamp_and_exact_target(ops, rec):
    """drop 0; drop > 0 in a tie group of 5000 ids spread over some 1000 threads' id ranges, with the dropped count ending exactly at a
    thread-range boundary (a member at the first id of the range) and at the group's last member; the clamp (top_p 1e-8); tg exactly equal
    to a running sum, and tg - 1 and tg + 1; zero-mass ids; top-k changing the total. The thresholds are chosen from the device masses."""
    V, G, stride = 152064, 5000, 29
    gen = torch.Generator().manual_seed(11)
    row = group_row(V, gen, G, stride)[None]
    t = ex.device_terms(row, None, 1.0, [5], 1.0, [2])
    x, m = t["score"][0], t["mass"][0]
    total = int(m.sum())
    order = np.lexsort((np.arange(V), ex.order_key(x)))
    csum = np.cumsum(m[order])
    gid = np.nonzero(x == np.float32(0.0))[0]
    assert len(gid) == G
    q = int(m[gid[0]])
    below = int(csum[np.nonzero(order == gid[0])[0][0]]) - q
    per = -(-V // ex.SELECT_THREADS)
    t0 = next(tt for tt in range(400, ex.SELECT_THREADS) if (tt * per - 11) % stride == 0)
    d_boundary = int((gid < t0 * per).sum())                # member d_boundary sits at id t0 * per, the first id of thread t0's range
    assert gid[d_boundary] == t0 * per
    for name, D in (("drop 0", 0), ("drop 1", 1), ("thread-range boundary", d_boundary), ("last member", G - 1)):
        p = top_p_for_target(total, below + D * q + 1, below + (D + 1) * q)
        (s,), _ = run(ops, rec, "cut", row, 1.0, 0, p, seeds=[5], lengths=[2])
        assert s.drop == D and len(s.group) == G, (name, s.drop, D)
    (s,), _ = run(ops, rec, "cut", row, 1.0, 0, 1e-8, seeds=[5], lengths=[2])
    assert s.clamped and s.kept.sum() == 1 and s.zero_mass_kept > 0
    # tg equal to a member-level running sum C of the -20.0 group, and C - 1, C + 1
    for j in range(int(np.searchsorted(csum, np.uint64(total >> 29))) + 1, len(csum) - 1):
        C = int(csum[j])
        found = [exact_target_top_p(total, w) for w in (C, C - 1, C + 1)]
        if csum[j + 1] != csum[j] and None not in found:
            break
    else:
        raise AssertionError("no exact running-sum target")
    for p in found:
        run(ops, rec, "cut", row, 1.0, 0, p, seeds=[5], lengths=[2])
    exact = rec.sel["cut"][-3]
    assert exact.tg == C and exact.tg_equals_cumsum and exact.drop > 0
    # top-k and top-p together: top-k removes ids with mass, so the total the cut is taken of changes
    (s,), _ = run(ops, rec, "cut", row, 1.0, 2000, 0.9, seeds=[5], lengths=[2])
    assert s.total < total
    rec.report("cut")
    print(f"    thread-range boundary: thread {t0}, member {d_boundary}; exact tg {C} (drop {exact.drop})")


# ------------------------------------------------------------------------------------------------ the threshold window
def window_rows(V, gen, p, n):
    """n rows of one maximum at 0 and V - 1 ids near the score whose total mass puts the cut at 1 - p among them: there the ascending
    running sum steps by the smallest mass that can still reach 1 - p, so some row is likely to have a step inside the few-ulp window."""
    thr = 1.0 - p
    d = float(np.log(1.5 * thr / (1 - thr) / (V - 1)))
    r = d + (torch.rand(n, V, generator=gen) - 0.5)
    r[:, 0] = 0.0
    return r.bfloat16()


@pytest.mark.parametrize("p", [0.9, 0.95, 0.99])
def test_threshold_window_separates_hf_from_the_float_round_trip(ops, rec, p):
    """A row with an ascending running sum strictly between the cut of HF's threshold fp32(1 - top_p) and that of fp32(1 - fp32(top_p)),
    chosen from candidate rows by their device masses: the two thresholds' kept sets differ on it, and the kernel's is HF's."""
    V = 152064
    gen = torch.Generator().manual_seed(int(p * 1000))
    for chunk in range(6):
        rows = window_rows(V, gen, p, 48)
        t = ex.device_terms(rows, None, 1.0, list(range(48)), 1.0, [0] * 48)
        for b in range(48):
            a = ex.select_row(t["score"][b], t["mass"][b], t["v"][b], 0, p)
            o = ex.select_row(t["score"][b], t["mass"][b], t["v"][b], 0, p, mutation="float_top_p")
            if not np.array_equal(a.kept, o.kept):
                (s,), _ = run(ops, rec, "window", rows[b:b + 1], 1.0, 0, p, seeds=[b], lengths=[0])
                assert np.array_equal(s.kept, a.kept)
                print(f"\n[sample exact window] top_p {p}: candidate row {chunk * 48 + b}: kept sets differ in "
                      f"{int((a.kept != o.kept).sum())} id(s)")
                return
    raise AssertionError(f"no candidate row separates the thresholds at top_p {p}")


# ------------------------------------------------------------------------------------------------ batch, state, temperatures
@pytest.mark.parametrize("T", [1e-38, 0.7, 1.0, 100.0])
@pytest.mark.parametrize("penalised", [True, False])
def test_batch_state_and_temperatures(ops, rec, T, penalised):
    """Six rows of different kinds in one launch at steps 0 .. 7 with positions, an EOS id and max_new 8: two rows are finished (state
    untouched, kept row not written), one reaches max_new. Without a penalty is how the T5 step calls the kernel."""
    V, B = 32128, 6
    gen = torch.Generator().manual_seed(int(T * 10) + penalised)
    logits = torch.cat([mixed_rows(V, gen), mixed_rows(V, gen)[:2]])
    bitmap = bitmap_of(torch.rand(B, V, generator=gen) < 0.25) if penalised else None
    first_pos = torch.arange(B, dtype=torch.int32) * 13 + 30
    for k, p in ((50, 0.9), (0, 0.99), (0, 1.0)):
        run(ops, rec, "batch", logits, T, k, p, bitmap, PEN if penalised else 1.0, seeds=SEEDS + [7, 8], lengths=[0, 3, 7, 1, 2, 5],
            done=[0, 0, 0, 1, 0, 1], eos=(17, 1999), first_pos=first_pos, max_new=8)
    rec.report("batch")


def test_draw_tie_to_the_lowest_id(ops, rec):
    """A constant row whose two largest Philox uniforms are equal (the seed is searched on the host): the two ids' perturbed values tie
    exactly, and the lower id is drawn."""
    V = 152064
    for seed in range(20000):
        m = ex.philox_bits(seed, 1, V) >> np.uint32(8)
        top = np.sort(m)[-2:]
        if top[0] == top[1]:
            break
    else:
        raise AssertionError("no tying seed")
    row = torch.zeros(1, V).bfloat16()
    (s,), t = run(ops, rec, "tie", row, 1.0, 0, 1.0, seeds=[seed], lengths=[1])
    ids = np.nonzero(m == top[1])[0]
    assert s.token == ids[0] and t["v"][0][ids[0]] == t["v"][0][ids[1]]
    print(f"\n[sample exact tie] seed {seed}: ids {ids.tolist()} tie, token {s.token}")


# ------------------------------------------------------------------------------------------------ coverage and mutations
def test_coverage_and_mutations(rec):
    """Runs last (pytest keeps file order): the fixtures above reached every branch, and each deliberately wrong restatement disagrees
    with the kernel on at least one of them. The Philox mutations recompute the perturbed values in fp64 from their own bits, and count
    only rows where the fp64 values of the right bits still give the kernel's token."""
    sels = [s for g in rec.sel.values() for s in g]
    if not sels:
        pytest.skip("the fixture tests did not run")
    assert {s.k_pass for s in sels if s.k_pass is not None} == {0, 1, 2}
    drops = {s.drop for s in sels if s.key_p}
    assert 0 in drops and any(d > 0 and len(s.group) >= 1000 for s in sels for d in [s.drop])
    assert any(s.clamped for s in sels) and any(s.tg_equals_cumsum for s in sels) and any(s.zero_mass_kept for s in sels)
    assert rec.sel["window"], "threshold window"
    caught = {}
    for mut in ex.MUTATIONS:
        n = 0
        for r in rec.rows:
            if mut in ("philox_id_step_swapped", "lanes_reversed"):
                right = ex.select_row(r["x"], r["mass"], ex.perturbed_f64(r["x"], r["mx"], r["bits"]), r["k"], r["p"])
                if right.token != r["token"]:
                    continue
                wrong = ex.select_row(r["x"], r["mass"], ex.perturbed_f64(r["x"], r["mx"], ex.philox_bits(r["seed"], r["step"], len(r["x"]), mut)),
                                      r["k"], r["p"])
            else:
                wrong = ex.select_row(r["x"], r["mass"], r["v"], r["k"], r["p"], mutation=mut)
            n += wrong.token != r["token"] or not np.array_equal(wrong.kept, r["kept"])
        caught[mut] = n
    print(f"\n[sample exact mutations] rows disagreeing with the kernel: {caught}")
    assert all(n > 0 for n in caught.values()), caught

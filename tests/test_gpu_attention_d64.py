"""Head-dim-64 attention (attn64_ws_kernel: persistent, warp-specialised, a K/V ring of 2 to 4 stages) through the C ABI.

Three kinds of checks, each in both rounding modes (round_scores: the bf16 score tensors of the reference's eager attention):
- exact selectors: inputs whose softmax is exactly one-hot, or uniform over 2 or 4 tied keys, so the output is known bit for bit;
- random inputs against an fp64 restatement under the per-element bound of attention_ref (one bf16 ulp of the output plus twice the largest
  error of the P-rounded restatement in that head); every group also shows that its fixture separates the kernel from plausible mistakes;
- invariance: the output of a (sample, head) is bit-identical whatever else the launch holds and whatever the padding rows contain.

Production shapes: the T5 encoder (S = 672, H = 64, relative-position bias, constant past distance 128) and the CLIP ViT (S = 577, H = 16,
scale 1/8). Lengths cover every last-tile width the kernel special-cases, whole padding query tiles and padding second 64-row blocks. The
long-sequence cases run the 3-stage and 2-stage rings, which the bias row forces past S = 8,304 and 12,400."""
import pytest
import torch

from attention_ref import assert_attn, attn_bound, bf16_ulp, exponent_reference, softmax_ref

pytestmark = pytest.mark.gpu

INVALID = -1

# len mod 128 = 1, 16, 17, 32, 33, 64, 65, 96, 97, 127, 0 and lengths 0 / 1. 576: the second 64-row block of the last query tile is padding;
# 640 / 256: whole 128-row query tiles are padding.
T5_LENS = [513, 528, 401, 672, 161, 576, 577, 480, 609, 639, 640, 256, 0, 1, 16, 97]
CLIP_LENS = [577, 513, 528, 529, 544, 545, 576, 480, 481, 511, 512, 0, 1, 64]
# len mod 128 = 1, 16, 17, 32, 64, 65, 127, 0. 576 / 513 leave the second 64-row block of the last query tile all padding, 512 / 640 / 1
# leave whole 128-row query tiles (both blocks) padding.
T5_LEN_PAIRS = [(672, 1), (656, 17), (576, 65), (639, 640), (513, 16), (512, 129), (192, 127)]
# 4 stages up to S = 8,304, 3 up to 12,400, 2 up to 16,496 (a bias row of 2S - 1 + 256 floats next to the ring); refused past that
RING_LENGTHS = [8304, 8305, 12400, 12401, 16496]
MAX_BIAS_LEN = 16496


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops(dev):
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


def bf16_rne(x):
    """fp64 x rounded to the nearest bf16, ties to even, in one step (a conversion through fp32 could round twice)."""
    u = bf16_ulp(x)
    return torch.round(x / u) * u


def on_grid(x):
    """Multiples of 1/4 with |x| <= 2: a q.k over 64 dims is a multiple of 1/16 with |s| <= 256, exact in fp32 whatever the summation
    order, so bf16(s) and bf16(bf16(s) + bias) are the same numbers in the kernel and in the reference."""
    return (x * 4).round().clamp(-8, 8) / 4


def saturating_table(H, S, gen, dist=128, mult=1.0):
    """T5's bias: one bf16 value per head and relative position, constant past |key - query| >= dist on each side."""
    rel = torch.arange(-(S - 1), S).clamp(-dist, dist) + dist
    return (torch.randn(H, 2 * dist + 1, generator=gen) * mult).bfloat16().float()[:, rel].contiguous()


def heads(t, B, S, H):
    """[B * S, 3 * H * 64] packed qkv -> q, k, v as [B, H, S, 64]."""
    return t.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)


def lens_tensor(lens, B, S, dev):
    return torch.tensor(lens if lens is not None else [S] * B, dtype=torch.int32, device=dev)


# ================================================================================================ fp64 restatement
def d64_ref(q, k, v, n, S, table, scale, round_scores, r0=0, mistake=None, const_from=0):
    """Attention of the query rows r0 .. r0 + len(q) of one sample: q [H, m, 64], k / v [H, S, 64], the first n keys valid. Rounding points
    of the kernel's comment above Attn64Params, P rounded at its exponent reference. `mistake` restates a plausible kernel error instead.
    Returns softmax_ref's pair."""
    dev = q.device
    s = torch.matmul(q.double(), k.double().transpose(-1, -2))
    bias = None
    if table is not None:
        i = torch.arange(r0, r0 + q.shape[-2], device=dev)[:, None]
        j = torch.arange(S, device=dev)[None, :]
        idx = ((i - j) if mistake == "bias read at query - key" else (j - i)) + S - 1
        t = table.double()
        if mistake == "constant bias from the wrong side":
            t = t.clone()
            t[:, S - 1 + const_from:] = table[:, S - 1 - const_from, None].double()
            t[:, :S - const_from] = table[:, S - 1 + const_from, None].double()
        bias = t[:, idx]
    if round_scores:
        s = bf16_rne(s)
        if bias is not None:
            s = s + bf16_rne(bias)
            if mistake != "ROUND without the rounding of score + bias":
                s = bf16_rne(s)
        s = s * scale
    elif bias is not None:
        s = (s + bias) * scale if mistake == "scale applied to the bias" else s * scale + bias
    else:
        s = s * scale
    n_keys = n + 1 if mistake == "one key past len" else n - 1 if mistake == "last valid key dropped" else n
    s[..., n_keys:] = float("-inf")
    return softmax_ref(s, v, exponent_reference(s))


def mistakes_for(n, S, table, scale, round_scores, const_from):
    m = ["last valid key dropped"] if n >= 2 else []
    if n < S:
        m.append("one key past len")
    if table is not None:
        m.append("bias read at query - key")
        if round_scores:
            m.append("ROUND without the rounding of score + bias")
        elif scale != 1.0:
            m.append("scale applied to the bias")
        if const_from > 0 and any(k0 >= const_from + 63 for k0 in range(0, n, 128)):     # some (64-row, key tile) block takes the fast path
            m.append("constant bias from the wrong side")
    return m


def check_d64(out, qkv, B, S, H, lens, table, scale, round_scores, const_from=0, discriminate=True, block=1024, what=""):
    """Every valid row of every (sample, head) within the bound, every padding row +0 bit for bit. With `discriminate`, every mistake that
    applies to some sample (mistakes_for) moves some element of the fixture by 4x the bound."""
    q, k, v = heads(qkv, B, S, H)
    got = out.view(B, S, H, 64).permute(0, 2, 1, 3)
    lens = [S] * B if lens is None else [int(x) for x in lens]
    applicable, seen = set(), set()
    for b, n in enumerate(lens):
        assert bool((got[b, :, n:].contiguous().view(torch.int16) == 0).all()), f"{what}: padding rows of sample {b} are not +0"
        for r0 in range(0, n, block):           # row blocks bound the fp64 score memory of long sequences
            r1 = min(n, r0 + block)
            ref, ref_p = d64_ref(q[b, :, r0:r1], k[b], v[b], n, S, table, scale, round_scores, r0)
            tol = assert_attn(got[b, :, r0:r1], ref, ref_p, f"{what}: sample {b} (len {n}) rows {r0}..{r1}")
            if not discriminate:
                continue
            for m in mistakes_for(n, S, table, scale, round_scores, const_from):
                applicable.add(m)
                if m not in seen:
                    wrong = d64_ref(q[b, :, r0:r1], k[b], v[b], n, S, table, scale, round_scores, r0, m, const_from)[0]
                    if bool(((wrong - ref).abs() > 4.0 * tol).any()):
                        seen.add(m)
    missed = applicable - seen
    assert not missed, f"{what}: the fixture cannot see {sorted(missed)}"
    return applicable


def random_qkv(B, S, H, gen, dev, round_scores, amp=0.5, grid_amp=1.0):
    """Gaussian q / k / v of standard deviation amp; with round_scores q and k are Gaussians of grid_amp put on the exact-score grid
    (on_grid: scores of standard deviation ~8 at grid_amp 1, ~18 at 2), v stays Gaussian."""
    x = torch.randn(B * S, 3, H * 64, generator=gen) * amp
    if round_scores:
        x[:, :2] = on_grid(x[:, :2] * (grid_amp / amp))
    return x.reshape(B * S, 3 * H * 64).bfloat16().to(dev)


# ================================================================================================ 1. exact selectors
PAIRS = torch.tensor([(a, b) for a in range(64) for b in range(a + 1, 64)])      # 2,016 key codes: a pair of head dimensions


def code_rows(codes, mult):
    """mult * (e_a + e_b) for every code (a, b): [..., 64]."""
    x = torch.zeros(*codes.shape, 64)
    x.scatter_(-1, PAIRS[codes], mult)
    return x


def int_v(shape, gen):
    """V on a coarse dyadic grid (integers in [-64, 64] / 16): every sum of values is exact in fp32 in any order."""
    return torch.randint(-64, 65, shape, generator=gen).float() / 16


def mean_bf16(sum_v, count):
    """bf16(fp32(sum) * fp32(1 / count)): the kernel's O * (1 / l) with l the exact count of its P = 1 keys (IEEE division)."""
    inv = torch.ones_like(sum_v[..., :1], dtype=torch.float32) / count.float()[..., None]
    return (sum_v.float() * inv).bfloat16()


def key_code_fixture(lens, S, H, gen, ties):
    """Key j of (sample, head) gets the code c_j, K_j = 32 (e_a + e_b); query i targets key t(i) of a per-(sample, head) permutation of the
    valid keys, Q_i = 32 (e_a + e_b) of c_t(i). Scores are 2048 (the target), 1024 (a shared dimension) or 0, exact in bf16 and fp32: at
    scale 1/8 the runner-up sits 184.7 below the winner in the exp2 domain and its exponential is +0. With `ties`, 2 keys (tile 0 and the
    last, partial tile) and 4 keys (tile 0, a middle tile, the last tile) share one code. Padding keys are decoys with K = 64 (e_a + e_b):
    a masking slip lets one win. Returns (qkv [B * S, 3 * H * 64] on the CPU, expected output)."""
    B = len(lens)
    x = torch.zeros(B, S, 3, H, 64)
    v = int_v((B, S, H, 64), gen)
    x[:, :, 2] = v
    codes = torch.stack([torch.stack([torch.randperm(len(PAIRS), generator=gen)[:S] for _ in range(H)]) for _ in range(B)])   # [B, H, S]
    target = torch.zeros(B, H, S, dtype=torch.long)
    valid = torch.zeros(B, S, dtype=torch.bool)
    for b, n in enumerate(lens):
        valid[b, :n] = True
        for h in range(H):
            if ties and n >= 8:
                for g in ([1, n - 1], [2, n // 2, n - 3, n - 2]):
                    codes[b, h, g[1:]] = int(codes[b, h, g[0]])
            target[b, h, :n] = codes[b, h, torch.randperm(n, generator=gen)]
            target[b, h, n:] = codes[b, h, torch.randint(0, S, (S - n,), generator=gen)]       # padding queries: anything
            if n > 0:                                   # decoys carry the codes of valid keys: a query of that code scores 4096 on them
                codes[b, h, n:] = codes[b, h, torch.randint(0, n, (S - n,), generator=gen)]
    kc = code_rows(codes, 32.0)                                            # [B, H, S, 64]
    x[:, :, 1] = torch.where(valid[:, None, :, None], kc, 2.0 * kc).permute(0, 2, 1, 3)
    x[:, :, 0] = code_rows(target, 32.0).permute(0, 2, 1, 3)
    # expected: the mean of V over the valid keys that carry the query's code
    slot = (torch.arange(B * H).view(B, H, 1) * len(PAIRS) + codes)        # [B, H, S] (sample, head, code) slots
    vh = v.permute(0, 2, 1, 3).double()                                    # [B, H, S, 64]
    keep = valid[:, None, :].expand(B, H, S)
    sums = torch.zeros(B * H * len(PAIRS), 64, dtype=torch.float64).index_add_(0, slot[keep], vh[keep])
    cnt = torch.zeros(B * H * len(PAIRS), dtype=torch.long).index_add_(0, slot[keep], torch.ones(int(keep.sum()), dtype=torch.long))
    tslot = torch.arange(B * H).view(B, H, 1) * len(PAIRS) + target
    want = mean_bf16(sums[tslot], cnt[tslot])                              # [B, H, S, 64]
    want = torch.where(valid[:, None, :, None], want, torch.zeros((), dtype=torch.bfloat16))
    assert bool((cnt[tslot][valid[:, None, :].expand(B, H, S)] >= 1).all()) and int(cnt.max()) == (4 if ties else 1)
    return x.reshape(B * S, 3 * H * 64).bfloat16(), want.permute(0, 2, 1, 3).reshape(B * S, H * 64)


def assert_bits(got, want, what):
    got, want = got.cpu(), want.cpu()
    diff = got.view(torch.int16) != want.view(torch.int16)
    assert not bool(diff.any()), (f"{what}: {int(diff.sum())} of {diff.numel()} elements differ, first at {diff.nonzero()[0].tolist()}: "
                                  f"{float(got[tuple(diff.nonzero()[0])])} vs {float(want[tuple(diff.nonzero()[0])])}")


KEY_CODE_LAUNCHES = {      # name: (S, H, lengths, scale, table kind, bias_const_from)
    "clip": (577, 16, CLIP_LENS, 0.125, None, 0),
    "t5 const 128": (672, 64, T5_LENS, 1.0, "random", 128),
    "t5 const 0": (672, 64, T5_LENS, 1.0, "random", 0),
    "t5 flat table": (672, 64, T5_LENS, 1.0, "flat", 128),
}


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("launch", list(KEY_CODE_LAUNCHES))
def test_key_code_selector(dev, ops, launch, round_scores):
    """One-hot softmax through the key codes: output row i is V[t(i)] bit for bit, padding rows +0. Every score position of every key tile
    and every lane / column mapping is checked once per head, a mix-up of heads or of samples shows, and a decoy that slips through the
    mask wins. The T5 launches add a bias with |b| <= 8 (it cannot move a winner that leads by 1024), read per score or, past distance 128,
    as the block's constant; the flat table (one value per head) keeps exact ties under the bias path, the CLIP launch has them without."""
    S, H, lens, scale, kind, const_from = KEY_CODE_LAUNCHES[launch]
    gen = torch.Generator().manual_seed(100 + len(launch))
    ties = kind != "random"
    qkv, want = key_code_fixture(lens, S, H, gen, ties)
    table = None
    if kind == "random":
        table = (torch.randint(-16, 17, (H, 257), generator=gen).float() / 2)[:, torch.arange(-(S - 1), S).clamp(-128, 128) + 128].contiguous()
    elif kind == "flat":
        table = (torch.randint(-16, 17, (H, 1), generator=gen).float() / 2).expand(H, 2 * S - 1).contiguous()
    B = len(lens)
    out = ops.attention(qkv.to(dev), B, S, H, seq_lens=lens_tensor(lens, B, S, dev), bias_table=None if table is None else table.to(dev),
                        scale=scale, bias_const_from=const_from, round_scores=round_scores)
    assert_bits(out, want, launch)


def bias_shifts(const_from):
    """The selected key - query of each of 16 heads: distinct, inside (-C, C) so that the table is constant past distance C, and +-(C - 1)
    next to the cut-off (C = 128 when nothing is promised)."""
    e = (const_from or 128) - 1
    return [0, 1, -1, e, -e, 2, -2, 64, -64, 100, -100, 31, -33, 96, -97, 17]


def bias_selector_fixture(lens, S, gen, shifts):
    """Q = K = 0 on valid rows; head h's table is 0 at key - query = d_h and -1024 elsewhere, so query i selects key i + d_h when that key
    is valid (output V[i + d_h]) and otherwise every valid key equally (the mean over the first len keys). Padding keys and queries hold
    32 (e_0 + e_1), which padding query rows must not show. A key past len that slipped through the mask would join the uniform mean or
    be selected. Returns (qkv on the CPU, table, expected output)."""
    B, H = len(lens), len(shifts)
    x = torch.zeros(B, S, 3, H, 64)
    v = int_v((B, S, H, 64), gen)
    x[:, :, 2] = v
    table = torch.full((H, 2 * S - 1), -1024.0)
    d = torch.tensor(shifts)
    table[torch.arange(H), d + S - 1] = 0.0
    want = torch.zeros(B, S, H, 64, dtype=torch.bfloat16)
    for b, n in enumerate(lens):
        x[b, n:, :2, :, :2] = 32.0
        if n == 0:
            continue
        uniform = mean_bf16(v[b, :n].double().sum(0), torch.full((H,), n))          # [H, 64]
        j = torch.arange(n)[:, None] + d[None, :]                                 # [n, H] the selected key
        ok = (j >= 0) & (j < n)
        sel = v[b, j.clamp(0, n - 1), torch.arange(H)[None, :]].bfloat16()       # [n, H, 64]
        want[b, :n] = torch.where(ok[..., None], sel, uniform[None])
    return x.reshape(B * S, 3 * H * 64).bfloat16(), table, want.reshape(B * S, H * 64)


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("const_from", [128, 130, 0])
@pytest.mark.parametrize("shape", ["t5", "clip"])
def test_bias_selector(dev, ops, shape, const_from, round_scores):
    """The bias alone picks the key: pins the bias index (key - query, not query - key), the head of each bias row, the constant value on
    both sides of the fast path (d_h = +-(C - 1) sits next to its cut-off), the masking of a selected key past len, and the lazy rescale (a
    winner in a later key tile resets O and l through corr = 2^-1477 = 0). Rows with no valid selected key are the exact uniform mean.
    The nearest key - query of a (64-row, key tile) block wholly past the cut-off, k0 - (qb + 63), is 1 mod 64: C = 130 puts such a block
    at exactly C - 1, where one pair still needs its own table entry."""
    S, lens = (672, T5_LENS) if shape == "t5" else (577, CLIP_LENS)
    gen = torch.Generator().manual_seed(200 + S)
    qkv, table, want = bias_selector_fixture(lens, S, gen, bias_shifts(const_from))
    B, H = len(lens), table.shape[0]
    out = ops.attention(qkv.to(dev), B, S, H, seq_lens=lens_tensor(lens, B, S, dev), bias_table=table.to(dev), scale=1.0,
                        bias_const_from=const_from, round_scores=round_scores)
    assert_bits(out, want, f"{shape} C={const_from}")


# ================================================================================================ 2. random inputs under the bound
@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("lens_pair", T5_LEN_PAIRS)
def test_t5_shape_ragged_tails(dev, ops, lens_pair, round_scores):
    gen = torch.Generator().manual_seed(1)
    B, S, H = 2, 672, 64
    qkv = random_qkv(B, S, H, gen, dev, round_scores)
    table = saturating_table(H, S, gen).to(dev)
    lens = torch.tensor(lens_pair, device=dev, dtype=torch.int32)
    out = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=table, scale=1.0, bias_const_from=128, round_scores=round_scores)
    check_d64(out, qkv, B, S, H, lens_pair, table, 1.0, round_scores, const_from=128, what=str(lens_pair))


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("lens_pair", [None, (577, 449), (513, 65), (576, 32)])
def test_clip_shape(dev, ops, lens_pair, round_scores):
    gen = torch.Generator().manual_seed(2)
    B, S, H = 2, 577, 16
    qkv = random_qkv(B, S, H, gen, dev, round_scores, amp=1.0)
    lens = torch.tensor(lens_pair, device=dev, dtype=torch.int32) if lens_pair else None
    out = ops.attention(qkv, B, S, H, seq_lens=lens, scale=0.125, round_scores=round_scores)
    check_d64(out, qkv, B, S, H, lens_pair, None, 0.125, round_scores, what=str(lens_pair))


@pytest.mark.parametrize("round_scores", [False, True])
def test_constant_bias_fast_path_is_exact(dev, ops, round_scores):
    """A table that is constant past distance 128 gives bit-identical output whether the kernel is told so (and skips the per-score
    lookups of far tiles) or not. A table that breaks the promise does give a different output under the promise, so the comparison
    does see the fast path."""
    gen = torch.Generator().manual_seed(3)
    B, S, H = 2, 672, 8
    qkv = random_qkv(B, S, H, gen, dev, round_scores)
    lens = torch.tensor([672, 600], device=dev, dtype=torch.int32)
    table = saturating_table(H, S, gen, mult=2.0).to(dev)
    fast = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=table, scale=1.0, bias_const_from=128, round_scores=round_scores)
    slow = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=table, scale=1.0, bias_const_from=0, round_scores=round_scores)
    assert torch.equal(fast.view(torch.int16), slow.view(torch.int16))
    check_d64(fast, qkv, B, S, H, [672, 600], table, 1.0, round_scores, const_from=128, what="saturating table")

    broken = table.clone()
    far = torch.arange(2 * S - 1, device=dev) - (S - 1)
    broken[:, far.abs() >= 200] += 3.0 * torch.sin(far[far.abs() >= 200].float())[None]       # no longer constant past 128
    fast_b = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=broken, scale=1.0, bias_const_from=128, round_scores=round_scores)
    slow_b = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=broken, scale=1.0, bias_const_from=0, round_scores=round_scores)
    assert not torch.equal(fast_b, slow_b)
    check_d64(slow_b, qkv, B, S, H, [672, 600], broken, 1.0, round_scores, what="broken promise, no fast path")


def test_persistent_schedule_every_row_and_guard_bands(dev, ops):
    """40 samples x 8 heads x 6 query tiles = 1920 work items, far more than one CTA per SM, with lengths from 0 to S: every output
    row is checked, and guard bands on both sides of the output buffer stay untouched."""
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _ptr, _stream_ptr, _check
    lib = _lib.load()
    gen = torch.Generator().manual_seed(4)
    B, S, H = 40, 672, 8
    qkv = random_qkv(B, S, H, gen, dev, False)
    lens_l = torch.randint(0, S + 1, (B,), generator=gen).tolist()
    lens_l[:6] = [0, 1, 672, 128, 64, 65]
    lens = torch.tensor(lens_l, device=dev, dtype=torch.int32)
    table = saturating_table(H, S, gen).to(dev)
    guard = 4096
    n = B * S * H * 64
    buf = torch.full((guard + n + guard,), 0x7F7B, dtype=torch.int16, device=dev)
    out = buf[guard:guard + n]
    torch.cuda.synchronize()
    _check(lib.vqa_op_attention_d64(_ptr(qkv), _ptr(out), B, S, H, _ptr(lens), _ptr(table), 1.0, 128, 0, _stream_ptr(qkv.device)),
           None, "vqa_op_attention_d64")
    torch.cuda.synchronize()
    assert bool((buf[:guard] == 0x7F7B).all()) and bool((buf[guard + n:] == 0x7F7B).all())
    got = out.view(torch.bfloat16).view(B * S, H * 64)
    check_d64(got, qkv, B, S, H, lens_l, table, 1.0, False, const_from=128, discriminate=False, what="persistent schedule")


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("B,S,H,use_bias,ragged,scale", [(2, 100, 4, True, True, 1.0), (3, 577, 16, False, False, 0.125),
                                                         (2, 672, 8, True, True, 1.0), (1, 64, 1, True, False, 1.0),
                                                         (2, 65, 2, False, True, 0.125), (2, 300, 4, True, True, 0.5),
                                                         (5, 300, 64, True, True, 1.0)])   # B*H >= 296: more items than CTAs
def test_attention_matches_torch(dev, ops, B, S, H, use_bias, ragged, scale, round_scores):
    """Small and odd shapes with an unstructured bias table (no constancy promise); scale 0.5 with a bias shows that the non-ROUND kernel
    scales the score, not the bias."""
    gen = torch.Generator().manual_seed(5)
    qkv = random_qkv(B, S, H, gen, dev, round_scores, grid_amp=2.0)
    lens = torch.randint(max(1, S // 2), S + 1, (B,), generator=gen).tolist() if ragged else None
    table = (torch.randn(H, 2 * S - 1, generator=gen) * 0.5).bfloat16().float().to(dev) if use_bias else None
    out = ops.attention(qkv, B, S, H, seq_lens=None if lens is None else lens_tensor(lens, B, S, dev), bias_table=table, scale=scale,
                        round_scores=round_scores)
    check_d64(out, qkv, B, S, H, lens, table, scale, round_scores, what=f"B={B} S={S} H={H}")


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("use_bias", [True, False])
def test_attention_edge_lengths_and_growing_maxima(dev, ops, use_bias, round_scores):
    """Lengths around the 32-key chunk, 64-key half and 128-key tile edges (a single valid key, query blocks that are all padding), and
    scores whose row maximum grows by far more than the lazy-rescale threshold (2^8) from one key tile to the next, so the deferred rescale
    of O and l runs in every tile."""
    gen = torch.Generator().manual_seed(21)
    lens = [1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128, 129, 160, 161, 255, 256, 257, 290, 300]
    B, S, H = len(lens), 300, 2
    x = torch.randn(B, S, 3, H, 64, generator=gen) * 0.5
    if round_scores:        # integer growth keeps q.k on the exact-score grid (multiples of 1/16, |s| < 2^14)
        x[:, :, :2] = on_grid(x[:, :, :2])
        ramp = 1.0 + (torch.arange(S) // 64).float()
    else:
        ramp = 1.0 + 0.9 * (torch.arange(S) // 64).float()        # later keys are longer vectors: maxima keep growing
    x[:, :, 1] *= ramp[None, :, None, None]
    x[:, :, 0] *= 2.0
    qkv = x.reshape(B * S, 3 * H * 64).bfloat16().to(dev)
    table = (torch.randn(H, 2 * S - 1, generator=gen) * 0.5).bfloat16().float().to(dev) if use_bias else None
    out = ops.attention(qkv, B, S, H, seq_lens=lens_tensor(lens, B, S, dev), bias_table=table, scale=1.0, round_scores=round_scores)
    q, k, _ = heads(qkv.double(), B, S, H)
    sc = torch.matmul(q, k.transpose(-1, -2))
    kmask = torch.arange(S, device=dev)[None, :] < torch.tensor(lens, device=dev)[:, None]
    sc = sc.masked_fill(~kmask[:, None, None, :], float("-inf"))
    assert float((sc.amax(-1) - sc[..., :128].amax(-1)).max()) > 16.0      # the fixture does exercise the rescale
    check_d64(out, qkv, B, S, H, lens, table, 1.0, round_scores, what="edge lengths")


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("S,dist,ragged", [(672, 128, False), (672, 128, True), (400, 40, True), (300, 299, False), (672, 130, True)])
def test_attention_saturating_t5_bias(dev, ops, S, dist, ragged, round_scores):
    """T5 buckets saturate at relative_attention_max_distance: the bias is one value per head and side for |key - query| >= dist (large
    magnitudes, many key tiles). With the constancy promise and without it (every tile reads the table), both against the reference."""
    gen = torch.Generator().manual_seed(11)
    B, H = 2, 3
    qkv = random_qkv(B, S, H, gen, dev, round_scores)
    lens = torch.randint(S // 2, S + 1, (B,), generator=gen).tolist() if ragged else None
    table = saturating_table(H, S, gen, dist=dist, mult=2.0).to(dev)
    sl = None if lens is None else lens_tensor(lens, B, S, dev)
    out = ops.attention(qkv, B, S, H, seq_lens=sl, bias_table=table, scale=1.0, bias_const_from=dist, round_scores=round_scores)
    generic = ops.attention(qkv, B, S, H, seq_lens=sl, bias_table=table, scale=1.0, round_scores=round_scores)
    check_d64(out, qkv, B, S, H, lens, table, 1.0, round_scores, const_from=dist, what=f"promise {dist}")
    check_d64(generic, qkv, B, S, H, lens, table, 1.0, round_scores, discriminate=False, what="no promise")


@pytest.mark.parametrize("S,use_bias,scale", [(672, True, 1.0), (577, False, 0.125), (200, True, 1.0)])
def test_attention_reference_rounding_points(dev, ops, S, use_bias, scale):
    """round_scores forms the bf16 tensors of the reference's eager attention before the fp32 softmax (modeling_t5.py:308-331: `scores =
    matmul(q, k^T)` is bf16, `scores += position_bias` is a bf16 add; modeling_clip.py: bf16 matmul * 2^-3). Large scores on the exact-score
    grid, where the rounding moves exponents by up to 0.125: the kernel must follow the rounded restatement element by element, and the
    fixture must tell it from one that skips the rounding of score + bias or, with a bias, that does not round at all."""
    gen = torch.Generator().manual_seed(3)
    B, H = 2, 4
    qkv = random_qkv(B, S, H, gen, dev, True, grid_amp=2.0)
    table = saturating_table(H, S, gen, mult=2.0).to(dev) if use_bias else None
    const_from = 128 if use_bias else 0
    got = ops.attention(qkv, B, S, H, bias_table=table, scale=scale, bias_const_from=const_from, round_scores=True)
    check_d64(got, qkv, B, S, H, None, table, scale, True, const_from=const_from, what="ROUND")
    if not use_bias:
        return
    q, k, v = heads(qkv, B, S, H)
    ref, ref_p = d64_ref(q[0], k[0], v[0], S, S, table, scale, True)
    unrounded = d64_ref(q[0], k[0], v[0], S, S, table, scale, False)[0]
    tol = attn_bound(ref, ref_p)
    assert bool(((unrounded - ref).abs() > 4.0 * tol).any()), "fixture cannot see a ROUND kernel that does not round"


# ================================================================================================ 3. schedule and padding invariance
def ragged_lens(B, S, gen):
    lens = torch.randint(0, S + 1, (B,), generator=gen).tolist()
    lens[:3] = [0, 1, S]
    return lens


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("use_bias", [True, False])
def test_schedule_invariance(dev, ops, use_bias, round_scores):
    """Work items are numbered head-major and split over about one CTA per SM, so where an item runs, which CTA ran the item before it and
    where in the ring and Q slots it starts all change with the launch. The output of every (sample, head) is bit-identical across the full
    launch, a B = 1 launch of that sample, the batch in reverse order, and an H = 1 launch of that head (its qkv columns and bias row)."""
    gen = torch.Generator().manual_seed(31)
    B, S, H = 40, 672, 8
    lens = ragged_lens(B, S, gen)
    qkv = random_qkv(B, S, H, gen, dev, round_scores)
    table = saturating_table(H, S, gen, mult=2.0).to(dev) if use_bias else None
    kw = dict(scale=1.0 if use_bias else 0.125, bias_const_from=128 if use_bias else 0, round_scores=round_scores)
    full = ops.attention(qkv, B, S, H, seq_lens=lens_tensor(lens, B, S, dev), bias_table=table, **kw).view(B, S, H, 64)
    check_d64(full.view(B * S, H * 64), qkv, B, S, H, lens, table, kw["scale"], round_scores, discriminate=False, what="full launch")
    x = qkv.view(B, S, 3 * H * 64)
    for b in range(B):
        one = ops.attention(x[b], 1, S, H, seq_lens=lens_tensor(lens[b:b + 1], 1, S, dev), bias_table=table, **kw)
        assert torch.equal(one.view(S, H, 64).view(torch.int16), full[b].view(torch.int16)), f"B = 1 launch of sample {b}"
    rev = ops.attention(x.flip(0).reshape(B * S, -1).contiguous(), B, S, H, seq_lens=lens_tensor(lens[::-1], B, S, dev), bias_table=table, **kw)
    assert torch.equal(rev.view(B, S, H, 64).flip(0).view(torch.int16), full.view(torch.int16)), "batch in reverse order"
    for h in range(H):
        xh = qkv.view(B * S, 3, H, 64)[:, :, h].reshape(B * S, 3 * 64).contiguous()
        th = None if table is None else table[h:h + 1].contiguous()
        one = ops.attention(xh, B, S, 1, seq_lens=lens_tensor(lens, B, S, dev), bias_table=th, **kw)
        assert torch.equal(one.view(B, S, 64).view(torch.int16), full[:, :, h].contiguous().view(torch.int16)), f"H = 1 launch of head {h}"


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("use_bias", [True, False])
def test_padding_content_is_invisible(dev, ops, use_bias, round_scores):
    """Q / K / V rows at or past a sample's length hold +-3.0e38 (finite in bf16; their scores overflow) or zeros: the outputs are
    bit-identical, padding rows +0 in both."""
    gen = torch.Generator().manual_seed(41)
    S, H = 672, 8
    lens = T5_LENS
    B = len(lens)
    qkv = random_qkv(B, S, H, gen, dev, round_scores)
    table = saturating_table(H, S, gen, mult=2.0).to(dev) if use_bias else None
    kw = dict(seq_lens=lens_tensor(lens, B, S, dev), bias_table=table, scale=1.0 if use_bias else 0.125,
              bias_const_from=128 if use_bias else 0, round_scores=round_scores)
    pad = (torch.arange(S)[None, :] >= torch.tensor(lens)[:, None]).reshape(B * S).to(dev)
    zero = qkv.clone()
    zero[pad] = 0
    huge = qkv.clone()
    sign = torch.randint(0, 2, (int(pad.sum()), 3 * H * 64), generator=gen).float() * 2 - 1
    huge[pad] = (sign * 3.0e38).bfloat16().to(dev)
    assert bool(torch.isfinite(huge.float()).all())
    a = ops.attention(zero, B, S, H, **kw)
    b = ops.attention(huge, B, S, H, **kw)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert bool((a[pad].view(torch.int16) == 0).all())


# ================================================================================================ 4. the 3-stage and 2-stage rings
@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("S", RING_LENGTHS)
def test_long_rings(dev, ops, S, round_scores):
    """Past S = 8,304 the bias row leaves room for 3 ring stages only, past 12,400 for 2: 8,305 and 12,401 are the first lengths of each.
    One sample of length S and one of S - 77 (a partial last key tile and a padding tail), T5's saturating table, against the fp64
    restatement in blocks of 1,024 query rows."""
    gen = torch.Generator().manual_seed(S)
    B, H = 2, 2
    lens = [S, S - 77]
    qkv = random_qkv(B, S, H, gen, dev, round_scores)
    table = saturating_table(H, S, gen, mult=2.0).to(dev)
    out = ops.attention(qkv, B, S, H, seq_lens=lens_tensor(lens, B, S, dev), bias_table=table, scale=1.0, bias_const_from=128,
                        round_scores=round_scores)
    check_d64(out, qkv, B, S, H, lens, table, 1.0, round_scores, const_from=128, discriminate=False, what=f"S = {S}")


@pytest.mark.parametrize("round_scores", [False, True])
def test_long_ring_bias_selector(dev, ops, round_scores):
    """The bias selector on the 2-stage ring at the longest sequence a bias row allows, bit for bit."""
    S = MAX_BIAS_LEN
    lens = [S, S - 77, 129]
    gen = torch.Generator().manual_seed(7)
    qkv, table, want = bias_selector_fixture(lens, S, gen, bias_shifts(128))
    B, H = len(lens), table.shape[0]
    out = ops.attention(qkv.to(dev), B, S, H, seq_lens=lens_tensor(lens, B, S, dev), bias_table=table.to(dev), scale=1.0,
                        bias_const_from=128, round_scores=round_scores)
    assert_bits(out, want, f"S = {S}")


def test_bias_row_longer_than_shared_memory_is_refused(dev):
    """One row more than the 2-stage ring leaves room for: refused before anything launches, the output untouched."""
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _ptr, _stream_ptr
    lib = _lib.load()
    S, H = MAX_BIAS_LEN + 1, 1
    qkv = torch.zeros(S, 3 * H * 64, dtype=torch.bfloat16, device=dev)
    out = torch.full((S, H * 64), 7.0, dtype=torch.bfloat16, device=dev)
    table = torch.zeros(H, 2 * S - 1, device=dev)
    torch.cuda.synchronize()
    for round_scores in (0, 1):
        assert lib.vqa_op_attention_d64(_ptr(qkv), _ptr(out), 1, S, H, None, _ptr(table), 1.0, 128, round_scores, _stream_ptr(dev)) == INVALID
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())

"""Kernel-level parity of the CLIP-FlanT5 scoring path's glue kernels on a real H100, through the C ABI (vqa_op_*): the patch gather, the
multimodal splice, the decoder-input shift and embedding, the encoder's relative-position bias table, the lm_head score (EPI_LSE GEMM +
lse_finalize_kernel), the T5 RMSNorm and the row sums of squares of the fused-norm chain.

References are plain torch restatements (the oracle's splice_multimodal, shift_right, scores_from_logits, transformers' T5 bucket
function), bit-exact where the kernel only moves data and in fp64 where it computes. Outputs sit between sentinel guard bands; input
elements a kernel must not read hold NaN. Each group also checks that its fixture discriminates: the reference with a plausible kernel
mistake applied differs from the correct one by far more than the tolerance."""
import math
from types import SimpleNamespace

import pytest
import torch

from oracle import clipt5_oracle as orc

pytestmark = pytest.mark.gpu

SENTINEL16 = 0x7FA5            # bf16 NaN bit pattern, distinct from the NaN arithmetic produces (0x7FC0)
SENTINEL32 = 0x7FA5A5A5        # fp32 NaN bit pattern
GUARD = 256                    # guard elements on either side (keeps 16-byte alignment)
IMG = orc.IMAGE_TOKEN_INDEX
IGNORE = -100


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


class Guarded:
    """A contiguous tensor of `shape` inside a sentinel-filled buffer with GUARD elements before and after."""

    def __init__(self, shape, dtype):
        self.n = math.prod(shape)
        itype, self.fill = (torch.int16, SENTINEL16) if dtype == torch.bfloat16 else (torch.int32, SENTINEL32)
        self.itype = itype
        self.raw = torch.full((GUARD + self.n + GUARD,), self.fill, dtype=itype, device="cuda")
        self.t = self.raw[GUARD:GUARD + self.n].view(dtype).view(shape)

    def bits(self):
        return self.raw[GUARD:GUARD + self.n].view(self.t.shape)

    def guards_intact(self):
        return bool((self.raw[:GUARD] == self.fill).all() and (self.raw[GUARD + self.n:] == self.fill).all())


def bits16(t):
    return t.contiguous().view(torch.int16)


def nan_row_table(V, D, nan_row, gen, scale=1.0):
    """A bf16 [V, D] embedding table with row `nan_row` all NaN: ids that must not be read point at it."""
    t = (torch.randn(V, D, generator=gen) * scale).bfloat16()
    t[nan_row] = float("nan")
    return t


# ================================================================================================ A. patch gather
def patchify_ref(pix, patch, kpad):
    """Conv2d-weight order k = c * patch^2 + ky * patch + kx of each patch (row-major over the grid), bf16, zero K padding."""
    n, _, S, _ = pix.shape
    g = S // patch
    rows = pix.float().reshape(n, 3, g, patch, g, patch).permute(0, 2, 4, 1, 3, 5).reshape(n * g * g, 3 * patch * patch)
    out = torch.zeros(n * g * g, kpad, dtype=torch.bfloat16, device=pix.device)
    out[:, :3 * patch * patch] = rows.bfloat16()
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n,size", [(1, 336), (5, 336), (3, 56), (64, 56)])
def test_patchify(ops, n, size, dtype):
    """336 / 14 (P = 576, kpad 640) and the tiny config's 56 / 14; fp32 pixels round to bf16 in the kernel, bit-exact; columns [588, 640)
    exactly +0."""
    patch, kpad = 14, 640
    gen = torch.Generator(device="cuda").manual_seed(n * 1000 + size)
    pix = (torch.randn(n, 3, size, size, device="cuda", generator=gen) * 1.7).to(dtype)
    P = (size // patch) ** 2
    out = Guarded((n * P, kpad), torch.bfloat16)
    ops.patchify(pix, patch, kpad, out=out.t)
    torch.cuda.synchronize()
    ref = patchify_ref(pix, patch, kpad)
    assert out.guards_intact()
    assert torch.equal(out.bits(), bits16(ref))
    assert bool((out.bits()[:, 588:] == 0).all()), "K padding must be +0"
    # discrimination: swapping ky / kx (a transposed patch) or truncating instead of rounding moves the rows
    swapped = pix.float().reshape(n, 3, size // patch, patch, size // patch, patch).permute(0, 2, 4, 1, 5, 3).reshape(n * P, -1).bfloat16()
    assert not torch.equal(bits16(swapped), bits16(ref[:, :588]))
    if dtype == torch.float32:
        trunc = (pix.view(torch.int32) & ~0xFFFF).view(torch.float32)
        assert not torch.equal(bits16(patchify_ref(trunc, patch, kpad)), bits16(ref))


# ================================================================================================ B. multimodal splice
def splice_case(B, L, P, D, n_images, gen, slots, lens, V=512, ldf_pad=8):
    """ids [B, L] with an image slot at slots[b] (None: no slot) inside lens[b] ids; ids past lens[b] point at the NaN row V - 1. The
    features are blocks of P + 1 rows (CLS first, NaN) with ldf = D + ldf_pad columns (the padding NaN)."""
    nan_id = V - 1
    shared = nan_row_table(V, D, nan_id, gen)
    ids = torch.randint(0, V - 1, (B, L), generator=gen, dtype=torch.int32)
    for b in range(B):
        ids[b, lens[b]:] = nan_id
        if slots[b] is not None:
            ids[b, slots[b]] = IMG
    feats = torch.full((n_images * (P + 1), D + ldf_pad), float("nan"), dtype=torch.bfloat16)
    body = torch.randn(n_images, P, D, generator=gen).bfloat16()
    feats.view(n_images, P + 1, D + ldf_pad)[:, 1:, :D] = body
    return shared, ids, torch.tensor(lens, dtype=torch.int32), feats, body


def run_splice(ops, shared, ids, lens, index, feats, P):
    B, L = ids.shape
    D = shared.shape[1]
    S = L - 1 + P
    out = Guarded((B, S, D), torch.bfloat16)
    sl = Guarded((B,), torch.float32)
    dev = lambda t: None if t is None else t.cuda()
    ops.splice_embed(dev(ids), dev(lens), dev(index), dev(shared), dev(feats), P, P + 1, 1, IMG, out=out.t, seq_lens=sl.t.view(torch.int32))
    torch.cuda.synchronize()
    assert out.guards_intact() and sl.guards_intact()
    return out, sl.t.view(torch.int32).cpu()


def splice_ref(shared, ids, lens, body, index):
    sd = {"shared.weight": shared}
    emb, mask = orc.splice_multimodal(sd, ids.long(), lens, body.float(), None if index is None else index.long(), mode="fp32")
    return emb.bfloat16(), mask.sum(1).to(torch.int32)


SPLICE_CASES = {
    # B = 6, L = 12, tiny width: slot at 0, middle, text_len - 1, none; text_lens 1 (slot only), L, ragged
    "tiny": dict(B=6, L=12, P=16, D=256, slots=[0, 5, 11, None, 0, 2], lens=[9, 12, 12, 7, 1, 3]),
    "tiny_no_text_slot": dict(B=3, L=5, P=16, D=256, slots=[None, None, 4], lens=[1, 5, 5]),
    "xxl_b64": dict(B=64, L=40, P=576, D=4096, slots=None, lens=None),
}


@pytest.mark.parametrize("index_kind", ["identity", "repeats"])
@pytest.mark.parametrize("case", list(SPLICE_CASES))
def test_splice(ops, case, index_kind):
    """Bit-exact against the oracle's splice_multimodal, seq_lens included; rows past seq_len +0. NaN sits in every CLS row, in the
    feature padding columns and in the embedding row that ids past text_len point at."""
    c = dict(SPLICE_CASES[case])
    gen = torch.Generator().manual_seed(len(case) * 31 + len(index_kind))
    B, L = c["B"], c["L"]
    if c["slots"] is None:          # B = 64: every slot position and text length, drawn
        c["lens"] = [L if b % 9 == 0 else (1 if b % 9 == 1 else int(torch.randint(2, L + 1, (1,), generator=gen))) for b in range(B)]
        c["slots"] = [None if b % 7 == 3 else [0, c["lens"][b] - 1, c["lens"][b] // 2][b % 3] for b in range(B)]
    if index_kind == "identity":
        n_images, index = B, None
    else:                           # repeats, out of order, some images unused
        n_images = max(2, B // 3 + 1)
        index = torch.randint(0, n_images, (B,), generator=gen, dtype=torch.int32)
        index[0], index[-1] = n_images - 1, n_images - 1
    shared, ids, lens, feats, body = splice_case(B, L, c["P"], c["D"], n_images, gen, c["slots"], c["lens"])
    out, sl = run_splice(ops, shared, ids, lens, index, feats, c["P"])
    ref, ref_len = splice_ref(shared, ids, lens, body, index)
    assert torch.equal(sl, ref_len), (sl, ref_len)
    assert torch.equal(out.bits().cpu(), bits16(ref))        # includes +0 past seq_len and no NaN anywhere
    # discrimination: the fixture sees the image index and the CLS offset
    if index is not None:
        ident = index.clone()
        ident.copy_(torch.arange(B, dtype=torch.int32) % n_images)
        assert not torch.equal(bits16(splice_ref(shared, ids, lens, body, ident)[0]), bits16(ref))
    cls_first = feats.view(n_images, c["P"] + 1, -1)[:, :c["P"], :c["D"]]       # offset 0: rows 0 .. P - 1 (CLS = NaN first)
    assert bool(torch.isnan(splice_ref(shared, ids, lens, cls_first, index)[0][[b for b in range(B) if c["slots"][b] is not None]]).any())


# ================================================================================================ C. decoder embedding
NEG_LABELS = [IGNORE, -1, -2, -101, -(2 ** 31)]


def decoder_labels(B, T, V, nan_id, gen):
    """Labels in [0, V - 1) with -100 and other negative labels at the start, middle and end of rows; the last label of every row (never
    read after the shift) is the NaN row."""
    lab = torch.randint(0, V - 1, (B, T), generator=gen, dtype=torch.int32)
    for b in range(B):
        neg = NEG_LABELS[b % len(NEG_LABELS)]
        if T >= 3:
            lab[b, [0, T // 2, T - 2][b % 3]] = neg
        elif T == 2:
            lab[b, 0] = neg
    lab[:, -1] = nan_id
    return lab


@pytest.mark.parametrize("T", [1, 2, 5, 33, 256])
def test_decoder_embed(ops, T):
    """Bit-exact shift_right + embedding; every negative label embeds the pad id (start id 3, pad id 5)."""
    gen = torch.Generator().manual_seed(T)
    V, D, B = 512, 256, 11
    shared = nan_row_table(V, D, V - 1, gen)
    labels = decoder_labels(B, T, V, V - 1, gen)
    cfg = SimpleNamespace(decoder_start_id=3, pad_token_id=5)
    out = Guarded((B * T, D), torch.bfloat16)
    ops.decoder_embed(labels.cuda(), shared.cuda(), B, T, start_id=3, pad_id=5, out=out.t)
    torch.cuda.synchronize()
    ids = orc.shift_right(labels.masked_fill(labels < 0, IGNORE), cfg)
    ref = shared[ids.long()].reshape(B * T, D)
    assert out.guards_intact() and torch.equal(out.bits().cpu(), bits16(ref))
    if T > 1:
        assert bool((labels[:, :-1] < 0).any()) and bool((labels[:, :-1] < -100).any()), "the fixture feeds negative labels"
        assert bool(torch.isnan(shared[labels.clamp(min=0).long()]).any()), "without the shift the NaN row is read"
    if T == 1:      # the generation prefill: no labels
        out1 = Guarded((B, D), torch.bfloat16)
        ops.decoder_embed(None, shared.cuda(), B, 1, start_id=3, pad_id=5, out=out1.t)
        torch.cuda.synchronize()
        assert out1.guards_intact() and torch.equal(out1.bits().cpu(), bits16(shared[3].expand(B, D)))


def test_decoder_embed_xxl_width(ops):
    """B = 64, T = 2 at D = 4096 (the benchmark's decoder input)."""
    gen = torch.Generator().manual_seed(77)
    V, D, B, T = 1024, 4096, 64, 2
    shared = nan_row_table(V, D, V - 1, gen)
    labels = decoder_labels(B, T, V, V - 1, gen)
    out = Guarded((B * T, D), torch.bfloat16)
    ops.decoder_embed(labels.cuda(), shared.cuda(), B, T, start_id=0, pad_id=0, out=out.t)
    torch.cuda.synchronize()
    ids = orc.shift_right(labels.masked_fill(labels < 0, IGNORE), SimpleNamespace(decoder_start_id=0, pad_token_id=0))
    assert out.guards_intact() and torch.equal(out.bits().cpu(), bits16(shared[ids.long()].reshape(B * T, D)))


# ================================================================================================ D. relative-position bias table
H_REL, BUCKETS, MAX_DIST = 64, 32, 128


def hf_bucket(rel):
    from transformers.models.t5.modeling_t5 import T5Attention
    return T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=BUCKETS, max_distance=MAX_DIST)


@pytest.fixture(scope="module")
def rel_fixture(ops):
    gen = torch.Generator().manual_seed(5)
    rel_emb = torch.randn(BUCKETS, H_REL, generator=gen).bfloat16()
    lut = ops.t5_bucket_lut(True, BUCKETS, MAX_DIST).cuda()
    return rel_emb, lut


@pytest.mark.parametrize("S", [1, 2, 128, 129, 257, 607, 672])
def test_bias_table(ops, rel_fixture, S):
    """table[h, r] = rel_emb[bucket(r - (S - 1)), h], bit-exact against transformers' bucket function; constant per head and side past
    max_distance (what bias_const_from = 128 assumes)."""
    rel_emb, lut = rel_fixture
    out = Guarded((H_REL, 2 * S - 1), torch.float32)
    ops.t5_bias_table(rel_emb.cuda(), lut, MAX_DIST, S, out=out.t)
    torch.cuda.synchronize()
    rel = torch.arange(2 * S - 1) - (S - 1)
    ref = rel_emb.float()[hf_bucket(rel)].t()
    got = out.t.cpu()
    assert out.guards_intact() and torch.equal(got.view(torch.int32), ref.contiguous().view(torch.int32))
    far = rel.abs() >= MAX_DIST
    if bool(far.any()):
        edge = torch.where(rel > 0, S - 1 + MAX_DIST, S - 1 - MAX_DIST)
        assert torch.equal(got[:, far], got[:, edge[far]])
    # discrimination: rel_emb read as [H, buckets]
    if S > 1:
        wrong = rel_emb.reshape(-1).float().view(H_REL, BUCKETS)[:, hf_bucket(rel)]
        assert not torch.equal(wrong, ref)


def test_bias_const_from_is_exact(ops, rel_fixture):
    """The encoder attention with the production table and bias_const_from = 128 is bit-identical to the same call that assumes nothing."""
    rel_emb, lut = rel_fixture
    B, S, H = 2, 672, H_REL
    table = ops.t5_bias_table(rel_emb.cuda(), lut, MAX_DIST, S)
    gen = torch.Generator(device="cuda").manual_seed(9)
    qkv = (torch.randn(B * S, 3 * H * 64, device="cuda", generator=gen) * 0.3).bfloat16()
    seq_lens = torch.tensor([S, 500], dtype=torch.int32, device="cuda")
    for round_scores in (False, True):
        a = ops.attention(qkv, B, S, H, seq_lens=seq_lens, bias_table=table, bias_const_from=MAX_DIST, round_scores=round_scores)
        b = ops.attention(qkv, B, S, H, seq_lens=seq_lens, bias_table=table, bias_const_from=0, round_scores=round_scores)
        torch.cuda.synchronize()
        assert torch.equal(bits16(a), bits16(b)), round_scores


# ================================================================================================ E. lm_head score
LSE_TOL = 1e-5          # fp32 log-sum-exp noise: the integer fixture's logits are exact


def score_labels(B, T, N, gen):
    """Labels in [0, N) with -100 holes at the start, middle and end of rows, and one row (1) whose labels are all -100."""
    lab = torch.randint(0, N, (B, T), generator=gen, dtype=torch.int32)
    lab[0, 0] = N - 1
    if T > 1:
        for b in range(2, B):
            lab[b, [0, T // 2, T - 1][b % 3]] = IGNORE
    lab[1] = IGNORE
    return lab


def fp64_score(logits, labels):
    """fp64 log_softmax of the bf16 logits, the label gather and the mean over non-ignored labels: (scores [B], logprobs [B, T])."""
    logp = torch.log_softmax(logits.bfloat16().double(), -1)
    valid = labels != IGNORE
    tok = logp.gather(-1, labels.clamp(min=0).long()[..., None])[..., 0] * valid
    return torch.exp(tok.sum(-1) / valid.sum(-1)), tok


@pytest.fixture(scope="module")
def int_lm_head():
    """Integer-valued lm_head weights (multiples of 1/16 in [-3/16, 3/16]) at K = 4096 for both vocabularies."""
    gen = torch.Generator().manual_seed(61)
    return {N: (torch.randint(-3, 4, (N, 4096), generator=gen).float() / 16).bfloat16().cuda() for N in (32128, 1000)}


def check_score(ops, h, w, labels, ref_scores, ref_tok, tol):
    B, T = labels.shape
    scores, logp = Guarded((B,), torch.float32), Guarded((B * T,), torch.float32)
    ops.lmhead_score(h, w, labels.cuda(), scores=scores.t, logprobs=logp.t)
    torch.cuda.synchronize()
    assert scores.guards_intact() and logp.guards_intact()
    valid = (labels != IGNORE).reshape(-1).cuda()
    assert bool((logp.bits()[~valid] == SENTINEL32).all()), "ignored positions are not written"
    err = (logp.t.double() - ref_tok.reshape(-1).cuda())[valid].abs().max()
    assert float(err) <= tol, float(err)
    s = scores.t.double().cpu()
    empty = ~(labels != IGNORE).any(1)
    assert bool(torch.isnan(s[empty]).all()) and bool(torch.isnan(ref_scores[empty]).all()), "a row without labels scores NaN"
    rel = (s[~empty].log() - ref_scores[~empty].log()).abs().max()
    assert float(rel) <= tol, float(rel)
    return s


@pytest.mark.parametrize("N", [32128, 1000])
@pytest.mark.parametrize("T", [1, 2, 5, 12, 33])
def test_lmhead_score(ops, int_lm_head, T, N):
    """h and W are small multiples of powers of two, so every logit is exact: log-probabilities and log-scores within LSE_TOL of fp64. The
    oracle's scores_from_logits agrees (fp32), NaN for the row without labels."""
    gen = torch.Generator().manual_seed(T * 17 + N)
    B, K = 9, 4096
    w = int_lm_head[N]
    h = (torch.randint(-3, 4, (B * T, K), generator=gen).float() / 8).bfloat16().cuda()
    logits = (h.double() @ w.double().t()).cpu()
    assert torch.equal(logits, (logits * 128).round() / 128) and float(logits.abs().max()) < 2 ** 16
    logits = logits.float().view(B, T, N)
    labels = score_labels(B, T, N, gen)
    ref_scores, ref_tok = fp64_score(logits, labels)
    check_score(ops, h, w, labels, ref_scores, ref_tok, LSE_TOL)
    orc_scores, _ = orc.scores_from_logits(logits.bfloat16().float(), labels.long())
    assert torch.isnan(orc_scores[1]) and float((orc_scores.double()[2:] / ref_scores[2:] - 1).abs().max()) < 1e-4
    # discrimination: a mean that counts the ignored labels moves every holed row's log-score by far more than the tolerance
    if T > 1:
        valid = labels != IGNORE
        wrong = ref_tok.sum(-1) / T
        holed = (valid.sum(-1) < T) & valid.any(-1)
        assert float((wrong[holed] - ref_scores[holed].log()).abs().min()) > 100 * LSE_TOL


def test_lmhead_score_random_values(ops):
    """Random-valued h and W at a 5e-3 bound on log-probabilities. A random logit within 1e-5 (relative) of a bf16 rounding midpoint may
    round either way after the kernel's fp32 accumulation, so the reference takes both roundings there and bounds each log-probability
    from below and above (it increases with the label logit and decreases with every other)."""
    gen = torch.Generator().manual_seed(62)
    B, T, N, K = 16, 5, 32128, 4096
    h = torch.randn(B * T, K, generator=gen).bfloat16().cuda()
    w = (torch.randn(N, K, generator=gen) * K ** -0.5 * 3).bfloat16().cuda()
    labels = score_labels(B, T, N, gen)
    scores, logp = ops.lmhead_score(h, w, labels.cuda())
    torch.cuda.synchronize()
    exact = h.double() @ w.double().t()
    a, b = (exact * (1 - 1e-5)).float().bfloat16().double(), (exact * (1 + 1e-5)).float().bfloat16().double()
    lo, hi = torch.minimum(a, b), torch.maximum(a, b)
    lab = labels.reshape(-1, 1).clamp(min=0).long().cuda()

    def logprob(label_x, other_x):
        x = other_x.scatter(1, lab, label_x.gather(1, lab))
        return (x.gather(1, lab) - torch.logsumexp(x, -1, keepdim=True))[:, 0]
    lower, upper = logprob(lo, hi), logprob(hi, lo)
    valid = (labels != IGNORE).reshape(-1).cuda()
    g = logp.double()
    assert bool(((g >= lower - 5e-3) & (g <= upper + 5e-3))[valid].all())
    mean = lambda x: (x * valid).view(B, T).sum(-1) / valid.view(B, T).sum(-1)
    s = scores.double().log()
    assert bool(((s >= mean(lower) - 5e-3) & (s <= mean(upper) + 5e-3))[valid.view(B, T).any(-1)].all())
    assert bool(torch.isnan(scores[1]))


# ================================================================================================ F. T5 RMSNorm
NORM_WIDTHS = [256, 512, 1024, 1280, 2048, 3584, 4096, 5120, 4104]
EPS = 1e-6
norm_mismatch = {}


def norm_rows(rows, D, gen):
    """Random rows, with special rows at the front: all zero, |x| ~ 1e4 outliers, and variances (~1e-6) at which eps 1e-6 and 1e-5 differ by
    many ulps."""
    x = torch.randn(rows, D, generator=gen)
    x[0] = 0.0
    x[1, ::97] = 1e4 * torch.sign(torch.randn(x[1, ::97].shape, generator=gen))
    x[2] *= 1e-3
    x[3] *= 3e-3
    x[4, :D // 2] *= 1e-3
    return x.bfloat16()


def norm_candidates(x, gamma, eps):
    """fp64 statistics and the kernel's two rounding points, y = bf16(gamma * bf16(x * rsqrt(mean(x^2) + eps))). Where x * rstd lies within
    1e-5 (relative) of a bf16 rounding midpoint the kernel's fp32 statistics may round it either way: both candidates, and the nearest."""
    xd = x.double()
    n = xd * torch.rsqrt((xd * xd).mean(-1, keepdim=True) + eps)
    g = gamma.double()
    y = lambda v: (g * v.float().bfloat16().double()).float().bfloat16()
    return y(n), y(n * (1 - 1e-5)), y(n * (1 + 1e-5))


@pytest.mark.parametrize("rows", [13, 1003])
@pytest.mark.parametrize("D", NORM_WIDTHS)
def test_rmsnorm(ops, D, rows):
    """Every element equals the fp64 reference with one of the two bf16 roundings of the normalised value (at most one bf16 ulp there, none
    at the gain's rounding); the all-zero row gives exactly 0."""
    gen = torch.Generator().manual_seed(D * 3 + rows)
    x = norm_rows(rows, D, gen).cuda()
    gamma = (1.0 + 0.4 * torch.randn(D, generator=gen)).bfloat16().cuda()
    out = Guarded((rows, D), torch.bfloat16)
    ops.norm(x, gamma, eps=EPS, out=out.t)
    torch.cuda.synchronize()
    assert out.guards_intact()
    near, lo, hi = norm_candidates(x, gamma, EPS)
    got = out.bits()
    ok = (got == bits16(lo)) | (got == bits16(hi)) | (got == bits16(near))
    assert bool(ok.all()), int((~ok).sum())
    assert bool((out.t[0] == 0).all())
    norm_mismatch[(D, rows)] = float((got != bits16(near)).double().mean())
    print(f"rmsnorm D={D} rows={rows}: {norm_mismatch[(D, rows)]:.2e} of the elements differ from the nearest-rounding reference")
    # discrimination: eps 1e-5 moves the small-variance rows by many ulps; no rounding before the gain moves many elements
    near5 = norm_candidates(x[2:4], gamma, 1e-5)[0].double()
    ulp = torch.exp2(torch.floor(torch.log2(near[2:4].double().abs().clamp_min(2.0 ** -100))) - 7)
    assert float(((near5 - near[2:4].double()).abs() / ulp).median()) > 8
    xd = x.double()
    unrounded = (gamma.double() * (xd * torch.rsqrt((xd * xd).mean(-1, keepdim=True) + EPS))).float().bfloat16()
    assert float((bits16(unrounded) != bits16(near)).double().mean()) > 0.1


# ================================================================================================ G. row sums of squares
@pytest.mark.parametrize("rows,D", [(1003, 256), (1003, 2048), (64 * 671, 4096)])
def test_row_ssq(ops, rows, D):
    """Column 0 of every [rows, stride] partial-sum row within 1e-6 relative of fp64; the other columns untouched."""
    gen = torch.Generator().manual_seed(rows + D)
    x = norm_rows(rows, D, gen).cuda()
    x[0, 0] = 1.0                                   # no zero row: a relative bound
    stride = (D // 32 + 3) // 4 * 4
    ssq = Guarded((rows, stride), torch.float32)
    ops.row_ssq(x, ssq.t)
    torch.cuda.synchronize()
    assert ssq.guards_intact()
    assert bool((ssq.bits()[:, 1:] == SENTINEL32).all()), "slots other than 0 are not written"
    ref = (x.double() ** 2).sum(-1)
    rel = ((ssq.t[:, 0].double() - ref).abs() / ref).max()
    assert float(rel) <= 1e-6, float(rel)

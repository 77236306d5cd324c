"""Kernel-level parity of the CLIP-FlanT5 scoring path on a real H100, through the C ABI (vqa_op_*): the CLIP tower's fp32-residual GEMM,
the batched GEMM and the absorbed cross-attention of the T5 decoder (with the reference association beside it), the fp32 LayerNorm of the
CLIP residual stream and the fused CLIP embeddings + pre_layrnorm.

References are plain torch in fp64 built from the same inputs, rounded where the kernel (and the autocast module it mirrors) rounds.
Outputs sit between sentinel guard bands and padding columns that must come back bit-identical; padding the kernels must not read holds
NaN. Each group also checks that its fixture discriminates: the reference with a plausible kernel mistake applied moves by far more than
the tolerance."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL16 = 0x7FA5            # bf16 NaN bit pattern, distinct from the NaN arithmetic produces (0x7FC0)
SENTINEL32 = 0x7FA5A5A5        # fp32 NaN bit pattern
GUARD = 256                    # guard elements on either side (keeps 16-byte alignment)


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


class Guarded:
    """A [rows, cols] view with row stride `ld` inside a sentinel-filled buffer with GUARD elements before and after."""

    def __init__(self, rows, cols, dtype, ld=None):
        self.ld = ld or cols
        self.n = rows * self.ld
        itype, fill = (torch.int16, SENTINEL16) if dtype == torch.bfloat16 else (torch.int32, SENTINEL32)
        self.fill = fill
        self.raw = torch.full((GUARD + self.n + GUARD,), fill, dtype=itype, device="cuda")
        self.t = self.raw[GUARD:GUARD + self.n].view(dtype).view(rows, self.ld)[:, :cols]

    def untouched_outside(self, written):
        """Every element outside the flat index set `written` (bool [n]) still holds the sentinel."""
        inner = self.raw[GUARD:GUARD + self.n]
        return bool((self.raw[:GUARD] == self.fill).all() and (self.raw[GUARD + self.n:] == self.fill).all()
                    and (inner[~written] == self.fill).all())

    def untouched_padding(self):
        mask = torch.zeros(self.n // self.ld, self.ld, dtype=torch.bool, device="cuda")
        mask[:, :self.t.shape[1]] = True
        return self.untouched_outside(mask.flatten())


def padded(t, pad_cols=8, pad_rows=0):
    """t copied into a NaN-filled buffer with pad_cols extra columns and pad_rows extra rows: the view keeps t's shape and values."""
    buf = torch.full((t.shape[0] + pad_rows, t.shape[1] + pad_cols), float("nan"), dtype=t.dtype, device=t.device)
    buf[:t.shape[0], :t.shape[1]] = t
    return buf[:t.shape[0], :t.shape[1]]


def bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (8 significant bits)."""
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -100))) - 7)


def f32_ulp(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -100))) - 23)


def acc_tol(ref, mag):
    """One bf16 ulp of the fp64-rounded value, plus the fp32 accumulation error of a sum whose terms have absolute sum `mag` (the only
    error left where the sum cancels to near zero)."""
    return bf16_ulp(ref) + 2.0 ** -16 * mag


def bf16(x):
    """Round to bf16 (through fp32, as the kernels' fp32 values are rounded) and return fp64."""
    return x.float().bfloat16().double()


# ================================================================================================ fp32-accumulate GEMM
# CLIP out_proj (N = K = 1024) and fc2 (K = 4096) at M = n_images * 577; the tiny config's width; an N tail off every tile width.
F32ACC_SHAPES = [(577, 1024, 1024), (1731, 1024, 4096), (64 * 577, 1024, 1024), (64 * 577, 1024, 4096), (1731, 1024, 1024), (577, 1024, 4096),
                 (51, 256, 256), (51, 256, 512), (577, 1000, 1024)]
VARIANTS = [2561, 1281, 641, 321]


def residual_stream(M, N, g):
    """An fp32 CLIP-like residual: O(1) values, and every 8th column an outlier dimension of magnitude 30..300."""
    c = torch.randn(M, N, device="cuda", generator=g) * 2.0
    big = (30.0 + 270.0 * torch.rand(M, N // 8, device="cuda", generator=g)) * torch.sign(torch.randn(M, N // 8, device="cuda", generator=g))
    c[:, ::8] = big
    return c


@pytest.mark.parametrize("M,N,K", F32ACC_SHAPES)
def test_f32acc_gemm(ops, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = padded(torch.randn(M, K, device="cuda", generator=g).bfloat16())
    w = padded((torch.randn(N, K, device="cuda", generator=g) * (0.1 / math.sqrt(K))).bfloat16())
    bias = (torch.randn(N, device="cuda", generator=g) * 0.05).bfloat16()
    c_in = residual_stream(M, N, g)
    # the Linear's bf16 output: fp64 accumulation + bias, rounded once
    y = bf16(torch.addmm(bias.double(), a.double(), w.double().t()))
    assert float(y.abs().max()) < 2.0                                        # the GEMM output is small against the residual
    tol_y = acc_tol(y, torch.addmm(bias.double().abs(), a.double().abs(), w.double().abs().t()))
    # discrimination: storing bf16(residual + y) (a bf16 residual stream) errs by orders of magnitude more than the tolerance,
    # and adding y unrounded moves most elements off the exact result
    c64 = c_in.double()
    wrong = bf16(c64 + y) - c64 - y
    assert float(wrong.abs().max()) > 100 * float((tol_y + f32_ulp(c64 + y)).max())
    unrounded = torch.addmm(bias.double(), a.double(), w.double().t())
    assert float(((unrounded - y).abs() > 0.5 * f32_ulp(c64 + y)).double().mean()) > 0.5
    del unrounded, wrong
    for variant in VARIANTS:
        out = Guarded(M, N, torch.float32, ld=N + 8)
        out.t.copy_(c_in)
        ops.gemm_f32acc(a, w, out.t, bias=bias, variant=variant)
        torch.cuda.synchronize()
        assert out.untouched_padding(), variant
        o = out.t.double()
        d = (o - c64 - y).abs()                         # o - c_in is exact in fp64
        half32 = 0.5 * f32_ulp(o)
        assert bool((d <= tol_y + half32).all()), (variant, float((d - tol_y - half32).max()))
        off = float((d > half32).double().mean())       # elements whose bf16 Linear output differs from the fp64-rounded one
        assert off <= 0.01, (variant, off)
        del out, o, d


# ================================================================================================ batched GEMM
def absorbed_specs(B, T, S, H, Dm):
    """The four BatchSpecs of clipt5_absorbed_cross_attention: (name, M, N, K, nb, a_off, w_off, c_stride, ldc, a_ext, w_ext, variant)."""
    inner, Md, TH, Sp = H * 64, B * T, T * H, (S + 7) // 8 * 8
    big = 2561 if Dm >= 256 else 1281
    return [
        ("q~ = Wk^T q", Md, Dm, 64, H, (0, 64), (0, 64), Dm, H * Dm, (Md, inner), (Dm, inner), big),
        ("scores", TH, Sp, Dm, B, (TH, 0), (S, 0), TH * Sp, Sp, (B * TH, Dm), (B * S, Dm), 1281),
        ("ctx = P x", TH, Dm, Sp, B, (TH, 0), (Dm, 0), TH * Dm, Dm, (B * TH, Sp), (B * Dm, Sp), big),
        ("out = Wv ctx", Md, 64, Dm, H, (0, Dm), (64, 0), 64, inner, (Md, H * Dm), (inner, Dm), 641),
    ]


def batched_reference(a, w, M, N, K, nb, a_off, w_off, a_ext, w_ext, wrong_w_k=False):
    """[nb, M, N] fp64: batch b of A (rows past a_ext read as zero) times W (rows past w_ext zero)."""
    A = torch.zeros(a_ext[0] + nb * a_off[0] + M, a_ext[1], dtype=torch.float64, device="cuda")
    A[:a_ext[0]] = a[:a_ext[0], :a_ext[1]].double()
    W = torch.zeros(w_ext[0] + nb * w_off[0] + N, w_ext[1], dtype=torch.float64, device="cuda")
    W[:w_ext[0]] = w[:w_ext[0], :w_ext[1]].double()
    out = []
    for b in range(nb):
        ab = A[b * a_off[0]:b * a_off[0] + M, b * a_off[1]:b * a_off[1] + K]
        wk = 0 if wrong_w_k else b * w_off[1]
        wb = W[b * w_off[0]:b * w_off[0] + N, wk:wk + K]
        out.append(ab @ wb.t())
    return torch.stack(out)


BATCHED_CASES = [(3, 1, 605, 64, 4096), (2, 2, 611, 64, 4096), (5, 2, 37, 4, 256), (4, 1, 22, 4, 256)]   # B, T, S, H, d_model


@pytest.mark.parametrize("B,T,S,H,Dm", BATCHED_CASES)
def test_batched_gemm_absorbed_specs(ops, B, T, S, H, Dm):
    """Each launch against a per-batch fp64 matmul. T * H < 128 puts several batches in one A tile; the score GEMM's last batch reads
    Sp - S rows past the encoder output, which must read as zero (the rows past the extent hold NaN). C has 16 padding columns per row and,
    for the row-batched GEMMs, 3 gap rows between batches: all of it must keep its sentinel."""
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + S)
    for name, M, N, K, nb, a_off, w_off, c_stride, ldc, a_ext, w_ext, variant in absorbed_specs(B, T, S, H, Dm):
        a = padded(torch.randn(*a_ext, device="cuda", generator=g).bfloat16(), pad_rows=64)
        w = padded((torch.randn(*w_ext, device="cuda", generator=g) / math.sqrt(K)).bfloat16(), pad_rows=64)
        ldc_p = ldc + 16
        row_batched = a_off[0] > 0
        cs = (M + 3) * ldc_p if row_batched else c_stride
        rows = (nb - 1) * cs // ldc_p + M + 1 if row_batched else M
        c = Guarded(rows, ldc_p, torch.bfloat16)
        ops.gemm_batched(a, w, c.t, M, N, K, nb, a_off, w_off, cs, a_ext, w_ext, variant)
        torch.cuda.synchronize()
        flat = c.raw[GUARD:GUARD + c.n].view(torch.bfloat16)
        idx = (torch.arange(nb, device="cuda")[:, None, None] * cs + torch.arange(M, device="cuda")[None, :, None] * ldc_p
               + torch.arange(N, device="cuda")[None, None, :])
        written = torch.zeros(c.n, dtype=torch.bool, device="cuda")
        written[idx.flatten()] = True
        assert c.untouched_outside(written), name
        got = flat[idx].double()
        ref = batched_reference(a, w, M, N, K, nb, a_off, w_off, a_ext, w_ext)
        r16 = bf16(ref)
        err = (got - r16).abs()
        tol = acc_tol(r16, batched_reference(a.abs(), w.abs(), M, N, K, nb, a_off, w_off, a_ext, w_ext))
        assert bool((err <= tol).all()), (name, float((err - tol).max()))
        assert float((err > 0).double().mean()) <= 0.01, name
        if w_off[1]:   # discrimination: every batch reading batch 0's W columns
            wrong = bf16(batched_reference(a, w, M, N, K, nb, a_off, w_off, a_ext, w_ext, wrong_w_k=True))
            assert float((wrong - r16).abs().max()) > 100 * float(bf16_ulp(r16).max()), name


# ================================================================================================ cross-attention
def cross_case(B, T, S, H, Dm, seed):
    """Decoder queries, encoder output, ragged lengths and the layer's weights. Per (b, t, h) the score scale is one of 0.05 (near-uniform
    rows), 5, 12 and 30 (near-one-hot); the encoder rows past a pair's length are 20x larger, so attending to any of them shows; the
    rows after the last sample are NaN."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    inner = H * 64
    lens = [S, 1] + [int(v) for v in torch.randint(1, S + 1, (max(0, B - 2),), generator=g, device="cuda")]
    lens = lens[:B]
    x = torch.randn(B, S, Dm, device="cuda", generator=g)
    for b, L in enumerate(lens):
        x[b, L:] *= 20.0
    xbuf = torch.full((B * S + 16, Dm), float("nan"), dtype=torch.bfloat16, device="cuda")
    xbuf[:B * S] = x.reshape(B * S, Dm).bfloat16()
    x = xbuf[:B * S]
    wk = (torch.randn(inner, Dm, device="cuda", generator=g) / math.sqrt(Dm)).bfloat16()
    wv = (torch.randn(inner, Dm, device="cuda", generator=g) / math.sqrt(Dm)).bfloat16()
    scale = torch.tensor([0.05, 5.0, 12.0, 30.0], device="cuda")[torch.randint(0, 4, (B * T, H, 1), generator=g, device="cuda")]
    q = (torch.randn(B * T, H, 64, device="cuda", generator=g) * scale / 8.0).reshape(B * T, inner).bfloat16()
    seq_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    return q, x, seq_lens, wk.t().contiguous(), torch.cat([wk, wv]).contiguous(), wk, wv


def exact_cross_attention(q, x, lens, wk, wv, B, T, S, H):
    """fp64 attention in the absorbed association (exact in real arithmetic): s = (Wk^T q).x, out = Wv (sum p x). [B * T, H * 64]."""
    Dm = x.shape[1]
    out = torch.empty(B, T, H, 64, dtype=torch.float64, device="cuda")
    wk64, wv64 = wk.double().view(H, 64, Dm), wv.double().view(H, 64, Dm)
    for b in range(B):
        L = int(lens[b])
        xb = x[b * S:b * S + L].double()                                       # [L, Dm]
        qb = q[b * T:(b + 1) * T].double().view(T, H, 64)
        qt = torch.einsum("thd,hdm->thm", qb, wk64)                            # [T, H, Dm]
        p = torch.softmax(qt @ xb.t(), -1)                                     # [T, H, L]
        ctx = p @ xb                                                           # [T, H, Dm]
        out[b] = torch.einsum("thm,hdm->thd", ctx, wv64)
    return out.reshape(B * T, H * 64)


def eager_bf16_cross_attention(q, x, lens, wk, wv, B, T, S, H, round_p=True):
    """The reference model's eager bf16 association: K = bf16(x Wk^T), V = bf16(x Wv^T), bf16 scores, P = bf16(softmax_fp32), bf16(P V)."""
    out = torch.empty(B, T, H, 64, dtype=torch.float64, device="cuda")
    for b in range(B):
        L = int(lens[b])
        xb = x[b * S:b * S + L].double()
        k = bf16(xb @ wk.double().t()).view(L, H, 64).transpose(0, 1)        # [H, L, 64]
        v = bf16(xb @ wv.double().t()).view(L, H, 64).transpose(0, 1)
        qb = q[b * T:(b + 1) * T].double().view(T, H, 64).transpose(0, 1)    # [H, T, 64]
        p = torch.softmax(bf16(qb @ k.transpose(1, 2)).float(), -1).double()
        if round_p:
            p = bf16(p)
        out[b] = (p @ v).transpose(0, 1)
    return bf16(out.reshape(B * T, H * 64))


def mode0_buffers(ws, B, T, S, H, Dm):
    """The documented mode-0 workspace layout (xt | q~ | csc | ctx, each at the next multiple of 256 bytes) as bf16 views."""
    r = lambda n: (n + 255) // 256 * 256
    Sp, TH = (S + 7) // 8 * 8, T * H
    sizes = [B * Dm * Sp * 2, B * TH * Dm * 2, (B * TH + 256) * Sp * 2, B * TH * Dm * 2]
    assert ws.numel() == sum(r(n) for n in sizes)
    views, off = [], 0
    for n in sizes:
        views.append(ws[off:off + n].view(torch.bfloat16))
        off += r(n)
    xt, qt, csc, ctx = views
    return xt.view(B, Dm, Sp), qt.view(B * TH, Dm), csc.view(B * TH + 256, Sp)[:B * TH], ctx.view(B * TH, Dm)


# B, T, S, H, d_model, modes: S covers every S mod 8; B = 64 at T = 1 is a generation step
CROSS_CASES = [
    (64, 1, 45, 4, 256, (0, 1)), (7, 2, 33, 4, 256, (0, 1)), (5, 5, 42, 4, 256, (0, 1)), (3, 8, 48, 4, 256, (0, 1)), (4, 2, 39, 4, 256, (0, 1)),
    (6, 1, 22, 4, 256, (0, 1)), (4, 12, 51, 4, 256, (0,)), (3, 33, 60, 4, 256, (0,)),
    (64, 1, 83, 64, 4096, (0, 1)), (3, 2, 606, 64, 4096, (0, 1)), (2, 5, 581, 64, 4096, (0, 1)), (2, 12, 97, 64, 4096, (0,)),
]


def run_cross(ops, q, x, seq_lens, wkT, wkv, B, T, S, H, mode, round_scores=False):
    out = Guarded(B * T, H * 64, torch.bfloat16)
    # a first call sizes the workspace; the second starts from all-NaN intermediates, so an element the sequence fails to write shows
    _, ws = ops.t5_cross_attention(q, x, seq_lens, wkT, wkv, B, T, S, H, mode=mode, round_scores=round_scores, out=out.t)
    ws.fill_(0xFF)
    ops.t5_cross_attention(q, x, seq_lens, wkT, wkv, B, T, S, H, mode=mode, round_scores=round_scores, out=out.t, workspace=ws)
    torch.cuda.synchronize()
    assert out.untouched_padding()
    return out.t.double(), ws


def error_stats(got, ref):
    e = (got - ref).abs()
    return float(e.max()), float(e.mean())


@pytest.mark.parametrize("B,T,S,H,Dm,modes", CROSS_CASES)
def test_cross_attention(ops, B, T, S, H, Dm, modes):
    q, x, seq_lens, wkT, wkv, wk, wv = cross_case(B, T, S, H, Dm, seed=B * 100 + T * 10 + S)
    lens = seq_lens.tolist()
    Sp, TH = (S + 7) // 8 * 8, T * H
    exact = exact_cross_attention(q, x, lens, wk, wv, B, T, S, H)
    emul = eager_bf16_cross_attention(q, x, lens, wk, wv, B, T, S, H)
    e_max, e_mean = error_stats(emul, exact)
    # discrimination: attending to the padded rows (a mask on S instead of seq_lens) moves the result by far more than the emulation error
    leak = exact_cross_attention(q, x, [S] * B, wk, wv, B, T, S, H)
    short = [b for b in range(B) if lens[b] < S]
    rows = torch.tensor([b * T + t for b in short for t in range(T)], device="cuda")
    assert float((leak[rows] - exact[rows]).abs().max()) > 100 * e_max
    outs = {}
    for mode in modes:
        got, ws = run_cross(ops, q, x, seq_lens, wkT, wkv, B, T, S, H, mode, round_scores=True)
        assert bool(torch.isfinite(got).all()), mode
        g_max, g_mean = error_stats(got, exact)
        # at most about twice the error the reference's own bf16 association makes against the same fp64 attention
        assert g_max <= 2.0 * e_max and g_mean <= 2.0 * e_mean, (mode, g_max, e_max, g_mean, e_mean)
        outs[mode] = got
        if mode == 0:
            xt, qt, csc, ctx = mode0_buffers(ws, B, T, S, H, Dm)
            xd = x.view(B, S, Dm)
            assert torch.equal(xt[:, :, :S].contiguous().view(torch.int16), xd.transpose(1, 2).contiguous().view(torch.int16))
            assert bool((xt[:, :, S:].contiguous().view(torch.int16) == 0).all())          # pad columns exactly +0
            # P against the softmax of the kernel's own bf16 scores, which the batched GEMM recomputes bit for bit from q~
            sc = torch.empty(B * TH, Sp, dtype=torch.bfloat16, device="cuda")
            ops.gemm_batched(qt, x, sc, TH, Sp, Dm, B, (TH, 0), (S, 0), TH * Sp, (B * TH, Dm), (B * S, Dm), 1281)
            len_row = seq_lens.long().repeat_interleave(TH)[:, None]
            valid = torch.arange(Sp, device="cuda")[None, :] < len_row
            p_ref = bf16(torch.softmax(sc.double().masked_fill(~valid, float("-inf")), -1))
            p = csc.double()
            assert bool((p[~valid] == 0).all()) and bool((csc.view(torch.int16)[~valid] == 0).all())   # [len, Sp) written as +0
            assert bool(((p - p_ref).abs() <= bf16_ulp(p_ref)).all()), float((p - p_ref).abs().max())
            # q~ rows (b * T + t) * H + h: bf16(Wk_h^T q_h) within one bf16 ulp
            qk = lambda qq, ww: torch.einsum("mhd,hdk->mhk", qq.double().view(B * T, H, 64), ww.double().view(H, 64, Dm)).reshape(B * TH, Dm)
            qt_ref = bf16(qk(q, wk))
            assert bool(((qt.double() - qt_ref).abs() <= acc_tol(qt_ref, qk(q.abs(), wk.abs()))).all())
            # ctx = bf16(P x) over the padded key axis, within one bf16 ulp
            pv = lambda pp, xx: torch.bmm(pp.double().view(B, TH, Sp), xx.double().transpose(1, 2)).reshape(B * TH, Dm)
            ctx_ref = bf16(pv(csc, xt))
            assert bool(((ctx.double() - ctx_ref).abs() <= acc_tol(ctx_ref, pv(csc, xt.abs()))).all())
        else:
            # the same kernel without score rounding, against fp64 attention over the kernel's own bf16 K / V: tight
            got_f, ws = run_cross(ops, q, x, seq_lens, wkT, wkv, B, T, S, H, 1, round_scores=False)
            kv = ws[:B * S * 2 * H * 64 * 2].view(torch.bfloat16).view(B * S, 2 * H * 64)
            kv_ref = bf16(x.double() @ wkv.double().t())
            # the plain 8192-wide projection accumulates K = d_model products of encoder rows up to 20x larger than the live ones: one ulp
            # plus 2^-12 of the absolute sum, and at most 1 % of the elements off the fp64-rounded value
            kv_err = (kv.double() - kv_ref).abs()
            assert bool((kv_err <= bf16_ulp(kv_ref) + 2.0 ** -12 * (x.double().abs() @ wkv.double().abs().t())).all())
            assert float((kv_err > 0).double().mean()) <= 0.01
            ref_f = torch.empty(B * T, H, 64, dtype=torch.float64, device="cuda")
            mag = torch.empty_like(ref_f)
            for b in range(B):
                L = lens[b]
                k = kv[b * S:b * S + L, :H * 64].double().view(L, H, 64).transpose(0, 1)
                v = kv[b * S:b * S + L, H * 64:].double().view(L, H, 64).transpose(0, 1)
                qb = q[b * T:(b + 1) * T].double().view(T, H, 64).transpose(0, 1)
                p = torch.softmax(qb @ k.transpose(1, 2), -1)
                ref_f[b * T:(b + 1) * T] = (p @ v).transpose(0, 1)
                mag[b * T:(b + 1) * T] = (p @ v.abs()).transpose(0, 1)
            ref_f, mag = ref_f.reshape(B * T, -1), mag.reshape(B * T, -1)
            err = (got_f - ref_f).abs()
            assert bool((err <= bf16_ulp(ref_f) + 2.0 ** -14 * mag).all()), float((err - bf16_ulp(ref_f) - 2.0 ** -14 * mag).max())
    if len(modes) == 2:
        d_mean = float((outs[0] - outs[1]).abs().mean())
        assert d_mean <= 2.0 * e_mean, (d_mean, e_mean)


# ================================================================================================ fp32 LayerNorm
def layernorm_input(rows, D, g):
    """fp32 rows bf16 cannot represent: unit-noise rows, rows with mean 100 and spread 0.5, and rows with a few +-300 outlier dimensions."""
    x = torch.randn(rows, D, device="cuda", generator=g) * 1.7 + 0.3
    x[1::3] = 100.0 + 0.5 * torch.randn(len(range(1, rows, 3)), D, device="cuda", generator=g)
    out_cols = torch.randint(0, D, (4,), generator=g, device="cuda")
    x[2::3, out_cols] = 300.0 * torch.sign(torch.randn(len(range(2, rows, 3)), 4, device="cuda", generator=g))
    return x


def layernorm64(x, gamma, beta, eps):
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * gamma.double() + beta.double()


@pytest.mark.parametrize("D", [256, 512, 768, 1024])
def test_layernorm_f32(ops, D):
    g = torch.Generator(device="cuda").manual_seed(D)
    rows, eps = 8 * 37 + 3, 1e-5
    x = layernorm_input(rows, D, g)
    xbuf = torch.full((rows + 8, D), float("nan"), device="cuda")       # a NaN row block past the input: the kernel must not read it
    xbuf[:rows] = x
    x = xbuf[:rows]
    gamma = (1.0 + 0.2 * torch.randn(D, device="cuda", generator=g)).bfloat16()
    beta = (0.1 * torch.randn(D, device="cuda", generator=g)).bfloat16()
    ref = bf16(layernorm64(x, gamma, beta, eps))
    # one bf16 ulp, plus 2^-14 absolute for the fp32 statistics where gamma * x^ and beta cancel (2e-6 relative to a row's mean in the
    # mean-100 rows)
    tol = bf16_ulp(ref) + 2.0 ** -14
    # discrimination: a kernel that reads its input through bf16
    wrong = bf16(layernorm64(x.bfloat16(), gamma, beta, eps))
    assert float(((wrong - ref).abs() / tol).max()) > 30
    y = Guarded(rows, D, torch.bfloat16)
    ops.layernorm_f32(x, gamma, beta, eps=eps, out=y.t)
    torch.cuda.synchronize()
    assert y.untouched_padding()
    err = (y.t.double() - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())
    assert float((err > 0).double().mean()) <= 0.01


# ================================================================================================ CLIP embeddings + pre_layrnorm
@pytest.mark.parametrize("D,P,n_images", [(1024, 576, 3), (1024, 576, 1), (1024, 16, 3), (256, 16, 3), (256, 576, 1), (256, 16, 1)])
def test_clip_embed_ln(ops, D, P, n_images):
    g = torch.Generator(device="cuda").manual_seed(D + P + n_images)
    eps = 1e-5
    patch = (torch.randn(n_images * P, D, device="cuda", generator=g) * 0.7).bfloat16()
    cls = torch.randn(D, device="cuda", generator=g).bfloat16()
    pos = (torch.randn(P + 1, D, device="cuda", generator=g) * 0.3).bfloat16()
    gamma = (1.0 + 0.2 * torch.randn(D, device="cuda", generator=g)).bfloat16()
    beta = (0.1 * torch.randn(D, device="cuda", generator=g)).bfloat16()
    src = torch.cat([torch.cat([cls[None], patch[i * P:(i + 1) * P]]) for i in range(n_images)]).double()
    e = src + pos.double().repeat(n_images, 1)
    ref = layernorm64(bf16(e), gamma, beta, eps)                          # the reference adds in bf16
    tol = 1e-5 * (1.0 + ref.abs())
    # discrimination: the add left in fp32
    assert float(((layernorm64(e, gamma, beta, eps) - ref).abs() / tol).max()) > 20
    y = Guarded(n_images * (P + 1), D, torch.float32)
    pbuf = torch.full((n_images * P + 8, D), float("nan"), dtype=torch.bfloat16, device="cuda")   # NaN rows past the patches
    pbuf[:n_images * P] = patch
    ops.clip_embed_ln(pbuf[:n_images * P], cls, pos, gamma, beta, n_images, eps=eps, out=y.t)
    torch.cuda.synchronize()
    assert y.untouched_padding()
    err = (y.t.double() - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())

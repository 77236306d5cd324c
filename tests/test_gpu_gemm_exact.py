"""Bit-exact conformance of the persistent GEMM (gemm_bf16_sm90_kernel) on a real H100, through the ops wrappers and the C ABI.

A holds integers in [-3, 3] and W multiples of 1/32 in [-3/32, 3/32]. Every product is a multiple of 2^-5 and |acc| <= K * 9 / 32, so for
K < 58 000 (K * 9 / 32 < 2^24 * 2^-5) every partial sum is a multiple of 2^-5 below 2^14 in magnitude and is exact in fp32, whatever order
the wgmma k steps, the k blocks, the split-K slices or the reduction add it in. The reference is then the fp64 product rounded to fp32
(exact), followed by the kernel's own rounding points in fp32: bf16(acc + bias), then + residual and a second rounding for the bf16 stream,
or c + float(bf16(acc + bias)) for the CLIP tower's fp32 stream. The store and ReLU epilogues, f32acc, split-K, batched, grouped and the
normfuse producer are therefore compared with torch.equal on their integer views: one flipped element anywhere is a failure. The other
activations use approximate exponentials and keep a two-ulp tolerance against the reference, but their bits must not change with the
tile variant, the tile order or the number of rows.

Outputs live inside sentinel-filled buffers (row stride wider than the output, rows past M, gap rows between batches) that must come back
untouched; operands are read through views whose padding columns (lda, ldw > K) and rows past M / w_rows hold NaN, so a tensor map sized
from the allocation instead of the logical extents poisons the result.

Covered: ring laps and K tails on every tile variant (4 / 6 / 8 / 8 stages), persistent CTAs starting a tile mid-ring, the staged
epilogue's forms, every tile order (vqa_set_gemm_schedule overrides and the automatic W-chunked and A-grouped walks), and the same work
with programmatic dependent launch (VQA_PDL=1) in a child process, compared bit for bit with serial launches."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# exact fp32 accumulation bound of the operands above, kept conservative: the sums stay exact while |acc| < 2^19 (multiples of 2^-5 with
# 24 significant bits), i.e. up to K ~ 1.86 million, but 58 000 already covers every K this file uses
K_MAX = 58000
SENTINEL16 = 0x7FA5            # bf16 NaN bit pattern, distinct from the NaN arithmetic produces (0x7FC0)
SENTINEL32 = 0x7FA5A5A5        # fp32 NaN bit pattern
VARIANTS = [2561, 1281, 641, 321]
STAGES = {2561: 4, 1281: 6, 641: 8, 321: 8}
BLOCK_N = {2561: 256, 2562: 256, 1281: 128, 1282: 128, 641: 64, 321: 32}
ALL_CODES = [2561, 2562, 1281, 1282, 641, 321, 0]      # 2562 / 1282 alias 2561 / 1281; 0 = pick_variant
GATED = ("gated_gelu", "gated_silu")
ACTIVATIONS = ["quick_gelu", "gelu", "gated_gelu", "gated_silu"]
# (group_rows, chunk in N tiles of the launch's BLOCK_N, -1 = one chunk)
SCHEDULES = [(128, -1), (384, -1), (1024, 1), (384, 3), (256, 5)]
# 23 M tiles and 11 N tiles: 23 % group_m != 0 for group_m = 3, 8, 2 and 11 % chunk_n != 0 for chunk_n = 3, 5
SCHED_M = 22 * 128 + 37


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


@pytest.fixture
def schedule(ops):
    """set(group_rows, chunk_rows) overrides the tile order of every GEMM launch in the process; (0, 0) is restored whatever happens."""
    from t2v_metrics_b200 import _lib
    lib = _lib.load()

    def set_(group_rows, chunk_rows):
        assert lib.vqa_set_gemm_schedule(int(group_rows), int(chunk_rows)) == 0

    try:
        yield set_
    finally:
        lib.vqa_set_gemm_schedule(0, 0)


def schedule_rows(sched, block_n):
    group_rows, chunk_tiles = sched
    return group_rows, (chunk_tiles * block_n if chunk_tiles > 0 else -1)


def auto_schedule(w_rows, K, M, N, block_n):
    """(group_m, chunk_n, num_m_tiles, num_n_tiles) that launch_gemm_t chooses without an override: a copy of its size rules
    (gemm_sm90.cuh), used only to assert that the automatic-order tests below reach the walk they are named for. A tuning change to those
    rules must update this copy (those tests then fail on their shape precondition, not on a GPU result)."""
    w_bytes, resident = w_rows * K * 2, 14 << 20
    if w_bytes <= resident:
        group_rows, chunk_rows = 1024, -1
    else:
        n_chunks = -(-w_bytes // resident)
        if n_chunks <= 3:
            rows = -(-w_rows // n_chunks)
            chunk_rows, group_rows = -(-rows // block_n) * block_n, 1024
        else:
            chunk_rows, group_rows = -1, max(512, min(8192, (12 << 20) // (K * 2) // 256 * 256))
    n_tiles = -(-N // block_n)
    chunk_n = min(chunk_rows // block_n if chunk_rows > 0 else n_tiles, n_tiles)
    return max(1, group_rows // 128), chunk_n, -(-M // 128), n_tiles


def pick_variant(M, N, epi="store"):
    """A copy of host.cuh pick_variant, used to predict the tile (and so the Σx² slot count) of the normfuse launches, which pick their
    own. A tuning change to pick_variant must update this copy."""
    if M <= 128:
        if epi in GATED:
            return 641 if N <= 16384 else 1281
        return 321 if N <= 4096 else 641 if N <= 12288 else 1281
    return 1281 if M <= 4096 and N <= 1024 else 2561


# ------------------------------------------------------------------------------------------------ operands, buffers, references
def nan_padded(t, pad_cols=24, pad_rows=5):
    """t inside a NaN-filled buffer with pad_cols more columns and pad_rows more rows; the view has t's shape and values."""
    buf = torch.full((t.shape[0] + pad_rows, t.shape[1] + pad_cols), float("nan"), dtype=t.dtype, device=t.device)
    buf[:t.shape[0], :t.shape[1]] = t
    return buf[:t.shape[0], :t.shape[1]]


def exact_a(rows, K, g):
    assert K < K_MAX
    return nan_padded(torch.randint(-3, 4, (rows, K), device="cuda", generator=g).bfloat16())


def exact_w(rows, K, g):
    assert K < K_MAX
    return nan_padded((torch.randint(-3, 4, (rows, K), device="cuda", generator=g).float() / 32).bfloat16())


def rand_bf16(shape, g, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def exact_acc(a, w):
    """The fp32 accumulator: the fp64 product, exact for these operands, then exactly representable in fp32."""
    return (a.double() @ w.double().t()).float()


class Sentinel:
    """A [rows, cols] output with row stride ld > cols inside a sentinel-filled [rows + extra_rows, ld] buffer (bf16 or fp32)."""

    def __init__(self, rows, cols, ld, dtype=torch.bfloat16, extra_rows=3):
        self.rows, self.cols = rows, cols
        itype, self.fill = (torch.int16, SENTINEL16) if dtype == torch.bfloat16 else (torch.int32, SENTINEL32)
        self.raw = torch.full((rows + extra_rows, ld), self.fill, dtype=itype, device="cuda")
        self.t = self.raw.view(dtype)[:rows, :cols]

    def untouched_outside(self):
        mask = torch.ones_like(self.raw, dtype=torch.bool)
        mask[:self.rows, :self.cols] = False
        return bool((self.raw[mask] == self.fill).all())


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def same_bits(x, y):
    return torch.equal(bits(x), bits(y))


def ref_store(acc, bias=None, residual=None, relu=False):
    """bf16(acc + bias) [relu] [+ residual, rounded again], in fp32 like the kernel."""
    y = (acc + bias.float() if bias is not None else acc).bfloat16().float()
    if relu:
        y = y.clamp_min(0.0)
    if residual is not None:
        y = y + residual.float()
    return y.bfloat16()


def ref_f32acc(acc, c, bias=None):
    return c + (acc + bias.float() if bias is not None else acc).bfloat16().float()


def bf16_ulp(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -100))) - 7)


def ref_activation(acc, bias, epi, n_out):
    b = bias.float()
    if epi in GATED:
        g = (acc[:, :n_out] + b[:n_out]).bfloat16().double()
        u = (acc[:, n_out:2 * n_out] + b[n_out:2 * n_out]).bfloat16().double()
        if epi == "gated_gelu":
            act = 0.5 * g * (1.0 + torch.tanh(0.7978845608028654 * (g + 0.044715 * g ** 3)))
        else:
            act = (g * torch.sigmoid(g)).float().bfloat16().double()
        return (act * u).float().bfloat16()
    y = (acc + b).bfloat16().float()
    if epi == "gelu":
        y = (0.5 * y.double() * (1.0 + torch.erf(y.double() / 2 ** 0.5))).float()
    else:   # quick_gelu as eager bf16 ops
        s = (1.702 * y).bfloat16().double()
        y = (y.double() * torch.sigmoid(s).float().bfloat16().double()).float()
    return y.bfloat16()


def check_activation(got, ref):
    """Two bf16 ulps (the kernels' fast exponentials), plus an absolute term for outputs near zero."""
    assert torch.isfinite(got.float()).all()
    err = (got.double() - ref.double()).abs()
    tol = 2 * bf16_ulp(ref.double()) + 2.0 ** -16
    assert bool((err <= tol).all()), float((err - tol).max())


# ------------------------------------------------------------------------------------------------ C ABI calls without an ops wrapper
def splitk(a, w, out, bias, residual, splits):
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _check, _ptr, _stream_ptr
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    ws = torch.empty(splits * M * N, dtype=torch.float32, device="cuda")
    used = C.c_int32(0)
    _check(lib.vqa_op_gemm_bf16_splitk(_ptr(a), a.stride(0), _ptr(w), w.stride(0), N, _ptr(out), out.stride(0), M, N, K, _ptr(bias),
                                       _ptr(residual), residual.stride(0) if residual is not None else 0, splits, _ptr(ws), ws.numel() * 4,
                                       C.byref(used), _stream_ptr(a.device)), None, "vqa_op_gemm_bf16_splitk")
    assert used.value == splits
    return out


def grouped(a, w, out, bias, group_in, group_out, variant):
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _check, _ptr, _stream_ptr
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    _check(lib.vqa_op_gemm_bf16_grouped(_ptr(a), a.stride(0), _ptr(w), w.stride(0), N, _ptr(out), out.stride(0), M, N, K, _ptr(bias),
                                        group_in, group_out, variant, _stream_ptr(a.device)), None, "vqa_op_gemm_bf16_grouped")
    return out


# ================================================================================================ A. ring laps, K tails, persistent tiles
# 8 / 56: one partial k block; 64 / 72: one full block, one block and a tail; 64 * STAGES (+ 8): exactly one lap (and a tail block that
# starts the second lap); 64 * (2 * STAGES + 1) + 8: two laps and two blocks into the third; 4096: 64 blocks
K_SWEEP = sorted({8, 56, 64, 72, 4096} | {k for s in set(STAGES.values()) for k in (64 * s, 64 * s + 8, 64 * (2 * s + 1) + 8)})


@pytest.mark.parametrize("K", K_SWEEP)
def test_ring_laps_and_k_tails_every_variant(ops, K):
    """store / relu x bias or not x no, a separate or an in-place residual, on every tile variant and alias, at ragged M and N (partial
    tiles in both directions on every tile width). Every code must write the bits of 2561 and those must be the reference's."""
    M, N = 333, 328
    g = torch.Generator(device="cuda").manual_seed(K)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    res = nan_padded(rand_bf16((M, N), g), pad_cols=40, pad_rows=0)   # its own row stride, different from C's
    acc = exact_acc(a, w)
    for epi in ("store", "relu"):
        for b in (None, bias):
            for mode in ("none", "separate", "inplace"):
                ref = ref_store(acc, b, None if mode == "none" else res, relu=epi == "relu")
                first = None
                for code in ALL_CODES:
                    out = Sentinel(M, N, ld=N + 24)
                    r = None
                    if mode == "separate":
                        r = res
                    elif mode == "inplace":
                        out.t.copy_(res)
                        r = out.t
                    ops.gemm(a, w, bias=b, residual=r, epilogue=epi, variant=code, out=out.t)
                    what = (epi, b is not None, mode, code)
                    assert out.untouched_outside(), what
                    if first is None:
                        first = out.t.clone()
                        assert same_bits(first, ref), what
                    else:
                        assert same_bits(out.t, first), what


@pytest.mark.parametrize("variant", [2561, 1281, 641])
def test_many_tiles_start_mid_ring(ops, variant):
    """5 k blocks per tile on 4-, 6- and 8-stage rings over 65 x 16..64 tiles: each CTA walks several tiles, and each tile after the first
    starts at a ring slot other than 0 with the barrier phase carried over. In-place residual with bias."""
    M, N, K = 8192 + 37, 4096, 5 * 64
    assert (K // 64) % STAGES[variant] != 0
    g = torch.Generator(device="cuda").manual_seed(variant)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    out = Sentinel(M, N, ld=N + 8)
    out.t.copy_(rand_bf16((M, N), g))
    ref = ref_store(exact_acc(a, w), bias, out.t.clone())
    ops.gemm(a, w, bias=bias, residual=out.t, variant=variant, out=out.t)
    assert same_bits(out.t, ref)
    assert out.untouched_outside()


# ================================================================================================ B. the staged epilogue, bit for bit
def residual_stream(M, N, g):
    """An fp32 CLIP-like residual: O(1) values, and every 8th column an outlier dimension of magnitude 30..300."""
    c = torch.randn(M, N, device="cuda", generator=g) * 2.0
    big = (30.0 + 270.0 * torch.rand(M, N // 8, device="cuda", generator=g)) * torch.sign(torch.randn(M, N // 8, device="cuda", generator=g))
    c[:, ::8] = big
    return c


@pytest.mark.parametrize("K", [1096, 4096])
def test_f32acc_exact_every_variant(ops, K):
    """fp32 C += bf16(A W^T + bias) on the CLIP stream: bit-exact on every variant, which all write the same bits."""
    M, N = 333, 1000
    g = torch.Generator(device="cuda").manual_seed(K + 1)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    c_in = residual_stream(M, N, g)
    ref = ref_f32acc(exact_acc(a, w), c_in, bias)
    first = None
    for code in ALL_CODES:
        out = Sentinel(M, N, ld=N + 8, dtype=torch.float32)
        out.t.copy_(c_in)
        ops.gemm_f32acc(a, w, out.t, bias=bias, variant=code)
        assert out.untouched_outside(), code
        if first is None:
            first = out.t.clone()
            assert same_bits(first, ref), code
        else:
            assert same_bits(out.t, first), code


@pytest.mark.parametrize("splits", [2, 3, 4, 8])
@pytest.mark.parametrize("M", [1, 7, 100, 128])
def test_splitk_exact(ops, M, splits):
    """K slices as the batches of one launch plus splitk_reduce_kernel: the reference bits, and the bits of the unsplit GEMM."""
    N, K = 1000, 3072
    g = torch.Generator(device="cuda").manual_seed(M * 10 + splits)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    res = nan_padded(rand_bf16((M, N), g), pad_cols=40, pad_rows=0)
    out = Sentinel(M, N, ld=N + 24)
    splitk(a, w, out.t, bias, res, splits)
    plain = ops.gemm(a, w, bias=bias, residual=res)
    assert out.untouched_outside()
    assert same_bits(out.t, ref_store(exact_acc(a, w), bias, res))
    assert same_bits(out.t, plain)


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


def batched_reference(a, w, M, N, K, nb, a_off, w_off, a_ext, w_ext):
    """[nb, M, N] fp64: batch b of A (rows past a_ext read as zero) times W (rows past w_ext zero)."""
    A = torch.zeros(a_ext[0] + nb * a_off[0] + M, a_ext[1], dtype=torch.float64, device="cuda")
    A[:a_ext[0]] = a[:a_ext[0], :a_ext[1]].double()
    W = torch.zeros(w_ext[0] + nb * w_off[0] + N, w_ext[1], dtype=torch.float64, device="cuda")
    W[:w_ext[0]] = w[:w_ext[0], :w_ext[1]].double()
    out = []
    for b in range(nb):
        ab = A[b * a_off[0]:b * a_off[0] + M, b * a_off[1]:b * a_off[1] + K]
        wb = W[b * w_off[0]:b * w_off[0] + N, b * w_off[1]:b * w_off[1] + K]
        out.append(ab @ wb.t())
    return torch.stack(out)


def run_batched(ops, a, w, M, N, K, nb, a_off, w_off, c_stride, ldc, a_ext, w_ext, variant):
    """Launch into a sentinel buffer (16 padding columns per row and, for row-batched launches, 3 gap rows between batches). Returns the
    [nb, M, N] result and whether everything else kept its sentinel."""
    ldc_p = ldc + 16
    row_batched = a_off[0] > 0
    cs = (M + 3) * ldc_p if row_batched else c_stride
    rows = (nb - 1) * cs // ldc_p + M + 1
    raw = torch.full((rows * ldc_p,), SENTINEL16, dtype=torch.int16, device="cuda")
    c = raw.view(torch.bfloat16).view(rows, ldc_p)
    ops.gemm_batched(a, w, c, M, N, K, nb, a_off, w_off, cs, a_ext, w_ext, variant)
    idx = (torch.arange(nb, device="cuda")[:, None, None] * cs + torch.arange(M, device="cuda")[None, :, None] * ldc_p
           + torch.arange(N, device="cuda")[None, None, :])
    written = torch.zeros(raw.numel(), dtype=torch.bool, device="cuda")
    written[idx.flatten()] = True
    return raw.view(torch.bfloat16)[idx], bool((raw[~written] == SENTINEL16).all())


@pytest.mark.parametrize("B,T,S,H,Dm", [(3, 1, 605, 64, 4096), (2, 2, 611, 64, 4096), (5, 2, 37, 4, 256), (4, 1, 22, 4, 256)])
def test_batched_absorbed_specs_exact(ops, B, T, S, H, Dm):
    """The absorbed cross-attention's four launches (K-batched and row-batched), bit-exact, gaps and padding untouched."""
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + S)
    for name, M, N, K, nb, a_off, w_off, c_stride, ldc, a_ext, w_ext, variant in absorbed_specs(B, T, S, H, Dm):
        a = nan_padded(torch.randint(-3, 4, a_ext, device="cuda", generator=g).bfloat16(), pad_cols=8, pad_rows=64)
        w = nan_padded((torch.randint(-3, 4, w_ext, device="cuda", generator=g).float() / 32).bfloat16(), pad_cols=8, pad_rows=64)
        got, untouched = run_batched(ops, a, w, M, N, K, nb, a_off, w_off, c_stride, ldc, a_ext, w_ext, variant)
        assert untouched, name
        ref = batched_reference(a, w, M, N, K, nb, a_off, w_off, a_ext, w_ext).float().bfloat16()
        assert same_bits(got, ref), name


# K tails in batched launches: the k blocks are clipped only at the extents, so the launch is accepted when A's or W's extent ends at K
# (its tail reads zero fill); the other operand holds real, finite columns past K inside its extent, which must add nothing.
K_TAIL_SPECS = [
    # (name, M, N, K, nb, a_off, w_off, a_ext, w_ext, variant)
    ("one batch, A extent at K", 200, 328, 72, 1, (0, 0), (0, 0), (200, 72), (328, 136), 1281),
    ("W offset along K, A extent at K", 150, 200, 200, 3, (0, 0), (0, 200), (150, 200), (200, 664), 641),
    ("row-batched, W extent at K", 70, 136, 584, 3, (70, 0), (136, 0), (210, 640), (408, 584), 2561),
]


@pytest.mark.parametrize("spec", K_TAIL_SPECS, ids=[s[0] for s in K_TAIL_SPECS])
def test_batched_k_tail_exact(ops, spec):
    name, M, N, K, nb, a_off, w_off, a_ext, w_ext, variant = spec
    assert K % 64 != 0 and (a_ext[1] == K) != (w_ext[1] == K)
    g = torch.Generator(device="cuda").manual_seed(K + nb)
    a = nan_padded(torch.randint(-3, 4, a_ext, device="cuda", generator=g).bfloat16(), pad_cols=8, pad_rows=64)
    w = nan_padded((torch.randint(-3, 4, w_ext, device="cuda", generator=g).float() / 32).bfloat16(), pad_cols=8, pad_rows=64)
    ldc = N if a_off[0] > 0 else nb * N
    got, untouched = run_batched(ops, a, w, M, N, K, nb, a_off, w_off, N, ldc, a_ext, w_ext, variant)
    assert untouched, name
    assert same_bits(got, batched_reference(a, w, M, N, K, nb, a_off, w_off, a_ext, w_ext).float().bfloat16()), name


@pytest.mark.parametrize("variant", VARIANTS + [0])
@pytest.mark.parametrize("group_in,group_out,groups", [(80, 128, 9), (48, 64, 7)])
def test_grouped_scatter_exact(ops, variant, group_in, group_out, groups):
    """Logical column c lands at (c / group_in) * group_out + c % group_in; slot padding, row padding and rows past M keep their sentinel."""
    M, K = 700, 264
    N = groups * group_in
    g = torch.Generator(device="cuda").manual_seed(group_in + variant)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    out = Sentinel(M, groups * group_out, ld=groups * group_out + 8)
    grouped(a, w, out.t, bias, group_in, group_out, variant)
    ref = ref_store(exact_acc(a, w), bias).view(M, groups, group_in)
    slots = out.t.view(M, groups, group_out)
    assert same_bits(slots[..., :group_in].contiguous(), ref)
    assert bool((bits(slots[..., group_in:]) == SENTINEL16).all()), "slot padding written"
    assert out.untouched_outside()


def ssq_slots(c, block_n):
    """fp64 [M, parts] sums of squares of the stored bf16 values, one per (N tile, 32-column half of each staged slice)."""
    M, N = c.shape
    epi_cols = 64 if block_n >= 64 else 32
    n_tiles = -(-N // block_n)
    x = torch.zeros(M, n_tiles * block_n, dtype=torch.float64, device="cuda")
    x[:, :N] = c.double() ** 2
    return x.view(M, n_tiles, block_n // epi_cols, epi_cols // 32, 32).sum(dim=(2, 4)).reshape(M, -1)


@pytest.mark.parametrize("M,N", [(333, 1000), (333, 2056), (100, 1000), (100, 5000), (4500, 1000)])
def test_normfuse_producer_exact(ops, M, N):
    """The residual-writing GEMM of the fused RMSNorm: C = residual + bf16(acc) bit-exact, `parts` as ssq_parts_for, every slot the fp64 sum
    of squares of its stored 32-column halves within the fp32 rounding of that sum, the slots past `parts` still zero."""
    K = 1096
    variant = pick_variant(M, N)
    bn = BLOCK_N[variant]
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    res = nan_padded(rand_bf16((M, N), g), pad_cols=40, pad_rows=0)
    expect_parts = -(-N // bn) * (2 if bn >= 64 else 1)
    stride = (expect_parts + 12 + 3) // 4 * 4
    ssq = torch.zeros(M, stride, device="cuda")
    out = Sentinel(M, N, ld=N + 24)
    _, parts = ops.gemm_normfuse(a, w, residual=res, ssq_out=ssq, norm_dim=N, out=out.t)
    assert parts == expect_parts, (parts, expect_parts, variant)
    assert same_bits(out.t, ref_store(exact_acc(a, w), None, res))
    assert out.untouched_outside()
    ref = ssq_slots(out.t, bn)
    terms = bn // 2 if bn >= 64 else bn      # values summed into one slot
    tol = terms * 2.0 ** -24 * ref + 1e-30
    assert bool(((ssq[:, :parts].double() - ref).abs() <= tol).all()), float((ssq[:, :parts].double() - ref).abs().max())
    assert bool((ssq[:, parts:] == 0).all())


# ================================================================================================ C. tile order
def sched_n(block_n, extra):
    """N with 11 tiles of block_n columns, the last one ragged by `extra` columns."""
    return 10 * block_n + extra


@pytest.mark.parametrize("variant", VARIANTS)
def test_schedules_store_residual(ops, schedule, variant):
    bn = BLOCK_N[variant]
    M, N, K = SCHED_M, sched_n(bn, 72 if bn > 72 else 24), 264
    g = torch.Generator(device="cuda").manual_seed(variant + 3)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    res = rand_bf16((M, N), g)
    ref = ref_store(exact_acc(a, w), bias, res)
    schedule(0, 0)
    base = ops.gemm(a, w, bias=bias, residual=res, variant=variant)
    assert same_bits(base, ref)
    for s in SCHEDULES:
        schedule(*schedule_rows(s, bn))
        out = Sentinel(M, N, ld=N + 8)
        ops.gemm(a, w, bias=bias, residual=res, variant=variant, out=out.t)
        assert same_bits(out.t, base), s
        assert out.untouched_outside(), s


@pytest.mark.parametrize("variant", [2561, 1281, 641])
@pytest.mark.parametrize("epi", GATED)
def test_schedules_gated(ops, schedule, epi, variant):
    """The gated tile holds BLOCK_N / 2 gate and BLOCK_N / 2 up rows (gate_up_offset apart); a chunk still counts BLOCK_N W rows per tile."""
    bn = BLOCK_N[variant]
    M, K = SCHED_M, 264
    n_out = 5 * bn + 24                      # 2 * n_out = 10 * bn + 48: 11 tiles
    g = torch.Generator(device="cuda").manual_seed(variant + len(epi))
    a, w = exact_a(M, K, g), exact_w(2 * n_out, K, g)
    bias = rand_bf16((2 * n_out,), g, 0.5)
    schedule(0, 0)
    base = ops.gemm(a, w, bias=bias, epilogue=epi, variant=variant, gate_up_offset=n_out)
    check_activation(base, ref_activation(exact_acc(a, w), bias, epi, n_out))
    for s in SCHEDULES:
        schedule(*schedule_rows(s, bn))
        out = ops.gemm(a, w, bias=bias, epilogue=epi, variant=variant, gate_up_offset=n_out)
        assert same_bits(out, base), s


@pytest.mark.parametrize("variant", [2561, 1281, 321])
def test_schedules_f32acc(ops, schedule, variant):
    bn = BLOCK_N[variant]
    M, N, K = SCHED_M, sched_n(bn, 24), 264
    g = torch.Generator(device="cuda").manual_seed(variant + 4)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    c_in = residual_stream(M, N, g)
    ref = ref_f32acc(exact_acc(a, w), c_in, bias)
    for s in [(0, 0)] + SCHEDULES:
        schedule(*(schedule_rows(s, bn) if s != (0, 0) else s))
        out = Sentinel(M, N, ld=N + 8, dtype=torch.float32)
        out.t.copy_(c_in)
        ops.gemm_f32acc(a, w, out.t, bias=bias, variant=variant)
        assert same_bits(out.t, ref), s
        assert out.untouched_outside(), s


@pytest.mark.parametrize("variant", [2561, 1281])
def test_schedules_batched(ops, schedule, variant):
    """Three row-batched GEMMs of 23 x 11 tiles in one launch: the tile walk restarts in every batch."""
    bn = BLOCK_N[variant]
    nb, M, N, K = 3, SCHED_M, sched_n(bn, 24), 264
    g = torch.Generator(device="cuda").manual_seed(variant + 5)
    a = nan_padded(torch.randint(-3, 4, (nb * M, K), device="cuda", generator=g).bfloat16(), pad_cols=8, pad_rows=64)
    w = nan_padded((torch.randint(-3, 4, (nb * N, K), device="cuda", generator=g).float() / 32).bfloat16(), pad_cols=8, pad_rows=64)
    spec = (M, N, K, nb, (M, 0), (N, 0), 0, N, (nb * M, K), (nb * N, K), variant)     # row-batched: C stride chosen by run_batched
    ref = batched_reference(a, w, *spec[:6], *spec[8:10]).float().bfloat16()
    schedule(0, 0)
    base, untouched = run_batched(ops, a, w, *spec)
    assert untouched and same_bits(base, ref)
    for s in SCHEDULES:
        schedule(*schedule_rows(s, bn))
        got, untouched = run_batched(ops, a, w, *spec)
        assert untouched, s
        assert same_bits(got, base), s


def test_schedules_splitk(ops, schedule):
    """Split-K slices are the batches of one 128-wide launch: each slice walks the 11 N tiles in chunks."""
    M, N, K, splits = 100, sched_n(128, 72), 3072, 4
    g = torch.Generator(device="cuda").manual_seed(6)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    res = rand_bf16((M, N), g)
    ref = ref_store(exact_acc(a, w), bias, res)
    for s in [(0, 0)] + SCHEDULES:
        schedule(*(schedule_rows(s, 128) if s != (0, 0) else s))
        out = Sentinel(M, N, ld=N + 8)
        splitk(a, w, out.t, bias, res, splits)
        assert same_bits(out.t, ref), s
        assert out.untouched_outside(), s


def test_schedules_lmhead_logprob(ops, schedule):
    """EPI_LSE: per-(row, N tile) partials combined in tile order, so the log-probabilities must not depend on the walk."""
    M, N, K = SCHED_M, sched_n(128, 72), 256
    g = torch.Generator(device="cuda").manual_seed(7)
    h = rand_bf16((M, K), g)
    w = rand_bf16((N, K), g, K ** -0.5)
    labels = torch.randint(0, N, (M,), device="cuda", generator=g, dtype=torch.int32)
    schedule(0, 0)
    base = ops.lmhead_logprob(h, w, labels)
    assert bool(torch.isfinite(base).all())
    for s in SCHEDULES:
        schedule(*schedule_rows(s, 128))
        assert same_bits(ops.lmhead_logprob(h, w, labels), base), s


def test_auto_w_chunked_walk_short_last_chunk(ops, schedule):
    """A 25.7 MB weight (14..42 MB: W-stationary chunks) whose last chunk holds fewer N tiles, with a partial M group; the automatic order
    gives the reference bits and the bits of a one-chunk walk."""
    M, N, K = 5 * 128 + 37, 3592, 3584
    for variant in (2561, 1281):
        group_m, chunk_n, m_tiles, n_tiles = auto_schedule(N, K, M, N, BLOCK_N[variant])
        assert 1 < chunk_n < n_tiles and n_tiles % chunk_n != 0 and m_tiles % group_m != 0, (variant, chunk_n, n_tiles)
    g = torch.Generator(device="cuda").manual_seed(8)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    res = rand_bf16((M, N), g)
    ref = ref_store(exact_acc(a, w), bias, res)
    for variant in (2561, 1281):
        schedule(0, 0)
        auto = ops.gemm(a, w, bias=bias, residual=res, variant=variant)
        assert same_bits(auto, ref), variant
        schedule(1024, -1)
        assert same_bits(ops.gemm(a, w, bias=bias, residual=res, variant=variant), auto), variant


def test_auto_a_grouped_walk_ragged_last_group(ops, schedule):
    """A 64 MB weight (> 42 MB: A-stationary groups of 12 M tiles) over 31 M tiles, so the last group has 7; in-place residual."""
    M, N, K = 30 * 128 + 37, 8192, 4096
    group_m, chunk_n, m_tiles, n_tiles = auto_schedule(N, K, M, N, 256)
    assert pick_variant(M, N) == 2561 and chunk_n == n_tiles and group_m == 12 and m_tiles % group_m != 0
    schedule(0, 0)
    g = torch.Generator(device="cuda").manual_seed(9)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    out = Sentinel(M, N, ld=N + 8)
    out.t.copy_(rand_bf16((M, N), g))
    ref = ref_store(exact_acc(a, w), bias, out.t.clone())
    ops.gemm(a, w, bias=bias, residual=out.t, out=out.t)
    assert same_bits(out.t, ref)
    assert out.untouched_outside()


# ================================================================================================ D. activations
@pytest.mark.parametrize("epi", ACTIVATIONS)
def test_activation_bits_across_variants_schedules_and_rows(ops, schedule, epi):
    """Within two ulps of the reference; the same bits on every variant that has the epilogue, under every tile order, and for decode
    rows (M = 1, 7) on the automatic variant."""
    M, K, N = SCHED_M, 264, 2624              # N / 2 a multiple of 8 for the gated forms; ragged on every tile width
    gated = epi in GATED
    n_out = N // 2 if gated else N
    g = torch.Generator(device="cuda").manual_seed(len(epi) * 17)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5)
    kw = dict(bias=bias, epilogue=epi, gate_up_offset=n_out if gated else 0)
    schedule(0, 0)
    base = ops.gemm(a, w, variant=2561, **kw)
    check_activation(base, ref_activation(exact_acc(a, w), bias, epi, n_out))
    for variant in [2562, 1281, 1282, 641] + ([] if gated else [321]):
        out = Sentinel(M, n_out, ld=n_out + 8)
        ops.gemm(a, w, variant=variant, out=out.t, **kw)
        assert same_bits(out.t, base), variant
        assert out.untouched_outside(), variant
    for variant in (2561, 1281):
        for s in SCHEDULES:
            schedule(*schedule_rows(s, BLOCK_N[variant]))
            assert same_bits(ops.gemm(a, w, variant=variant, **kw), base), (variant, s)
    schedule(0, 0)
    for rows in (1, 7):
        out = Sentinel(rows, n_out, ld=n_out + 8)
        ops.gemm(a[:rows], w, variant=0, out=out.t, **kw)
        assert same_bits(out.t, base[:rows]), rows
        assert out.untouched_outside(), rows


# ================================================================================================ E. dependent launches (VQA_PDL=1)
def pdl_workload():
    """A chain of launches on one stream with no synchronisation between them, each consuming the previous one's output, then the tiny
    CLIP-FlanT5 and Qwen2.5-VL engines. Returns every output (on the CPU)."""
    import dataclasses
    from oracle import clipt5_oracle as orc
    from oracle import qwen25vl_oracle as qo
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.config import ClipT5Config, Qwen25VLConfig
    from t2v_metrics_b200.engine import ClipT5Engine, QwenVLEngine, fold_norm_gain
    from t2v_metrics_b200.engine import ops

    out = {"pdl_enabled": int(_lib.load().vqa_debug_pdl_enabled())}
    g = torch.Generator(device="cuda").manual_seed(11)
    B, S, H = 2, 200, 8
    D, F, Ms = H * 64, 1024, 100
    M = B * S
    x = rand_bf16((M, D), g)
    gamma = (1.0 + 0.1 * torch.randn(D, device="cuda", generator=g)).bfloat16()
    wqkv, wo, wp = rand_bf16((3 * D, D), g, D ** -0.5), rand_bf16((D, D), g, D ** -0.5), rand_bf16((D, D), g, D ** -0.5)
    wg = fold_norm_gain(rand_bf16((2 * F, D), g, D ** -0.5), gamma)
    wd, wc = rand_bf16((D, F), g, F ** -0.5), rand_bf16((D, D), g, D ** -0.5)
    bias = rand_bf16((D,), g, 0.1)
    ssq = torch.zeros(M, 64, device="cuda")
    y = torch.empty(Ms, D, dtype=torch.bfloat16, device="cuda")
    c32 = residual_stream(Ms, D, g)
    torch.cuda.synchronize()
    n = ops.norm(x, gamma)
    qkv = ops.gemm(n, wqkv)
    att = ops.attention(qkv, B, S, H, scale=0.125)
    ops.gemm(att, wo, residual=x, out=x)                         # in place over the stream the norm read
    x2, _ = ops.gemm_normfuse(x, wp, residual=x, ssq_out=ssq, norm_dim=D)
    h, _ = ops.gemm_normfuse(x2, wg, epilogue="gated_silu", gate_up_offset=F, ssq_in=ssq, norm_dim=D)
    splitk(h[:Ms], wd, y, bias, x2[:Ms], 4)
    ops.gemm_f32acc(y, wc, c32, bias=bias)
    torch.cuda.synchronize()
    out.update(norm=n, qkv=qkv, attention=att, x=x, x2=x2, ssq=ssq, h=h, splitk=y, f32acc=c32)

    ocfg = orc.ClipT5Config.tiny()
    label_ids = (37, 1)
    sd = orc.make_synthetic_state_dict(ocfg, seed=0, label_ids=label_ids)
    inp = orc.make_synthetic_inputs(ocfg, 3, 12, seed=1, ragged=True, label_ids=label_ids)
    orc.calibrate_lm_head(sd, ocfg, inp)
    eng = ClipT5Engine(ClipT5Config(**dataclasses.asdict(ocfg)), "cuda:0")
    eng.load_state_dict(sd)
    i32 = lambda t: t.to("cuda:0", torch.int32)
    args = [inp["pixels"].to("cuda:0"), i32(inp["input_ids"]), i32(inp["text_lens"]), i32(inp["labels"])]
    out["clipt5_score"] = eng.score_tensors(*args).clone()
    out["clipt5_score_graphed"] = eng.score_tensors_graphed(*args).clone()

    qcfg = qo.Qwen25VLConfig.tiny(hidden=256, heads=2, kv_heads=1, mrope_section=(16, 24, 24))
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    qeng = QwenVLEngine(Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(qcfg).items() if k in fields}), "cuda:0")
    qeng.load_state_dict(qo.make_synthetic_state_dict(qcfg, seed=0))
    qin = qo.make_synthetic_inputs(qcfg, 4, (84, 56), 12, ragged=True)
    out["qwen_score_prompts"] = qeng.score_prompts(qin["pixel_patches"], qin["grid_thw"], [t.tolist() for t in qin["input_ids"]],
                                                   qin["answer_ids"], qin["image_of_sample"]).clone()
    torch.cuda.synchronize()
    return {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in out.items()}


def test_pdl_launches_match_serial_launches(ops, tmp_path):
    """The same work in a child process with VQA_PDL=1 (read once per process): every output equal to this process's serial launches."""
    from t2v_metrics_b200 import _lib
    if _lib.load().vqa_debug_pdl_enabled():
        pytest.skip("this process already launches with PDL: nothing to compare against")
    path = tmp_path / "pdl.pt"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "pdl-child", str(path)]
    r = subprocess.run(cmd, env={**os.environ, "VQA_PDL": "1"}, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    child = torch.load(path, weights_only=False)
    serial = pdl_workload()
    assert child.pop("pdl_enabled") == 1 and serial.pop("pdl_enabled") == 0
    assert set(child) == set(serial)
    for k in serial:
        assert same_bits(child[k], serial[k]), k


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "pdl-child":
        sys.path.insert(0, ROOT)
        torch.save(pdl_workload(), sys.argv[2])
    else:
        sys.exit(f"usage: {sys.argv[0]} pdl-child <out.pt>")

"""The GEMM's TMA-store epilogue on a real H100, through the C ABI: every epilogue that writes dense bf16 C, on every tile variant, at ragged
M and N, with the output inside a sentinel-filled buffer whose rows are wider than the output (ldc > n_out) and which has rows past M.

Operands are small integers (A) and multiples of 1/32 (W), so the fp32 accumulator is exact whatever the summation order: the store and
ReLU epilogues are checked bit for bit against torch; the other activations, whose kernels use fast exponentials, within two bf16 ulps.
The in-place residual case walks many tiles per CTA, so the box buffers and their barriers are reused across tiles. The last group checks
that the TMA-store path and the staged path (which keeps the batched launches and the fused-RMSNorm partial sums) write the same bits."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL16 = 0x7FA5     # bf16 NaN bit pattern, distinct from the NaN arithmetic produces (0x7FC0)
EPILOGUES = ["store", "relu", "quick_gelu", "gelu", "gated_gelu", "gated_silu"]
GATED = ("gated_gelu", "gated_silu")
VARIANTS = [2561, 1281, 641, 321]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


def operands(M, N, K, g):
    a = torch.randint(-3, 4, (M, K), device="cuda", generator=g).bfloat16()
    w = (torch.randint(-3, 4, (N, K), device="cuda", generator=g).float() / 32).bfloat16()
    bias = (torch.randn(N, device="cuda", generator=g) * 0.5).bfloat16()
    return a, w, bias


class Sentinel:
    """A [rows, cols] bf16 output with row stride ld > cols inside a sentinel-filled [rows + extra_rows, ld] buffer."""

    def __init__(self, rows, cols, ld, extra_rows=3):
        self.rows, self.cols = rows, cols
        self.raw = torch.full((rows + extra_rows, ld), SENTINEL16, dtype=torch.int16, device="cuda")
        self.t = self.raw.view(torch.bfloat16)[:rows, :cols]

    def untouched_outside(self):
        mask = torch.ones_like(self.raw, dtype=torch.bool)
        mask[:self.rows, :self.cols] = False
        return bool((self.raw[mask] == SENTINEL16).all())


def bf16_ulp(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -100))) - 7)


def reference(a, w, bias, residual, epi, n_out):
    """fp32 arithmetic at the kernel's rounding points; the accumulator is exact for these operands."""
    acc = (a.double() @ w.double().T).float()
    b = bias.float() if bias is not None else torch.zeros(acc.shape[1], device="cuda")
    if epi in GATED:
        g = (acc[:, :n_out] + b[:n_out]).bfloat16().double()
        u = (acc[:, n_out:2 * n_out] + b[n_out:2 * n_out]).bfloat16().double()
        if epi == "gated_gelu":
            act = 0.5 * g * (1.0 + torch.tanh(0.7978845608028654 * (g + 0.044715 * g ** 3)))
        else:
            act = (g * torch.sigmoid(g)).float().bfloat16().double()
        return (act * u).float().bfloat16()
    y = (acc + b).bfloat16().float()
    if epi == "relu":
        y = y.clamp_min(0.0)
    elif epi == "gelu":
        y = (0.5 * y.double() * (1.0 + torch.erf(y.double() / 2 ** 0.5))).float()
    elif epi == "quick_gelu":
        s = (1.702 * y).bfloat16().double()
        y = (y.double() * torch.sigmoid(s).float().bfloat16().double()).float()
    if residual is not None:
        y = y + residual.float()
    return y.bfloat16()


def check(got, ref, epi):
    if epi in ("store", "relu"):
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), "not bit-identical"
    else:
        assert torch.isfinite(got.float()).all()
        err = (got.double() - ref.double()).abs()
        # the absolute term covers outputs near zero, where gelu_new's tanh = 1 - 2 / (exp(2u) + 1) cancels (|error| ~ 1e-6)
        tol = 2 * bf16_ulp(ref.double()) + 2.0 ** -16
        assert bool((err <= tol).all()), float((err - tol).max())


def run(ops, a, w, bias, epi, variant, out, residual=None):
    N = w.shape[0]
    return ops.gemm(a, w, bias=bias, residual=residual, epilogue=epi, variant=variant, out=out,
                    gate_up_offset=N // 2 if epi in GATED else 0)


# ragged M and n_out on every tile width: partial boxes in both directions, boxes wholly past M (M = 65 on a 128-row tile)
RAGGED = [(200, 328), (65, 40), (1000, 1000), (128, 256)]


@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("M,n_out", RAGGED)
def test_ragged_sentinel(ops, epi, variant, M, n_out):
    if epi in GATED and variant == 321:
        pytest.skip("the gated epilogue needs a tile of >= 64 columns")
    g = torch.Generator(device="cuda").manual_seed(M * 7 + n_out)
    N = 2 * n_out if epi in GATED else n_out
    a, w, bias = operands(M, N, 256, g)
    with_res = epi not in GATED
    out = Sentinel(M, n_out, ld=n_out + 24)
    res = None
    if with_res:   # its own row stride, different from C's
        rbuf = torch.randn(M, n_out + 40, device="cuda", generator=g).bfloat16()
        res = rbuf[:, :n_out]
    run(ops, a, w, bias, epi, variant, out.t, residual=res)
    torch.cuda.synchronize()
    check(out.t, reference(a, w, bias, res, epi, n_out), epi)
    assert out.untouched_outside(), "wrote outside [M, n_out]"


@pytest.mark.parametrize("variant", [2561, 1281])
def test_inplace_residual_many_tiles(ops, variant):
    """C = C + bf16(A W^T + bias) in place over 65 x 16 (or 32) tiles: each CTA reuses its box buffers across about eight tiles."""
    g = torch.Generator(device="cuda").manual_seed(5)
    M, N, K = 8192 + 37, 4096, 256
    a, w, bias = operands(M, N, K, g)
    out = Sentinel(M, N, ld=N + 8)
    out.t.copy_(torch.randn(M, N, device="cuda", generator=g).bfloat16())
    ref = reference(a, w, bias, out.t.clone(), "store", N)
    run(ops, a, w, bias, "store", variant, out.t, residual=out.t)
    torch.cuda.synchronize()
    check(out.t, ref, "store")
    assert out.untouched_outside()


@pytest.mark.parametrize("epi", GATED)
@pytest.mark.parametrize("M", [1, 7, 128])
@pytest.mark.parametrize("variant", [0, 2561, 1281, 641])
def test_gated_decode_rows(ops, epi, M, variant):
    g = torch.Generator(device="cuda").manual_seed(M)
    n_out = 1024
    a, w, bias = operands(M, 2 * n_out, 512, g)
    out = Sentinel(M, n_out, ld=n_out + 8)
    run(ops, a, w, bias, epi, variant, out.t)
    torch.cuda.synchronize()
    check(out.t, reference(a, w, bias, None, epi, n_out), epi)
    assert out.untouched_outside()


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("M,N,K", [(1000, 1000, 1024), (4096, 4096, 512)])
def test_tma_path_matches_staged_path(ops, variant, M, N, K):
    """Random operands (an inexact accumulator): the TMA-store epilogue writes the same bits as the staged one, which a batched launch of
    one batch (plain store) and a fused-norm launch with per-row sums of squares (residual store) keep."""
    g = torch.Generator(device="cuda").manual_seed(variant)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).bfloat16()
    tma = ops.gemm(a, w, variant=variant)
    staged = torch.empty_like(tma)
    ops.gemm_batched(a, w, staged, M, N, K, 1, variant=variant)
    torch.cuda.synchronize()
    assert torch.equal(tma.view(torch.int16), staged.view(torch.int16))
    if variant != 2561:   # the fused-norm launch picks its own tile; compare it once per shape
        return
    r = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    tma_r = ops.gemm(a, w, residual=r)
    ssq = torch.zeros(M, 256, device="cuda")
    staged_r, _ = ops.gemm_normfuse(a, w, residual=r, ssq_out=ssq, norm_dim=N)
    torch.cuda.synchronize()
    assert torch.equal(tma_r.view(torch.int16), staged_r.view(torch.int16))


def test_rejects_misaligned_output(ops):
    """TMA needs C on 16 bytes; a view 8 bytes into a buffer is refused, not written."""
    a = torch.ones(64, 64, device="cuda").bfloat16()
    w = torch.ones(64, 64, device="cuda").bfloat16()
    buf = torch.full((64 * 72 + 4,), SENTINEL16, dtype=torch.int16, device="cuda")
    out = buf[4:].view(torch.bfloat16)[:64 * 72].view(64, 72)[:, :64]
    with pytest.raises(RuntimeError):
        ops.gemm(a, w, out=out)
    torch.cuda.synchronize()
    assert bool((buf == SENTINEL16).all())

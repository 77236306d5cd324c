"""Kernel-level parity on a real H100, through the C ABI (vqa_op_*). Reference = plain PyTorch fp32 math of the same op
with the same bf16 rounding points."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


def ref_gemm(a, w, bias=None, residual=None, epilogue="store", gate_off=0):
    acc = a.float() @ w.float().t()
    if epilogue in ("gated_gelu", "gated_silu"):
        if bias is not None:            # [gate bias | up bias], gate_off apart like the weight rows
            acc = acc + bias.float()
        g = acc[:, :gate_off].bfloat16().float()
        u = acc[:, gate_off:].bfloat16().float()
        if epilogue == "gated_silu":    # Qwen2MLP: act_fn(gate_proj(x)) * up_proj(x), every op a bf16 tensor
            return (torch.nn.functional.silu(g).bfloat16().float() * u).bfloat16()
        return (torch.nn.functional.gelu(g, approximate="tanh").bfloat16().float() * u).bfloat16()
    if bias is not None:
        acc = acc + bias.float()
    y = acc.bfloat16().float()
    if epilogue == "quick_gelu":
        y = y * torch.sigmoid(1.702 * y)
    elif epilogue == "gelu":
        y = torch.nn.functional.gelu(y)
    elif epilogue == "relu":
        y = torch.relu(y)
    if residual is not None:
        y = y + residual.float()
    return y.bfloat16()


def close(c, ref, what):
    d = (c.float() - ref.float()).abs()
    bad = int((d > 0.02 + 0.01 * ref.float().abs()).sum())     # 1 bf16 ulp of slack on top of fp32 accumulation-order noise
    assert bad == 0, (what, bad, float(d.max()))


@pytest.mark.parametrize("variant", [2562, 2561, 1282, 1281, 641, 321, 0])
@pytest.mark.parametrize("shape", [(128, 256, 64), (512, 512, 512), (1000, 776, 1032), (300, 4096, 640)])
def test_gemm_store_bias_residual(ops, variant, shape):
    M, N, K = shape
    torch.manual_seed(1)
    a = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
    bias = (torch.randn(N, device="cuda") * 0.1).bfloat16()
    res = torch.randn(M, N, device="cuda").bfloat16()
    close(ops.gemm(a, w, variant=variant), ref_gemm(a, w), "plain")
    close(ops.gemm(a, w, bias=bias, residual=res, variant=variant), ref_gemm(a, w, bias, res), "bias+res")
    # in-place residual (the residual stream is updated in place by the engine)
    c = res.clone()
    ops.gemm(a, w, bias=bias, residual=c, variant=variant, out=c)
    close(c, ref_gemm(a, w, bias, res), "in-place residual")


@pytest.mark.parametrize("variant", [2562, 2561, 1281, 641, 0])
@pytest.mark.parametrize("epi", ["quick_gelu", "gelu", "relu", "gated_gelu", "gated_silu"])
def test_gemm_fused_epilogues(ops, variant, epi):
    torch.manual_seed(2)
    M, N, K = 700, 1024, 512
    a = (torch.randn(M, K, device="cuda")).bfloat16()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
    bias = None if epi == "gated_gelu" else (torch.randn(N, device="cuda") * 0.1).bfloat16()
    c = ops.gemm(a, w, bias=bias, epilogue=epi, variant=variant, gate_up_offset=N // 2)
    close(c, ref_gemm(a, w, bias, None, epi, N // 2), epi)


@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("M", [1, 7, 128])
def test_gemm_gated_silu_decode_rows(ops, M, with_bias):
    """The gated-SiLU GEMM at decode-step row counts (M = B <= 128) with the padded vision-MLP width (2 x 3456, up block 3456 rows below
    the gate block) and the tower's gate / up biases."""
    torch.manual_seed(13)
    N, K = 2 * 3456, 1280
    a = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
    bias = (torch.randn(N, device="cuda") * 0.5).bfloat16() if with_bias else None
    c = ops.gemm(a, w, bias=bias, epilogue="gated_silu", gate_up_offset=N // 2)
    assert c.shape == (M, N // 2)
    ref = ref_gemm(a, w, bias, None, "gated_silu", N // 2)
    close(c, ref, (M, with_bias))
    if with_bias:       # the bias does move the result: a kernel that dropped it (or read the up bias at the gate offset) would fail
        assert float((ref_gemm(a, w, None, None, "gated_silu", N // 2).float() - ref.float()).abs().max()) > 0.5


@pytest.mark.parametrize("M,N,K,splits", [(128, 4096, 4096, 0), (2, 4096, 10240, 0), (100, 1024, 2048, 4), (7, 512, 4096, 8)])
def test_gemm_split_k_for_decoder_rows(ops, M, N, K, splits):
    """Skinny store-GEMM with K cut into slices (one launch, fp32 partials, one reduction): C = residual + bf16(A W^T + bias), the same rounding
    points as the plain epilogue, so it must agree with it to the last bit of the bf16 sum order."""
    import ctypes as C
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _ptr, _stream_ptr, _check
    lib = _lib.load()
    torch.manual_seed(12)
    a = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
    bias = (torch.randn(N, device="cuda") * 0.1).bfloat16()
    res = torch.randn(M, N, device="cuda").bfloat16()
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(8 * M * N, dtype=torch.float32, device="cuda")
    used = C.c_int32(0)
    _check(lib.vqa_op_gemm_bf16_splitk(_ptr(a), K, _ptr(w), K, N, _ptr(out), N, M, N, K, _ptr(bias), _ptr(res), N, splits, _ptr(ws), ws.numel() * 4,
                                       C.byref(used), _stream_ptr(a.device)), None, "vqa_op_gemm_bf16_splitk")
    torch.cuda.synchronize()
    assert used.value >= 2, used.value          # every case here is meant to split
    plain = ops.gemm(a, w, bias=bias, residual=res)
    close(out, ref_gemm(a, w, bias, res, "store", 0), (M, N, K, used.value))
    assert float((out.float() - plain.float()).abs().max()) <= 0.0625          # one bf16 ulp of the rounded Linear output at |y| <= 8


def test_gemm_empty_and_ragged_edges(ops):
    torch.manual_seed(3)
    for (M, N, K) in [(1, 8, 8), (129, 264, 72), (257, 40, 200)]:
        a = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
        for variant in (0, 2562, 321):
            close(ops.gemm(a, w, variant=variant), ref_gemm(a, w), (M, N, K, variant))


def test_gemm_linearity_full_size(ops):
    """Size-independent property at the BASELINE shape (M = 64*672): GEMM(a1 + a2) == GEMM(a1) + GEMM(a2) up to rounding,
    and a checksum against cuBLAS via torch.matmul."""
    torch.manual_seed(4)
    M, N, K = 43008, 4096, 4096
    a = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
    c = ops.gemm(a, w)
    ref = torch.matmul(a, w.t())
    d = (c.float() - ref.float()).abs()
    assert float(d.max()) <= 0.0625 and float(d.mean()) < 1e-3
    assert abs(float(c.float().sum()) - float(ref.float().sum())) <= 1e-3 * float(ref.float().abs().sum()) ** 0.5 + 50


@pytest.mark.parametrize("M,D,N", [(700, 4096, 4096), (300, 256, 256), (130, 2048, 512)])
def test_gemm_fused_rmsnorm_hooks(ops, M, D, N):
    """north_star: 'RMSNorm ... fused into the adjacent matmul epilogue'. Producer: a residual GEMM leaves per-row partial sums of squares of
    the bf16 rows it stores. Consumer: GEMM on the UN-normalised rows with gamma folded into W, accumulator rows scaled by rsqrt(mean(x^2)+eps)
    == the Linear applied to T5LayerNorm(x) (modeling_t5.py:55-68) up to where the bf16 roundings sit."""
    from t2v_metrics_b200.engine import fold_norm_gain
    torch.manual_seed(8)
    a = (torch.randn(M, 512, device="cuda") * 0.5).bfloat16()
    wo = (torch.randn(D, 512, device="cuda") * 512 ** -0.5).bfloat16()
    res = (torch.randn(M, D, device="cuda") * 3.0).bfloat16()
    stride = (D // 32 + 3) // 4 * 4
    ssq = torch.zeros(M, stride, dtype=torch.float32, device="cuda")
    x, parts = ops.gemm_normfuse(a, wo, residual=res, ssq_out=ssq, norm_dim=D)
    ref_x = ((a.float() @ wo.float().t()).bfloat16().float() + res.float()).bfloat16()
    assert float((x.float() - ref_x.float()).abs().max()) <= 0.07
    assert 1 <= parts <= stride and bool((ssq[:, parts:] == 0).all())
    tot = ssq.sum(-1)
    assert float(((tot - x.float().pow(2).sum(-1)).abs() / tot).max()) < 1e-5          # exactly the rows that were stored
    # consumer: plain and gated
    gamma = (1 + 0.1 * torch.randn(D, device="cuda")).bfloat16()
    w = (torch.randn(N, D, device="cuda") * D ** -0.5).bfloat16()
    y, _ = ops.gemm_normfuse(x, fold_norm_gain(w, gamma), ssq_in=ssq, norm_dim=D, eps=1e-6)
    var = x.float().pow(2).mean(-1, keepdim=True)
    xn = (gamma.float() * (x.float() * torch.rsqrt(var + 1e-6)).bfloat16().float()).bfloat16()
    ref_y = (xn.float() @ w.float().t())
    err = (y.float() - ref_y).abs()
    assert float(err.max()) <= 0.05 * float(ref_y.abs().max()) and float(err.mean()) <= 6e-3 * float(ref_y.abs().mean()) + 2e-3
    wg = (torch.randn(2 * N, D, device="cuda") * D ** -0.5).bfloat16()
    h, _ = ops.gemm_normfuse(x, fold_norm_gain(wg, gamma), epilogue="gated_gelu", gate_up_offset=N, ssq_in=ssq, norm_dim=D, eps=1e-6)
    g_, u_ = (xn.float() @ wg[:N].float().t()).bfloat16().float(), (xn.float() @ wg[N:].float().t()).bfloat16().float()
    ref_h = torch.nn.functional.gelu(g_, approximate="tanh") * u_
    assert float((h.float() - ref_h).abs().mean()) <= 1e-2 * float(ref_h.abs().mean()) + 2e-3


def test_rmsnorm(ops):
    torch.manual_seed(6)
    for D in (4096, 3584, 2048, 1280, 256, 128, 5120):   # warp-per-row (D % 256 == 0, <= 4096) and the generic block-per-row path
        x = torch.randn(333, D, device="cuda").bfloat16()
        g = (1 + 0.1 * torch.randn(D, device="cuda")).bfloat16()
        var = x.float().pow(2).mean(-1, keepdim=True)
        ref = (g.float() * (x.float() * torch.rsqrt(var + 1e-6)).bfloat16().float()).bfloat16()
        assert float((ops.norm(x, g, 1e-6).float() - ref.float()).abs().max()) <= 0.016


def test_lmhead_logprob_never_materialises_logits(ops):
    torch.manual_seed(7)
    for (M, N, K) in [(128, 32128, 512), (6, 1000, 256), (2, 130, 64)]:
        h = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * K ** -0.5 * 3).bfloat16()
        labels = torch.randint(0, N, (M,), device="cuda", dtype=torch.int32)
        labels[0] = N - 1
        lp = ops.lmhead_logprob(h, w, labels)
        logits = (h.float() @ w.float().t()).bfloat16().float()
        ref = torch.log_softmax(logits, -1).gather(-1, labels.long()[:, None])[:, 0]
        assert float((lp - ref).abs().max()) < 5e-3

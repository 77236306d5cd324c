"""The Qwen2.5-VL-3B shapes on a real H100, at kernel level: the head-dim-128 prefill attention at 8 query heads per K/V head (16 / 2
heads: causal with ragged lengths around the 128-row tiles and at 448x448 prompt lengths, and the shared-prefix layout) against fp64
torch, and the language model's GEMMs at 2048 width (qkv N = 2560, o / down N = 2048, gate_up N = 2 x 11008; K = 2048 / 11008) in the
bit-exact harness of test_gpu_gemm_exact.py, with the decode step's split-K at the slice counts splitk_slices() picks for them."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_gemm_exact import Sentinel, exact_a, exact_acc, exact_w, nan_padded, rand_bf16, ref_activation, ref_store, same_bits, \
    check_activation
from test_gpu_qwen_kernels import assert_attn, assert_guards, attn_ref, guarded, make_qkv, split_heads

HQ, HKV = 16, 2
D, MLP, QKV = 2048, 11008, (HQ + 2 * HKV) * 128


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


# ------------------------------------------------------------------------------------------------ prefill attention, kv_group = 8
@pytest.mark.parametrize("S,lens", [(320, [320, 1, 257, 129]), (330, [330, 300, 17]), (1100, [1100, 1023])])
def test_attention_causal_group8(ops, S, lens):
    """Fixed-stride causal launch over padded rows: every query head h reads K/V head h // 8; padded rows zero, guards untouched."""
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(S + 8)
    n = len(lens)
    qkv, L = make_qkv(n * S, HQ, HKV, dev, gen)
    big, out = guarded(n * S, HQ * 128, dev)
    ops.attention_d128(qkv, out, L["q0"], L["k0"], L["v0"], n, S, HQ, HQ // HKV, 128 ** -0.5, True, S=S,
                       seq_lens=torch.tensor(lens, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    assert_guards(big, n * S, HQ * 128, what="output")
    for b, ln in enumerate(lens):
        r = slice(b * S, b * S + ln)
        q, k, v = split_heads(qkv, r, HQ, HKV, L)
        ref, ref_p = attn_ref(q, k, v, 128 ** -0.5, True)
        tol = assert_attn(out[r].view(ln, HQ, 128).transpose(0, 1), ref, ref_p, f"sequence {b}")
        assert bool((out[b * S + ln:(b + 1) * S] == 0).all())
        if b == 0:
            # the fixture tells K/V head h // 8 from h % 2
            kv_h = torch.arange(HQ, device=dev) % HKV
            kk = qkv[r, L["k0"]:L["k0"] + HKV * 128].view(ln, HKV, 128).transpose(0, 1)[kv_h]
            vv = qkv[r, L["v0"]:L["v0"] + HKV * 128].view(ln, HKV, 128).transpose(0, 1)[kv_h]
            assert bool(((attn_ref(q, kk, vv, 128 ** -0.5, True)[0] - ref).abs() > 4 * tol).any())


@pytest.mark.parametrize("pre_len", [17, 128, 300])
def test_attention_kv_prefix_group8(ops, pre_len):
    """Shared-prefix layout: three suffixes over one prefix next to a prefix-less sequence, against fp64 attention over [prefix | suffix]."""
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(pre_len + 80)
    lens = [pre_len, 1, 77, 200, 150]
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    qkv, L = make_qkv(cu[-1], HQ, HKV, dev, gen)
    big, out = guarded(cu[-1], HQ * 128, dev)
    ops.attention_d128(qkv, out, L["q0"], L["k0"], L["v0"], len(lens), max(lens), HQ, HQ // HKV, 128 ** -0.5, True,
                       cu_seqlens=torch.tensor(cu, dtype=torch.int32, device=dev),
                       kv_prefix=torch.tensor([-1, 0, 0, 0, -1], dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    assert_guards(big, cu[-1], HQ * 128, what="output")
    kp, vp = split_heads(qkv, slice(0, pre_len), HQ, HKV, L)[1:]
    for sq in range(len(lens)):
        q, k, v = split_heads(qkv, slice(cu[sq], cu[sq + 1]), HQ, HKV, L)
        if 1 <= sq <= 3:
            ref, ref_p = attn_ref(q, torch.cat([kp, k], 1), torch.cat([vp, v], 1), 128 ** -0.5, True, q_off=pre_len)
        else:
            ref, ref_p = attn_ref(q, k, v, 128 ** -0.5, True)
        assert_attn(out[cu[sq]:cu[sq + 1]].view(-1, HQ, 128).transpose(0, 1), ref, ref_p, f"sequence {sq}")


# ------------------------------------------------------------------------------------------------ GEMMs at 2048 width, bit for bit
def splitk_auto(a, w, out, bias, residual):
    """vqa_op_gemm_bf16_splitk with splits = 0: the slice count splitk_slices() picks (returned)."""
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _check, _ptr, _stream_ptr
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    ws = torch.empty(8 * M * N, dtype=torch.float32, device="cuda")
    used = C.c_int32(0)
    _check(lib.vqa_op_gemm_bf16_splitk(_ptr(a), a.stride(0), _ptr(w), w.stride(0), N, _ptr(out), out.stride(0), M, N, K, _ptr(bias),
                                       _ptr(residual), residual.stride(0) if residual is not None else 0, 0, _ptr(ws), ws.numel() * 4,
                                       C.byref(used), _stream_ptr(a.device)), None, "vqa_op_gemm_bf16_splitk")
    return used.value


def expected_slices(M, N, K, nsm):
    """host.cuh splitk_slices, restated so that a change of the rule at these shapes is seen here."""
    if M > 128 or N % 8 or K < 2048:
        return 1
    s = min(nsm // ((N + 127) // 128), 8)
    while s >= 2 and K % (s * 64):
        s -= 1
    return s if s >= 2 else 1


# (name, N, K, bias, residual): the decode step's split launches
DECODE = [("qkv", QKV, D, True, False), ("o", D, HQ * 128, False, True), ("down", D, MLP, False, True)]


@pytest.mark.parametrize("M", [1, 8, 32])
@pytest.mark.parametrize("name,N,K,has_bias,has_res", DECODE, ids=[d[0] for d in DECODE])
def test_decode_splitk_at_3b_shapes_exact(ops, M, name, N, K, has_bias, has_res):
    """The decode GEMMs at 3B width with the automatic slice count: on 132 SMs qkv (20 N tiles) 4, o (16) 8, down (16, K = 11008) 4 slices;
    the bits are the reference's and the unsplit GEMM's, and slices x M x N fits the step's workspace of 8 x M x max(qkv cols, hidden)."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N + K)
    a, w = exact_a(M, K, g), exact_w(N, K, g)
    bias = rand_bf16((N,), g, 0.5) if has_bias else None
    res = nan_padded(rand_bf16((M, N), g), pad_cols=40, pad_rows=0) if has_res else None
    out = Sentinel(M, N, ld=N + 24)
    s = splitk_auto(a, w, out.t, bias, res)
    print(f"\n[3b decode {name}] M={M} N={N} K={K}: {s} slices on {nsm} SMs")
    assert s == expected_slices(M, N, K, nsm)
    if nsm == 132:
        assert s == {"qkv": 4, "o": 8, "down": 4}[name]
    assert s * M * N <= 8 * M * max(QKV, D)
    assert out.untouched_outside()
    assert same_bits(out.t, ref_store(exact_acc(a, w), bias, res))
    assert same_bits(out.t, ops.gemm(a, w, bias=bias, residual=res))


@pytest.mark.parametrize("M", [1, 32, 330, 2 * 330])
def test_prefill_gemms_at_3b_shapes_exact(ops, M):
    """The prefill / decode launches without split-K at 3B width: qkv with bias, o and down with the residual (K = 2048 / 11008),
    gate_up with the fused SiLU gate (N = 2 x 11008), every one on the tile variant the host picks."""
    g = torch.Generator(device="cuda").manual_seed(M + 3)
    for N, K, kind in ((QKV, D, "bias"), (D, HQ * 128, "res"), (D, MLP, "res")):
        a, w = exact_a(M, K, g), exact_w(N, K, g)
        bias = rand_bf16((N,), g, 0.5) if kind == "bias" else None
        res = rand_bf16((M, N), g) if kind == "res" else None
        out = Sentinel(M, N, ld=N + 8)
        ops.gemm(a, w, bias=bias, residual=res, out=out.t)
        assert out.untouched_outside(), (N, K)
        assert same_bits(out.t, ref_store(exact_acc(a, w), bias, res)), (N, K)
    a, w = exact_a(M, D, g), exact_w(2 * MLP, D, g)
    bias = torch.zeros(2 * MLP, dtype=torch.bfloat16, device="cuda")
    got = ops.gemm(a, w, epilogue="gated_silu", gate_up_offset=MLP)
    check_activation(got, ref_activation(exact_acc(a, w), bias, "gated_silu", MLP))

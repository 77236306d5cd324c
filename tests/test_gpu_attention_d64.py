"""Head-dim-64 attention (attn64_ws_kernel: persistent, warp-specialised) against an fp64 torch reference, through the C ABI.

Covers the production shapes (T5 encoder S = 672, H = 64; CLIP S = 577, H = 16) in both rounding modes with ragged lengths whose last key
tile has every width the kernel special-cases, the constant-bias fast path, a persistent launch with many more work items than CTAs, and
guard bands around the output."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# len mod 128 = 1, 16, 17, 32, 64, 65, 127, 0. 576 / 513 leave the second 64-row block of the last query tile all padding, 512 / 640 / 1
# leave whole 128-row query tiles (both blocks) padding.
T5_LEN_PAIRS = [(672, 1), (656, 17), (576, 65), (639, 640), (513, 16), (512, 129), (192, 127)]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


def saturating_table(H, S, dist=128, seed=0, mult=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rel = torch.arange(-(S - 1), S, device="cuda").clamp(-dist, dist) + dist
    return (torch.randn(H, 2 * dist + 1, device="cuda", generator=g) * mult).bfloat16().float()[:, rel].contiguous()


def reference(qkv, B, S, H, lens, table, scale, round_scores):
    """fp64 attention with the kernel's rounding points when round_scores: bf16(bf16(q k^T) + bf16(bias)) * scale, P rounded to bf16."""
    q, k, v = qkv.double().view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = torch.matmul(q, k.transpose(-1, -2))
    idx = (torch.arange(S, device="cuda")[None, :] - torch.arange(S, device="cuda")[:, None]) + S - 1
    bias = table.double()[:, idx][None] if table is not None else None
    if round_scores:
        s = s.bfloat16().double()
        if bias is not None:
            s = (s + bias.bfloat16().double()).bfloat16().double()
        s = s * scale
    else:
        s = s * scale + (bias if bias is not None else 0.0)
    kmask = torch.arange(S, device="cuda")[None, :] < lens[:, None]
    s = s.masked_fill(~kmask[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1).nan_to_num(0.0)
    if round_scores:
        p = p.bfloat16().double()
    out = torch.matmul(p, v).permute(0, 2, 1, 3).reshape(B * S, H * 64)
    return out, kmask.reshape(B * S)


def check_rows(out, ref, qmask, tol):
    err = (out[qmask].double() - ref[qmask]).abs().max()
    assert float(err) < tol, float(err)
    pad = out[~qmask]
    assert pad.numel() == 0 or bool((pad.view(torch.int16) == 0).all()), "padded query rows must be +0"


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("lens_pair", T5_LEN_PAIRS)
def test_t5_shape_ragged_tails(ops, lens_pair, round_scores):
    torch.manual_seed(1)
    B, S, H = 2, 672, 64
    qkv = (torch.randn(B * S, 3 * H * 64, device="cuda") * 0.5).bfloat16()
    table = saturating_table(H, S)
    lens = torch.tensor(lens_pair, device="cuda", dtype=torch.int32)
    out = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=table, scale=1.0, bias_const_from=128, round_scores=round_scores)
    ref, qmask = reference(qkv, B, S, H, lens, table, 1.0, round_scores)
    check_rows(out, ref, qmask, 0.03)


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("lens_pair", [None, (577, 449), (513, 65), (576, 32)])
def test_clip_shape(ops, lens_pair, round_scores):
    torch.manual_seed(2)
    B, S, H = 2, 577, 16
    qkv = torch.randn(B * S, 3 * H * 64, device="cuda").bfloat16()
    lens = torch.tensor(lens_pair, device="cuda", dtype=torch.int32) if lens_pair else None
    out = ops.attention(qkv, B, S, H, seq_lens=lens, scale=0.125, round_scores=round_scores)
    L = lens if lens is not None else torch.full((B,), S, device="cuda", dtype=torch.int32)
    ref, qmask = reference(qkv, B, S, H, L, None, 0.125, round_scores)
    check_rows(out, ref, qmask, 0.03)


@pytest.mark.parametrize("round_scores", [False, True])
def test_constant_bias_fast_path_is_exact(ops, round_scores):
    """A table that is constant past distance 128 gives bit-identical output whether the kernel is told so (and skips the per-score
    lookups of far tiles) or not. A table that breaks the promise does give a different output under the promise, so the comparison
    does see the fast path."""
    torch.manual_seed(3)
    B, S, H = 2, 672, 8
    qkv = (torch.randn(B * S, 3 * H * 64, device="cuda") * 0.5).bfloat16()
    lens = torch.tensor([672, 600], device="cuda", dtype=torch.int32)
    table = saturating_table(H, S, mult=2.0)
    fast = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=table, scale=1.0, bias_const_from=128, round_scores=round_scores)
    slow = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=table, scale=1.0, bias_const_from=0, round_scores=round_scores)
    assert torch.equal(fast.view(torch.int16), slow.view(torch.int16))

    broken = table.clone()
    far = torch.arange(2 * S - 1, device="cuda") - (S - 1)
    broken[:, far.abs() >= 200] += 3.0 * torch.sin(far[far.abs() >= 200].float())[None]       # no longer constant past 128
    fast_b = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=broken, scale=1.0, bias_const_from=128, round_scores=round_scores)
    slow_b = ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=broken, scale=1.0, bias_const_from=0, round_scores=round_scores)
    assert not torch.equal(fast_b, slow_b)
    ref, qmask = reference(qkv, B, S, H, lens, broken, 1.0, round_scores)
    check_rows(slow_b, ref, qmask, 0.03)


def test_persistent_schedule_every_row_and_guard_bands(ops):
    """40 samples x 8 heads x 6 query tiles = 1920 work items, far more than one CTA per SM, with lengths from 0 to S: every output
    row is checked, and guard bands on both sides of the output buffer stay untouched."""
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _ptr, _stream_ptr, _check
    lib = _lib.load()
    torch.manual_seed(4)
    B, S, H = 40, 672, 8
    qkv = (torch.randn(B * S, 3 * H * 64, device="cuda") * 0.5).bfloat16()
    lens = torch.randint(0, S + 1, (B,), device="cuda", dtype=torch.int32)
    lens[:6] = torch.tensor([0, 1, 672, 128, 64, 65], device="cuda", dtype=torch.int32)
    table = saturating_table(H, S, seed=5)
    guard = 4096
    n = B * S * H * 64
    buf = torch.full((guard + n + guard,), 0x7F7B, dtype=torch.int16, device="cuda")
    out = buf[guard:guard + n]
    torch.cuda.synchronize()
    _check(lib.vqa_op_attention_d64(_ptr(qkv), _ptr(out), B, S, H, _ptr(lens), _ptr(table), 1.0, 128, 0, _stream_ptr(qkv.device)),
           None, "vqa_op_attention_d64")
    torch.cuda.synchronize()
    assert bool((buf[:guard] == 0x7F7B).all()) and bool((buf[guard + n:] == 0x7F7B).all())
    got = out.view(torch.bfloat16).view(B * S, H * 64)
    ref, qmask = reference(qkv, B, S, H, lens, table, 1.0, False)
    check_rows(got, ref, qmask, 0.03)

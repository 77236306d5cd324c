"""Kernel-level parity of the Qwen2.5-VL scoring path on a real H100: head-dim-128 prefill attention, M-RoPE, the vision re-orders, the
embedding splice, the penalty bitmaps, the penalised lm_head and the trace top-k, each against a plain torch restatement (fp64 where it is
not exact) written here from the same bf16 inputs and rounded where the kernel and the HF module round.

Outputs sit between sentinel guard bands, and what a kernel must not write has to come back bit-identical; qkv columns the attention never
reads hold NaN. Every group also checks that its fixture tells a correct kernel from a plausibly wrong one."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from attention_ref import assert_attn, assert_discriminates, attn_ref, bf16_ulp
from t2v_metrics_b200 import qwen_host

SENTINEL = -1280.0          # exact in bf16 and fp32
IMAGE_TOKEN = 151655        # Qwen2.5-VL's <|image_pad|>
VOCAB = 152064


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops(dev):
    from t2v_metrics_b200.engine import ops
    return ops


def guarded(rows, cols, dev, dtype=torch.bfloat16, pad_rows=8, pad_cols=64):
    """A [rows, cols] view (row stride cols + pad_cols) into a sentinel-filled buffer with pad_rows guard rows on each side."""
    big = torch.full((rows + 2 * pad_rows, cols + pad_cols), SENTINEL, dtype=dtype, device=dev)
    return big, big[pad_rows:pad_rows + rows, :cols]


def assert_guards(big, rows, cols, pad_rows=8, what=""):
    """Everything of `big` outside the [rows, cols] window still holds the sentinel, bit for bit."""
    keep = torch.ones_like(big, dtype=torch.bool)
    keep[pad_rows:pad_rows + rows, :cols] = False
    assert bool((big[keep] == SENTINEL).all()), f"{what}: a guard element was written"


# ================================================================================================ A. head-dim-128 attention
def qkv_layout(Hq, Hkv):
    """qwen_prefill's packed qkv row: q heads, then k heads, then v heads; 64 unread NaN columns after them."""
    return dict(ld=(Hq + 2 * Hkv) * 128 + 64, q0=0, k0=Hq * 128, v0=(Hq + Hkv) * 128)


def make_qkv(rows, Hq, Hkv, dev, gen, amp=0.5):
    L = qkv_layout(Hq, Hkv)
    qkv = torch.full((rows, L["ld"]), float("nan"), dtype=torch.bfloat16, device=dev)
    qkv[:, :L["ld"] - 64] = (torch.randn(rows, L["ld"] - 64, generator=gen) * amp).bfloat16().to(dev)
    return qkv, L


def split_heads(qkv, rows, Hq, Hkv, L):
    """[H, rows, 128] views of q and of k / v repeated to the q heads (GQA: q head h reads KV head h // group)."""
    g = Hq // Hkv
    q = qkv[rows, L["q0"]:L["q0"] + Hq * 128].view(-1, Hq, 128).transpose(0, 1)
    k = qkv[rows, L["k0"]:L["k0"] + Hkv * 128].view(-1, Hkv, 128).transpose(0, 1).repeat_interleave(g, 0)
    v = qkv[rows, L["v0"]:L["v0"] + Hkv * 128].view(-1, Hkv, 128).transpose(0, 1).repeat_interleave(g, 0)
    return q, k, v


GQA_CASES = [       # (q heads, KV heads, S, sequence lengths): groups 1, 2, 5, 7, 8; S around the 128-row tiles
    (28, 4, 320, [320, 1, 257, 129]),
    (28, 4, 1100, [1100, 1023]),
    (28, 4, 64, [64]),
    (2, 2, 1, [1, 1, 1]),
    (4, 2, 127, [127, 64]),
    (10, 2, 128, [128, 1, 100]),
    (16, 2, 129, [129, 128]),
    (2, 1, 255, [255, 2]),
    (4, 2, 256, [256, 255, 129]),
    (10, 2, 257, [257, 256, 17]),
    (4, 2, 320, [320, 200, 161]),
    (2, 1, 130, [130, 70]),
]


@pytest.mark.parametrize("Hq,Hkv,S,lens", GQA_CASES)
def test_attention_causal_gqa_padded(dev, ops, Hq, Hkv, S, lens):
    """The language model's fixed-stride causal GQA launch: padded rows exactly zero, nothing written past n_seq * S rows or Hq * 128 columns."""
    gen = torch.Generator().manual_seed(Hq * 1000 + S)
    n = len(lens)
    extra = 40                                              # qkv / out rows past the n * S the launch describes
    qkv, L = make_qkv(n * S + extra, Hq, Hkv, dev, gen)
    big, out = guarded(n * S + extra, Hq * 128, dev)
    seq_lens = torch.tensor(lens, dtype=torch.int32, device=dev)
    ops.attention_d128(qkv, out, L["q0"], L["k0"], L["v0"], n, S, Hq, Hq // Hkv, 128 ** -0.5, True, S=S, seq_lens=seq_lens)
    torch.cuda.synchronize()
    rows_written = torch.zeros(n * S + extra, Hq * 128, dtype=torch.bool, device=dev)
    rows_written[:n * S] = True
    assert bool((out[~rows_written] == SENTINEL).all()), "rows past n_seq * S were written"
    assert_guards(big, n * S + extra, Hq * 128, what="output")
    for b, ln in enumerate(lens):
        r = slice(b * S, b * S + ln)
        q, k, v = split_heads(qkv, r, Hq, Hkv, L)
        ref, ref_p = attn_ref(q, k, v, 128 ** -0.5, True)
        got = out[r].view(ln, Hq, 128).transpose(0, 1)
        tol = assert_attn(got, ref, ref_p, f"sequence {b}")
        assert bool((out[b * S + ln:(b + 1) * S] == 0).all()), f"padded rows of sequence {b} are not zero"
        if b == 0 and ln > 1:
            # the fixture sees a mask that drops the diagonal and a KV head of h % kv_heads
            s = torch.matmul(q.double(), k.double().transpose(1, 2)) * 128 ** -0.5
            s = s.masked_fill(torch.ones(ln, ln, dtype=torch.bool, device=dev).triu(0), float("-inf"))[:, 1:]
            wrong = torch.matmul(torch.softmax(s, -1), v.double())
            assert_discriminates(wrong, ref[:, 1:], tol[:, 1:], "a mask that drops the diagonal")
            kv_h = torch.arange(Hq, device=dev) % Hkv
            if bool((kv_h != torch.arange(Hq, device=dev) // (Hq // Hkv)).any()):      # the two mappings differ
                kk = qkv[r, L["k0"]:L["k0"] + Hkv * 128].view(ln, Hkv, 128).transpose(0, 1)[kv_h]
                vv = qkv[r, L["v0"]:L["v0"] + Hkv * 128].view(ln, Hkv, 128).transpose(0, 1)[kv_h]
                assert_discriminates(attn_ref(q, kk, vv, 128 ** -0.5, True)[0], ref, tol, "a KV head of h % kv_heads")


def test_attention_lazy_rescale(dev, ops):
    """Row maxima that grow by ~20 (log2) per key tile and by 140 over the row: the exponent reference has to be raised past 2^8, or the
    exponentials overflow fp32."""
    gen = torch.Generator().manual_seed(11)
    S, Hq, Hkv = 1024, 7, 1
    qkv, L = make_qkv(S, Hq, Hkv, dev, gen, amp=0.3)
    step = 20.0 / (16 * 128 ** -0.5 * math.log2(math.e))           # k[:, 0] per tile so that q.k scale log2(e) grows by 20 per tile
    tile = torch.arange(S) // 128
    qkv[:, L["q0"]:L["q0"] + Hq * 128].view(S, Hq, 128)[:, :, 0] = 16.0
    k0 = (tile * step + torch.randn(S, generator=gen) * 0.1).bfloat16().to(dev)
    qkv[:, L["k0"]] = k0
    big, out = guarded(S, Hq * 128, dev)
    ops.attention_d128(qkv, out, L["q0"], L["k0"], L["v0"], 1, S, Hq, Hq, 128 ** -0.5, True, S=S)
    torch.cuda.synchronize()
    assert_guards(big, S, Hq * 128, what="output")
    q, k, v = split_heads(qkv, slice(0, S), Hq, Hkv, L)
    ref, ref_p = attn_ref(q, k, v, 128 ** -0.5, True)
    assert_attn(out.view(S, Hq, 128).transpose(0, 1), ref, ref_p, "lazy rescale")
    # the fixture exercises the raise: the last row's reference (first tile's maximum, raised past +8) is raised on every tile
    x = (q[0, -1].double() @ k[0].double().t()) * 128 ** -0.5 * math.log2(math.e)
    tmax = x.view(8, 128).amax(-1).tolist()
    m, raises = tmax[0], 0
    for t in tmax[1:]:
        if t > m + 8:
            m, raises = t, raises + 1
    assert raises >= 6 and tmax[-1] - tmax[0] > 128, (raises, tmax)


@pytest.mark.parametrize("pre_len", [17, 128, 132, 256, 300])
def test_attention_kv_prefix(dev, ops, pre_len):
    """Shared-prefix mode: three suffixes (1, 77, 200 rows) over one prefix next to a prefix-less sequence, against fp64 attention over
    [prefix | suffix] and against the unshared launch of the concatenated sequences (bit-identical when the prefix fills whole key tiles)."""
    gen = torch.Generator().manual_seed(pre_len)
    Hq, Hkv = 28, 4
    sufs, alone = [1, 77, 200], 150
    lens = [pre_len] + sufs + [alone]
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    rows = cu[-1]
    qkv, L = make_qkv(rows, Hq, Hkv, dev, gen)
    big, out = guarded(rows, Hq * 128, dev)
    cu_t = torch.tensor(cu, dtype=torch.int32, device=dev)
    kvp = torch.tensor([-1, 0, 0, 0, -1], dtype=torch.int32, device=dev)
    ops.attention_d128(qkv, out, L["q0"], L["k0"], L["v0"], len(lens), max(lens), Hq, Hq // Hkv, 128 ** -0.5, True, cu_seqlens=cu_t,
                       kv_prefix=kvp)
    # the unshared launch: [prefix | suffix] for every suffix, then the prefix-less sequence
    parts = [torch.cat([qkv[:pre_len], qkv[cu[1 + i]:cu[2 + i]]]) for i in range(3)] + [qkv[cu[4]:cu[5]]]
    qkv2 = torch.cat(parts).contiguous()
    cu2 = [0]
    for p in parts:
        cu2.append(cu2[-1] + p.shape[0])
    out2 = torch.zeros(qkv2.shape[0], Hq * 128, dtype=torch.bfloat16, device=dev)
    ops.attention_d128(qkv2, out2, L["q0"], L["k0"], L["v0"], 4, max(cu2[i + 1] - cu2[i] for i in range(4)), Hq, Hq // Hkv, 128 ** -0.5, True,
                       cu_seqlens=torch.tensor(cu2, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    assert_guards(big, rows, Hq * 128, what="output")
    for sq in range(len(lens)):
        r = slice(cu[sq], cu[sq + 1])
        q, k, v = split_heads(qkv, r, Hq, Hkv, L)
        if 1 <= sq <= 3:            # a suffix: keys [prefix | own rows]
            kp, vp = split_heads(qkv, slice(0, pre_len), Hq, Hkv, L)[1:]
            ref, ref_p = attn_ref(q, torch.cat([kp, k], 1), torch.cat([vp, v], 1), 128 ** -0.5, True, q_off=pre_len)
        else:
            ref, ref_p = attn_ref(q, k, v, 128 ** -0.5, True)
        got = out[r].view(-1, Hq, 128).transpose(0, 1)
        tol = assert_attn(got, ref, ref_p, f"sequence {sq}")
        if 1 <= sq <= 3:
            unshared = out2[cu2[sq - 1] + pre_len:cu2[sq]]
            if pre_len % 128 == 0:
                assert torch.equal(out[r], unshared), f"suffix {sq}: differs from the unshared launch"
            else:
                assert_attn(unshared.view(-1, Hq, 128).transpose(0, 1), ref, ref_p, f"unshared suffix {sq}")
            if sq == 1:
                # the fixture sees prefix tiles masked with the suffix length
                n_vis = min(pre_len, sufs[0])
                wrong = attn_ref(q, torch.cat([kp[:, :n_vis], k], 1), torch.cat([vp[:, :n_vis], v], 1), 128 ** -0.5, True, q_off=n_vis)[0]
                assert_discriminates(wrong, ref, tol, "prefix tiles masked with the suffix length")


def _grid_windows(grids):
    _, cu_win, cu_frames = qwen_host.vision_window_index(grids, 2, 112, 14)
    return torch.diff(cu_win).tolist(), torch.diff(cu_frames).tolist()


VISION_CASES = [    # (name, sequence lengths, heads, compact 80-wide output, two windows per tile)
    ("windows 22x38", _grid_windows([(1, 22, 38)])[0], 16, True, True),
    ("windows 22x38 unpaired", _grid_windows([(1, 22, 38)])[0], 16, True, False),
    ("six full windows", [64] * 6, 3, True, True),
    ("ragged windows", [64, 64, 40, 64, 17], 3, True, True),
    ("short first window", [8, 64, 64], 3, True, True),
    ("one odd window", [33], 3, True, True),
    ("2 frames of 1024", _grid_windows([(2, 32, 32)])[1], 16, True, False),
    ("frame of 4096", _grid_windows([(1, 64, 64)])[1], 16, True, False),
]


def check_vision_attention(dev, ops, name, lens, H, compact, pair):
    """The vision tower's launch: 80-wide heads in 128-wide slots (Q / K pad columns zero as the memset leaves them; V pad columns NaN with a
    compact output, which must never reach it; zero with 128-wide output heads, whose pad columns must then come out zero)."""
    gen = torch.Generator().manual_seed(len(lens) * 7 + H)
    hd = 80
    rows = sum(lens)
    x = torch.zeros(rows, 3, H, 128)
    x[..., :hd] = torch.randn(rows, 3, H, hd, generator=gen) * 0.6
    if compact:
        x[:, 2, :, hd:] = float("nan")
    qkv = x.reshape(rows, 3 * H * 128).bfloat16().to(dev)
    d_out = hd if compact else 128
    big, out = guarded(rows, H * d_out, dev)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=dev)
    ops.attention_d128(qkv, out, 0, H * 128, 2 * H * 128, len(lens), max(lens), H, 1, hd ** -0.5, False, cu_seqlens=cu, pair_sequences=pair,
                       o_head_stride=d_out, d_out=d_out)
    torch.cuda.synchronize()
    assert_guards(big, rows, H * d_out, what="output")
    xv = qkv.view(rows, 3, H, 128)
    o = 0
    for n in lens:
        q, k, v = (xv[o:o + n, i, :, :d_out].transpose(0, 1) for i in range(3))
        got = out[o:o + n].view(n, H, d_out).transpose(0, 1)
        for r0 in range(0, n, 1024):                # row blocks bound the fp64 score memory of the 4096-row frame
            ref, ref_p = attn_ref(q[:, r0:r0 + 1024, :hd], k[:, :, :hd], v, hd ** -0.5, False)
            assert_attn(got[:, r0:r0 + 1024], ref, ref_p, f"{name}: sequence at row {o}")
        o += n
    if not compact:
        assert bool((out.view(rows, H, 128)[..., hd:] == 0).all()), "zero V pad columns must give zero output columns"


@pytest.mark.parametrize("name,lens,H,compact,pair", VISION_CASES, ids=[c[0] for c in VISION_CASES])
def test_attention_vision(dev, ops, name, lens, H, compact, pair):
    """Compact 80-wide output heads: windows two per tile or one per tile, whole frames of 1024 and 4096 rows."""
    check_vision_attention(dev, ops, name, lens, H, compact, pair)


def test_attention_vision_padded_heads(dev, ops):
    """80-wide heads zero-padded to 128 columns, written as 128-wide output heads, over variable-length windows one per tile (one longer
    than a tile)."""
    check_vision_attention(dev, ops, "padded heads", [64, 64, 16, 48, 130, 2], 4, False, False)


# ================================================================================================ B. rotary embeddings
def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat([-x[..., h:], x[..., :h]], -1)


def table_ref(pos, axis, inv_freq):
    """fp32 angle pos[axis[i], row] * inv_freq[i] -> (cos, sin) [rows, 2 * half] on CUDA, the halves duplicated."""
    ang = pos.float()[axis.long(), :].t() * inv_freq[None, :]
    c, s = torch.cos(ang), torch.sin(ang)
    return torch.cat([c, c], -1), torch.cat([s, s], -1)


def assert_table(got, ref_f32, round_bf16, what):
    """torch.equal to torch's CUDA cos / sin of the same fp32 angle (both reach libdevice cosf / sinf); failing that, within one fp32 ulp
    before the bf16 rounding. Returns which case held."""
    want = ref_f32.bfloat16().float() if round_bf16 else ref_f32
    if torch.equal(got, want):
        return "equal"
    lo, hi = torch.nextafter(ref_f32, torch.full_like(ref_f32, -2.0)), torch.nextafter(ref_f32, torch.full_like(ref_f32, 2.0))
    if round_bf16:
        lo, hi = lo.bfloat16().float(), hi.bfloat16().float()
    assert bool(((got >= torch.minimum(lo, hi)) & (got <= torch.maximum(lo, hi))).all()), f"{what}: table off by more than one fp32 ulp"
    return "one fp32 ulp"


def test_rope_text(dev, ops):
    """The language model's M-RoPE at 7B (theta 1e6, sections 16 / 24 / 24) on the q and k heads of a packed qkv row: bf16 tables, every product
    rounded to bf16 as apply_multimodal_rotary_pos_emb's bf16 tensor ops round it. Positions reach 131071 (cosf's slow argument reduction
    starts near 1.05e5 rad)."""
    t_inv, t_axis, _, _ = qwen_host.rope_tables(128, 1e6, (16, 24, 24), 80)
    gen = torch.Generator().manual_seed(21)
    rows, Hq, Hkv = 640, 28, 4
    pos = torch.randint(0, 131072, (3, rows), generator=gen, dtype=torch.int32)
    pos[:, :6] = torch.tensor([[131071, 105000, 0, 1, 70000, 99999], [131070, 104999, 3, 65536, 1, 2], [131069, 110000, 5, 7, 131071, 0]])
    pos = pos.to(dev)
    axis, inv = t_axis.to(dev), t_inv.to(dev)
    ld = (Hq + 2 * Hkv) * 128 + 64
    x = (torch.randn(rows, ld, generator=gen) * 2).bfloat16().to(dev)
    x0 = x.clone()
    tbig_c, cos_t = guarded(rows, 128, dev, torch.float32, pad_cols=0)
    tbig_s, sin_t = guarded(rows, 128, dev, torch.float32, pad_cols=0)
    ops.qwen_rope(pos, axis, inv, x, 0, Hq + Hkv, 128, 128, True, cos_t=cos_t, sin_t=sin_t)
    torch.cuda.synchronize()
    assert_guards(tbig_c, rows, 128, what="cos table")
    assert_guards(tbig_s, rows, 128, what="sin table")
    c32, s32 = table_ref(pos, axis, inv)
    held = {assert_table(cos_t, c32, True, "cos"), assert_table(sin_t, s32, True, "sin")}
    print(f"text rope tables vs torch.cos / torch.sin on CUDA: {sorted(held)}")
    cb, sb = cos_t.bfloat16()[:, None, :], sin_t.bfloat16()[:, None, :]
    xh = x0[:, :(Hq + Hkv) * 128].view(rows, Hq + Hkv, 128)
    want = xh * cb + rotate_half(xh) * sb                            # bf16 tensors: each product and the sum rounded
    assert torch.equal(x[:, :(Hq + Hkv) * 128].view(rows, Hq + Hkv, 128), want)
    assert torch.equal(x[:, (Hq + Hkv) * 128:], x0[:, (Hq + Hkv) * 128:]), "V heads or unrotated columns changed"
    # the fixture sees fp32 products and a first section read from the h axis
    assert bool(((xh.float() * cb.float() + rotate_half(xh).float() * sb.float()).bfloat16() != want).any())
    wrong_axis = axis.clone()
    wrong_axis[:16] = 1
    assert not torch.equal(table_ref(pos, wrong_axis, inv)[0].bfloat16(), c32.bfloat16())


def test_rope_vision(dev, ops):
    """The vision tower's rotary embedding: fp32 tables and products on 80 of the 128 dims of 16 q and 16 k heads; pad columns untouched."""
    _, _, v_inv, v_axis = qwen_host.rope_tables(128, 1e6, (16, 24, 24), 80)
    grid = [(1, 22, 38)]
    pos = qwen_host.vision_rot_pos_ids(grid, 2).t().contiguous().to(torch.int32).to(dev)      # [2, L] (h, w)
    rows, H, hd = pos.shape[1], 16, 80
    gen = torch.Generator().manual_seed(22)
    x = torch.full((rows, 3 * H, 128), SENTINEL)
    x[..., :hd] = torch.randn(rows, 3 * H, hd, generator=gen) * 2
    x = x.reshape(rows, 3 * H * 128).bfloat16().to(dev)
    x0 = x.clone()
    tbig_c, cos_t = guarded(rows, hd, dev, torch.float32, pad_cols=0)
    tbig_s, sin_t = guarded(rows, hd, dev, torch.float32, pad_cols=0)
    axis, inv = v_axis.to(dev), v_inv.to(dev)
    ops.qwen_rope(pos, axis, inv, x, 0, 2 * H, 128, hd, False, cos_t=cos_t, sin_t=sin_t)
    torch.cuda.synchronize()
    assert_guards(tbig_c, rows, hd, what="cos table")
    assert_guards(tbig_s, rows, hd, what="sin table")
    c32, s32 = table_ref(pos, axis, inv)
    held = {assert_table(cos_t, c32, False, "cos"), assert_table(sin_t, s32, False, "sin")}
    xh = x0.view(rows, 3 * H, 128)[:, :2 * H, :hd].float()
    want = xh * cos_t[:, None, :] + rotate_half(xh) * sin_t[:, None, :]        # fp32 throughout, one rounding to bf16
    got = x.view(rows, 3 * H, 128)[:, :2 * H, :hd].float()
    assert float(((got.double() - want.double()).abs() - bf16_ulp(want)).max()) <= 0.0, "vision rope: more than one bf16 ulp from fp32"
    frac = float((got != want.bfloat16().float()).double().mean())
    print(f"vision rope tables vs torch on CUDA: {sorted(held)}; rotated values not bit-equal to bf16(fp32 restatement): {frac:.2e}")
    assert frac < 0.01
    rest = torch.ones(rows, 3 * H, 128, dtype=torch.bool, device=dev)
    rest[:, :2 * H, :hd] = False
    assert torch.equal(x.view(rows, 3 * H, 128)[rest], x0.view(rows, 3 * H, 128)[rest]), "pad columns or V heads changed"
    # the fixture sees a rotation over the 128-wide slot: the pad columns it would pull in hold the sentinel
    assert bool((x0.view(rows, 3 * H, 128)[:, :2 * H, hd:] == SENTINEL).all())


# ================================================================================================ C. re-orders, splice, bitmaps
GRIDS = [(1, 22, 38), (1, 16, 16), (2, 20, 28)]        # two images (one not a multiple of 8 patches) and a 2-frame video grid


def test_gather_rows_window_order_and_inverse(dev, ops):
    """The window re-order of 2x2 patch groups (group 4) and its inverse on the merged features (group 1), against torch indexing."""
    window_index, _, _ = qwen_host.vision_window_index(GRIDS, 2, 112, 14)
    L = sum(t * h * w for t, h, w in GRIDS)
    assert not torch.equal(window_index, torch.arange(L // 4)), "the window order must not be the identity"
    gen = torch.Generator().manual_seed(31)
    idx = window_index.to(torch.int32).to(dev)
    src = torch.randn(L, 1288, generator=gen).bfloat16().to(dev)
    big, out = guarded(L, 1288, dev, pad_cols=0)
    ops.gather_rows(src, idx, 4, out=out)
    feats = torch.randn(L // 4, 3584, generator=gen).bfloat16().to(dev)
    reverse = torch.argsort(window_index).to(torch.int32).to(dev)
    big2, back = guarded(L // 4, 3584, dev, pad_cols=0)
    ops.gather_rows(feats, reverse, 1, out=back)
    torch.cuda.synchronize()
    assert torch.equal(out, src.view(L // 4, 4, -1)[window_index.long().to(dev)].reshape(L, -1))
    assert torch.equal(back, feats[reverse.long()])
    assert_guards(big, L, 1288, what="group 4")
    assert_guards(big2, L // 4, 3584, what="group 1")


def _prompts(gen, shared):
    """Prompts with one vision run each: (ids, image of each prompt). shared: three prompts over image 0 with one prefix."""
    feats = [t * h * w // 4 for t, h, w in GRIDS]
    rnd = lambda n: torch.randint(100, 150000, (n,), generator=gen).tolist()
    pre = rnd(5)
    prompts, imgs = [], []
    for b, img in enumerate([0, 0, 0, 1, 2] if shared else [0, 1, 2, 0]):
        head = pre if shared and img == 0 else rnd(3 + b)
        prompts.append(head + [IMAGE_TOKEN] * feats[img] + rnd(4 + 9 * b))
        imgs.append(img)
    return prompts, imgs


def _embed_tables(gen, dev, D):
    embed = torch.randn(VOCAB, D, generator=gen).bfloat16()
    embed[0] = 7.0                          # the pad id: padded rows must not take it
    embed[IMAGE_TOKEN] = float("nan")       # ids are read only where feat_index < 0
    n_feat = sum(t * h * w // 4 for t, h, w in GRIDS)
    return embed.to(dev), torch.randn(n_feat, D, generator=gen).bfloat16().to(dev)


def _embed_ref(ids, feat, valid, embed, feats):
    out = torch.where((feat >= 0)[:, None], feats[feat.clamp_min(0)], embed[ids.clamp(0, VOCAB - 1)])
    return torch.where(valid[:, None], out, torch.zeros_like(out))


@pytest.mark.parametrize("packed", [False, True])
def test_qwen_embed(dev, ops, packed):
    """The feature splice in the padded layout (rows at or past seq_len zero) and in the packed layout qwen_prefill uses (cu_seqlens + n_seq, S = M)."""
    gen = torch.Generator().manual_seed(41 + packed)
    D = 1288
    embed, feats = _embed_tables(gen, dev, D)
    prompts, imgs = _prompts(gen, shared=packed)
    if packed:
        pk = qwen_host.build_packed_indices(prompts, GRIDS, imgs, IMAGE_TOKEN, 2, 2)
        assert pk["n_shared"] == 1
        rows = pk["total_rows"]
        ids, feat = pk["input_ids"].to(dev), pk["feat_index"].to(dev)
        cu = pk["cu_seqlens"].to(dev)
        seq_lens, S = cu[pk["n_seq"]:], rows
        valid = torch.ones(rows, dtype=torch.bool, device=dev)
    else:
        bi = qwen_host.build_batch_indices(prompts, GRIDS, imgs, IMAGE_TOKEN, 2, 2)
        B, S = bi["input_ids"].shape
        rows = B * S
        ids, feat = bi["input_ids"].reshape(-1).to(dev), bi["feat_index"].reshape(-1).to(dev)
        seq_lens = bi["seq_lens"].to(dev)
        valid = (torch.arange(S, device=dev)[None, :] < seq_lens[:, None]).reshape(-1)
        assert not bool(valid.all()), "the padded fixture needs padded rows"
    big, out = guarded(rows, D, dev, pad_cols=0)
    ops.qwen_embed(ids, feat, seq_lens, embed, feats, S, out=out)
    torch.cuda.synchronize()
    assert torch.equal(out, _embed_ref(ids.long(), feat.long(), valid, embed, feats))
    assert_guards(big, rows, D, what="embed")


def _bits(id_lists, vocab):
    """Bit id of row b set for every id of id_lists[b] in [0, vocab): int32 [B, ceil(vocab / 32)], the uint32 words' bit patterns."""
    words = (vocab + 31) // 32
    bits = torch.zeros(len(id_lists), words * 32, dtype=torch.bool)
    for b, ids in enumerate(id_lists):
        t = torch.as_tensor(list(ids), dtype=torch.int64)
        bits[b, t[(t >= 0) & (t < vocab)]] = True
    w = (bits.view(len(id_lists), words, 32).to(torch.int64) << torch.arange(32)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


@pytest.mark.parametrize("vocab", [VOCAB, 1000])
def test_token_bitmap_padded(dev, ops, vocab):
    """Ids outside [0, vocab), repeated ids, ids in padded positions (not counted)."""
    gen = torch.Generator().manual_seed(51)
    B, S = 5, 300
    ids = torch.randint(0, vocab, (B, S), generator=gen, dtype=torch.int32)
    ids[:, :6] = torch.tensor([-5, vocab, vocab + 7, -1, 31, 31], dtype=torch.int32)
    lens = [300, 1, 17, 256, 257]
    ids[2, 17:] = vocab - 1                       # only in padded positions
    ids_d, lens_d = ids.to(dev), torch.tensor(lens, dtype=torch.int32, device=dev)
    bm = ops.token_bitmap(ids_d, vocab, B, seq_lens=lens_d, S=S)
    torch.cuda.synchronize()
    ref = _bits([ids[b, :lens[b]].tolist() for b in range(B)], vocab)
    assert torch.equal(bm.cpu(), ref)
    assert not torch.equal(ref, _bits([ids[b].tolist() for b in range(B)], vocab)), "padded ids must matter to the fixture"


def test_token_bitmap_packed(dev, ops):
    """Packed rows: a pair's prompt is its shared prefix sequence's rows followed by its own, ids outside the vocabulary ignored."""
    gen = torch.Generator().manual_seed(52)
    prompts, imgs = _prompts(gen, shared=True)
    pk = qwen_host.build_packed_indices(prompts, GRIDS, imgs, IMAGE_TOKEN, 2, 2)
    ids = pk["input_ids"].clone()
    cu, kvp, pair_seq = pk["cu_seqlens"].tolist(), pk["kv_prefix"].tolist(), pk["pair_seq"].tolist()
    own1 = cu[pair_seq[1]]
    ids[own1:own1 + 3] = torch.tensor([-7, VOCAB, VOCAB + 100], dtype=torch.int32)
    bm = ops.token_bitmap(ids.to(dev), VOCAB, len(prompts), cu_seqlens=pk["cu_seqlens"].to(dev), kv_prefix=pk["kv_prefix"].to(dev),
                          pair_seq=pk["pair_seq"].to(dev), max_prompt_len=pk["max_prompt_len"])
    torch.cuda.synchronize()
    lists, own_only = [], []
    for sq in pair_seq:
        own = ids[cu[sq]:cu[sq + 1]].tolist()
        pre = ids[cu[kvp[sq]]:cu[kvp[sq] + 1]].tolist() if kvp[sq] >= 0 else []
        lists.append(pre + own)
        own_only.append(own)
    ref = _bits(lists, VOCAB)
    assert torch.equal(bm.cpu(), ref)
    assert not torch.equal(ref, _bits(own_only, VOCAB)), "the prefix rows must matter to the fixture"


# ================================================================================================ D. penalised lm_head
def process_logits(logits_f32, bitmap, penalty, temperature):
    """The score's logit processing in fp32: bf16 logits, HF's repetition penalty on the ids in the bitmap, times fp32(1 / T)."""
    x = logits_f32.bfloat16().float()
    if bitmap is not None and penalty != 1.0:
        n = torch.arange(x.shape[1], device=x.device)
        bit = ((bitmap[:, n // 32] >> (n % 32)) & 1).bool()
        x = torch.where(bit, torch.where(x < 0, x * penalty, x / torch.full_like(x, penalty)), x)      # IEEE division, as __fdiv_rn
    return x * torch.tensor(1.0 / temperature, dtype=torch.float32)


def bitmap_of(sets, V, dev):
    return _bits(sets, V).to(dev)


@pytest.fixture(scope="module")
def int_weights(dev):
    """Integer-valued lm_head weights (multiples of 1/16 in [-3/16, 3/16]) at K = 3584 for both vocabularies."""
    gen = torch.Generator().manual_seed(61)
    return {N: (torch.randint(-3, 4, (N, 3584), generator=gen).float() / 16).bfloat16().to(dev) for N in (VOCAB, 1000)}


LSE_TOL = 1e-5          # fp32 log-sum-exp noise: the integer fixture's logits and the label logit are exact


@pytest.mark.parametrize("N", [VOCAB, 1000])
@pytest.mark.parametrize("M", [1, 7, 64, 128])
def test_lmhead_logprob_penalised(dev, ops, int_weights, M, N):
    """h and W are small multiples of powers of two, so the fp32 accumulation is exact in any order and the bf16 rounding of every logit is
    determined: the fp64 log-softmax of the processed logits is exact, and the kernel may differ by fp32 LSE noise only (LSE_TOL)."""
    gen = torch.Generator().manual_seed(M * 7 + N)
    K = 3584
    w = int_weights[N]
    h = (torch.randint(-3, 4, (M, K), generator=gen).float() / 8).bfloat16().to(dev)
    logits = torch.cat([h.double() @ w[i:i + 16384].double().t() for i in range(0, N, 16384)], 1)
    assert torch.equal(logits, (logits * 128).round() / 128) and float(logits.abs().max()) < 2 ** 16
    logits = logits.float()                                         # exact
    labels = torch.randint(0, N, (M,), generator=gen, dtype=torch.int32)
    labels[0] = N - 1
    for m in range(2, M, 2):                                        # penalised label logits of alternating sign
        cand = torch.nonzero(logits[m] > 0 if m % 4 == 2 else logits[m] < 0)[:, 0].cpu()
        labels[m] = int(cand[torch.randint(0, cand.numel(), (1,), generator=gen)])
    sets = [torch.randint(0, N, (N // 8,), generator=gen).tolist() + ([int(labels[m])] if m % 2 == 0 else []) for m in range(M)]
    bitmap = bitmap_of(sets, N, dev)
    lab = labels.long().to(dev)
    pen_rows = [m for m in range(M) if m % 2 == 0]
    lab_logit = logits[pen_rows, lab[pen_rows]]
    if M >= 7:
        assert bool((lab_logit > 0).any()) and bool((lab_logit < 0).any()), "penalised label logits of both signs"
    for T in (1.0, 0.5, 2.0):
        for pen in (1.0, 0.8, 1.3, 1.5):
            got = ops.lmhead_logprob(h, w, labels.to(dev), temperature=T, pen_bitmap=bitmap, repetition_penalty=pen)
            torch.cuda.synchronize()
            ref = torch.log_softmax(process_logits(logits, bitmap, pen, T).double(), -1).gather(1, lab[:, None])[:, 0]
            err = float((got.double() - ref).abs().max())
            assert err <= LSE_TOL, (T, pen, err)
            if pen != 1.0:
                # the fixture sees a penalty that multiplies positive logits
                x = logits.bfloat16().float()
                n = torch.arange(N, device=dev)
                bit = ((bitmap[:, n // 32] >> (n % 32)) & 1).bool()
                wrong = torch.log_softmax((torch.where(bit, x * pen, x) * (1.0 / T)).double(), -1).gather(1, lab[:, None])[:, 0]
                assert float((wrong - ref).abs().max()) > 10 * LSE_TOL


def test_lmhead_logprob_random_values(dev, ops):
    """Random-valued h and W at the lm_head test's bound (5e-3), with a temperature and a penalty. A random logit whose exact value lies
    within 1e-5 (relative) of a bf16 rounding midpoint may round either way after the kernel's fp32 accumulation; the reference takes both
    roundings there and bounds the log-probability from below and above (it increases with the label logit, decreases with every other)."""
    gen = torch.Generator().manual_seed(62)
    M, N, K = 64, VOCAB, 3584
    h = torch.randn(M, K, generator=gen).bfloat16().to(dev)
    w = (torch.randn(N, K, generator=gen) * K ** -0.5 * 3).bfloat16().to(dev)
    labels = torch.randint(0, N, (M,), generator=gen, dtype=torch.int32)
    bitmap = bitmap_of([torch.randint(0, N, (500,), generator=gen).tolist() + [int(labels[m])] for m in range(M)], N, dev)
    got = ops.lmhead_logprob(h, w, labels.to(dev), temperature=0.5, pen_bitmap=bitmap, repetition_penalty=1.3)
    torch.cuda.synchronize()
    exact = torch.cat([h.double() @ w[i:i + 16384].double().t() for i in range(0, N, 16384)], 1)
    a, b = (exact * (1 - 1e-5)).float(), (exact * (1 + 1e-5)).float()
    lo, hi = process_logits(torch.minimum(a, b), bitmap, 1.3, 0.5).double(), process_logits(torch.maximum(a, b), bitmap, 1.3, 0.5).double()
    lab = labels.long().to(dev)[:, None]

    def logprob(label_x, other_x):
        x = other_x.scatter(1, lab, label_x.gather(1, lab))
        return (x.gather(1, lab) - torch.logsumexp(x, -1, keepdim=True))[:, 0]
    lower, upper = logprob(lo, hi), logprob(hi, lo)
    g = got.double()
    assert bool(((g >= lower - 5e-3) & (g <= upper + 5e-3)).all()), float(torch.maximum(lower - g, g - upper).max())


# ================================================================================================ E. trace top-k
TOPK_PROB_RTOL = 2e-5   # __expf and an fp32 sum over the vocabulary


@pytest.mark.parametrize("V", [VOCAB, 1000])
@pytest.mark.parametrize("K", [1, 5, 8])
def test_topk_softmax(dev, ops, V, K):
    """Planted exact ties straddling the 256-thread strides (lower id first), columns past V that must never be read, the penalty and
    temperature of the score; ids equal to the fp64 reference's, probabilities within TOPK_PROB_RTOL."""
    gen = torch.Generator().manual_seed(V + K)
    B, ldl = 5, V + 24
    x = (torch.randn(B, ldl, generator=gen) * 2).bfloat16()
    x[:, V:] = 1e4                                              # past V: never a candidate
    ties = {0: [700, 3, 259, 4], 1: [999, 0, 256, 512, 1, 768, 5, 261, 517], 2: [10, 266, 11]}
    for r, t in ties.items():
        x[r, t] = 16.0
    sets = [torch.randint(0, V, (V // 6,), generator=gen).tolist() for _ in range(B)]
    for r in (0, 1):
        sets[r] = [i for i in sets[r] if i not in ties[r]]
    sets[2] = [i for i in sets[2] if i not in ties[2]] + ties[2]          # a penalised tie stays a tie
    bitmap = bitmap_of(sets, V, dev)
    logits = x.to(dev)
    for T, pen in ((1.0, 1.0), (0.5, 1.3), (2.0, 0.8), (1.0, 1.5)):
        ids, probs = ops.topk_softmax(logits, K, V=V, temperature=T, pen_bitmap=bitmap, repetition_penalty=pen)
        torch.cuda.synchronize()
        xp = process_logits(logits[:, :V].float(), bitmap, pen, T)
        order = torch.sort(xp, dim=1, descending=True, stable=True).indices[:, :K]      # ties keep the lower id first
        p = torch.softmax(xp.double(), -1).gather(1, order)
        assert torch.equal(ids.long(), order), (T, pen, ids.tolist(), order.tolist())
        assert float(((probs.double() - p).abs() / p).max()) <= TOPK_PROB_RTOL, (T, pen)
        # the fixture sees ties going to the higher id: row 0's winner is a tie
        assert int(order[0, 0]) == 3 and xp[0, 700] == xp[0, 3]

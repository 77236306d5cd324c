"""Head-dim-128 attention (attn_wgmma_kernel) and the flash-decoding kernel over the K/V cache, through the C ABI.

1. Exact selectors in every launch mode (key codes of attention_ref: one-hot or tied softmax, so the output is known bit for bit): fixed
   stride causal GQA at every group size and last-tile width, packed causal sequences, shared kv_prefix (a 15,616-row image prefix), the
   vision tower's paired 64-patch windows and whole frames of 62,208 and 64,896 patches. Decoys the mask must hide sit in the partner
   window, the future of the causal diagonal, padding rows, neighbouring sequences and just past a prefix.
2. Random inputs at production lengths under the per-element bound of attention_ref, P rounded at the kernel's exponent reference (first
   key tile's maximum, raised past 2^8), query rows sampled in 1,024-row blocks; every group shows which named mistakes its fixture sees.
3. Invariance: fixed stride vs packed rows, row offsets, neighbours, batch size, padding content, shared vs unshared prefix, bit for bit.
4. Flash decoding: selectors across split boundaries for every group size and split count, and row-for-row parity with the prefill
   kernel over a cache filled from a 15,616-token prompt."""
import math

import pytest
import torch

from attention_ref import (Layout, Selector, assert_attn, attn_bound, decode_selector, masked_ref, sample_row_blocks)
from t2v_metrics_b200 import qwen_host

pytestmark = pytest.mark.gpu

LM_SCALE = 128 ** -0.5
VIS_HD = 80
VIS_SCALE = VIS_HD ** -0.5
PROMPT = 15616             # a 3024x4032 photo: 15,552 image tokens (62,208 patches / 4) plus a prompt
FRAMES = [62208, 64896]    # 216x288 and 208x312 patch grids: 3024x4032 and 6000x4000 under the plugin's default max_pixels


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops(dev):
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


def gen_on(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def assert_bits(got, want, what):
    diff = got.contiguous().view(torch.int16) != want.contiguous().view(torch.int16)
    if bool(diff.any()):
        i = tuple(diff.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(diff.sum())} of {diff.numel()} elements differ, first at {list(i)}: {float(got[i])} vs {float(want[i])}")


# ================================================================================================ launches
def lm_qkv(q, k, v):
    """The language model's packed qkv row from [R, H, 128] parts: q heads, k heads, v heads, then 64 unread NaN columns."""
    R = q.shape[0]
    x = torch.cat([q.reshape(R, -1), k.reshape(R, -1), v.reshape(R, -1), torch.full((R, 64), float("nan"), device=q.device)], 1)
    return x.bfloat16().contiguous()


def run_lm(ops, qkv, Hq, Hkv, L, seq_lens=None):
    """A causal launch of the Layout's sequences (fixed stride when L.S is set, else packed cu_seqlens with its kv_prefix)."""
    dev = qkv.device
    out = torch.full((qkv.shape[0], Hq * 128), -1280.0, dtype=torch.bfloat16, device=dev)
    k0, v0 = Hq * 128, (Hq + Hkv) * 128
    n = len(L.groups)
    if L.S is not None:
        lens = torch.tensor(L.groups, dtype=torch.int32, device=dev) if seq_lens is None else seq_lens
        ops.attention_d128(qkv, out, 0, k0, v0, n, L.S, Hq, Hq // Hkv, LM_SCALE, True, S=L.S, seq_lens=lens)
    else:
        cu = torch.tensor([0] + L.lens.cumsum(0).tolist(), dtype=torch.int32, device=dev)
        kvp = None if bool((L.prefix_of < 0).all()) else L.prefix_of.to(torch.int32).to(dev)
        ops.attention_d128(qkv, out, 0, k0, v0, n, max(L.groups), Hq, Hq // Hkv, LM_SCALE, True, cu_seqlens=cu, kv_prefix=kvp)
    torch.cuda.synchronize()
    return out


def vision_qkv(q, k, v, compact):
    """[R, 3 * H * 128] rows of 80-wide heads in 128-wide slots; V pad columns NaN for a compact launch (they must never reach the output)."""
    v = v.clone()
    if compact:
        v[..., VIS_HD:] = float("nan")
    R = q.shape[0]
    return torch.cat([q.reshape(R, -1), k.reshape(R, -1), v.reshape(R, -1)], 1).bfloat16().contiguous()


def run_vision(ops, qkv, H, groups, compact, pair):
    dev = qkv.device
    d_out = VIS_HD if compact else 128
    out = torch.full((qkv.shape[0], H * d_out), -1280.0, dtype=torch.bfloat16, device=dev)
    cu = torch.tensor([0] + torch.tensor(groups).cumsum(0).tolist(), dtype=torch.int32, device=dev)
    ops.attention_d128(qkv, out, 0, H * 128, 2 * H * 128, len(groups), max(groups), H, 1, VIS_SCALE, False, cu_seqlens=cu,
                       pair_sequences=pair, o_head_stride=d_out, d_out=d_out)
    torch.cuda.synchronize()
    return out


def windows(grids):
    _, cu_win, _ = qwen_host.vision_window_index(grids, 2, 112, 14)
    return torch.diff(cu_win).tolist()


# ================================================================================================ 1. exact selectors
# len mod 128 = 0, 1, 16, 17, 64, 65, 127, len 1, and 256 / 1 in S = 1152: whole padding query tiles
FIXED_LENS = [1024, 897, 912, 913, 960, 961, 1023, 1, 256]
GROUPS = [(2, 2), (4, 2), (8, 2), (10, 2), (28, 4), (16, 2)]      # group sizes 1, 2, 4, 5, 7 (7B: 28 / 4), 8 (3B: 16 / 2)


@pytest.mark.parametrize("Hq,Hkv", GROUPS)
def test_selector_fixed_stride_causal_gqa(dev, ops, Hq, Hkv):
    """Query i selects a key <= i (one in eight its own diagonal); the keys just past the diagonal and the padding rows carry a query's
    code as decoys; codes are per KV head, so a wrong head mapping selects other values. Padding rows come out +0."""
    L = Layout(FIXED_LENS, True, S=1152, device=dev)
    sel = Selector(L, Hq, Hkv, 128, gen_on(dev, Hq * 100 + Hkv), ties=40)
    want, cnt = sel.expected()
    out = run_lm(ops, lm_qkv(*sel.tensors()), Hq, Hkv, L)
    assert_bits(out.view(L.rows, Hq, 128), want, f"fixed stride {Hq}/{Hkv}")
    assert int(cnt.max()) >= 2 and len(sel.victims[0]) > 500


@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2)])
def test_selector_packed_causal(dev, ops, Hq, Hkv):
    """Packed sequences that start mid-tile; the rows of neighbouring sequences are decoys."""
    L = Layout([300, 1, 129, 700, 64, 1000, 17, 255], True, device=dev)
    sel = Selector(L, Hq, Hkv, 128, gen_on(dev, 7 + Hq), ties=40)
    want, _ = sel.expected()
    out = run_lm(ops, lm_qkv(*sel.tensors()), Hq, Hkv, L)
    assert_bits(out.view(L.rows, Hq, 128), want, "packed")


def test_selector_kv_prefix(dev, ops):
    """Prefixes of 15,616 (whole tiles), 129 and 255 rows, each shared by suffixes; a suffix query selects a prefix key or one of its own
    keys <= i, and the rows of other sequences, including those right after its prefix's last tile, are decoys."""
    groups = [PROMPT, 77, 200, 1, 129, 50, 300, 255, 130, 90]
    prefix_of = [-1, 0, 0, 0, -1, 4, 4, -1, 7, -1]
    L = Layout(groups, True, prefix_of=prefix_of, device=dev)
    Hq, Hkv = 28, 4
    sel = Selector(L, Hq, Hkv, 128, gen_on(dev, 11), ties=60)
    want, _ = sel.expected()
    out = run_lm(ops, lm_qkv(*sel.tensors()), Hq, Hkv, L)
    assert_bits(out.view(L.rows, Hq, 128), want, "kv_prefix")


# 2160x3840: merged grid 77 x 137, windows of 64 patches with 16- and 4-patch edge windows (700 windows); one more 4-patch window makes the
# count odd (an unpaired last tile)
PAIR_CASES = {"2160x3840": windows([(1, 154, 274)]), "2160x3840 odd": windows([(1, 154, 274)]) + [4], "ragged": [64, 64, 40, 64, 17]}


@pytest.mark.parametrize("case", list(PAIR_CASES))
def test_selector_vision_windows(dev, ops, case):
    """Windows two per tile (block-diagonal mask) and one per tile give the same exact output; the partner window's keys are decoys."""
    groups = PAIR_CASES[case]
    L = Layout(groups, False, device=dev)
    H = 16
    sel = Selector(L, H, H, VIS_HD, gen_on(dev, len(groups)), ties=min(30, L.rows // 64), near=64)
    want, _ = sel.expected()
    qkv = vision_qkv(*sel.tensors(), compact=True)
    for pair in (True, False):
        out = run_vision(ops, qkv, H, groups, True, pair)
        assert_bits(out.view(L.rows, H, VIS_HD), want, f"{case} pair={pair}")


@pytest.mark.parametrize("compact", [True, False])
@pytest.mark.parametrize("frame", FRAMES)
def test_selector_whole_frames(dev, ops, frame, compact):
    """Frames of 62,208 and 64,896 patches, 16 heads: ~490 key tiles per row, ties spread over distant tiles (the lazy-rescale reset and l
    sums over every key are exact), the rows of a 1,000-patch frame after it are decoys next to the boundary. Compact output (80 columns,
    NaN V pad) and 128-wide output (zero V pad: the pad columns come out +0). Triples of 80 dimensions give 82,160 codes, enough for one
    such frame and its neighbour per launch."""
    groups = [frame, 1000]
    L = Layout(groups, False, device=dev)
    H = 16
    sel = Selector(L, H, H, VIS_HD, gen_on(dev, frame + compact), ties=400, tie_sizes=(2, 3, 4))
    want, cnt = sel.expected()
    assert int(cnt.max()) >= 3
    out = run_vision(ops, vision_qkv(*sel.tensors(), compact), H, groups, compact, False)
    if compact:
        assert_bits(out.view(L.rows, H, VIS_HD), want, "frames, compact")
    else:
        o = out.view(L.rows, H, 128)
        assert_bits(o[..., :VIS_HD], want, "frames, 128-wide")
        assert bool((o[..., VIS_HD:].contiguous().view(torch.int16) == 0).all())


# ================================================================================================ 2. bounds at production lengths
def rand_heads(R, H, dev, gen, amp=0.5, hd=128):
    x = torch.zeros(R, H, 128, device=dev)
    x[..., :hd] = torch.randn(R, H, hd, generator=gen, device=dev) * amp
    return x.bfloat16().float()


def check_rows(got, q, k, v, scale, vis, mistakes, seen, what):
    """got [H, n, d] against masked_ref(q, k, v, vis); mistakes: name -> (k, v, vis, scale) of a plausibly wrong kernel, checked until
    one block shows it."""
    ref, ref_p = masked_ref(q, k, v, scale, vis)
    tol = assert_attn(got, ref, ref_p, what)
    for name, (k2, v2, vis2, sc2) in mistakes.items():
        if name in seen:
            continue
        rows = vis2.reshape(-1, vis2.shape[-1]).any(-1).view(vis2.shape[:-1]) if vis2.dim() == 3 else vis2.any(-1)
        wrong = masked_ref(q, k2, v2, sc2, vis2)[0]
        moved = ((wrong - ref).abs() > 4.0 * tol) & rows[..., None]
        if bool(moved.any()):
            seen.add(name)


def lm_bounds(ops, dev, Hq, Hkv, lens, gen):
    """Fixed stride with ragged seq_lens, then the same sequences packed: bit-identical valid rows, every sampled block within the bound,
    the named mistakes seen."""
    S, G = max(lens), Hq // Hkv
    L = Layout(lens, True, S=S, device=dev)
    q, k, v = rand_heads(L.rows, Hq, dev, gen), rand_heads(L.rows, Hkv, dev, gen), rand_heads(L.rows, Hkv, dev, gen)
    qkv = lm_qkv(q, k, v)
    out = run_lm(ops, qkv, Hq, Hkv, L)
    valid = (L.seq >= 0)
    Lp = Layout(lens, True, device=dev)
    packed = run_lm(ops, qkv[valid].contiguous(), Hq, Hkv, Lp)
    assert_bits(packed, out[valid], "packed vs fixed stride")
    assert bool((out[~valid].view(torch.int16) == 0).all())
    seen, hk = set(), torch.arange(Hq, device=dev)
    for b, n in enumerate(lens):
        base = b * S
        kk, vv = k[base:base + n].transpose(0, 1), v[base:base + n].transpose(0, 1)
        for r0, r1 in sample_row_blocks(n):
            i, j = torch.arange(r0, r1, device=dev)[:, None], torch.arange(r1, device=dev)[None, :]
            for h0 in range(0, Hq, G):
                hs = hk[h0:h0 + G]
                qq = q[base + r0:base + r1, hs].transpose(0, 1)
                mistakes = {"diagonal dropped": (kk[hs // G, :r1], vv[hs // G, :r1], j < i, LM_SCALE),
                            "KV head h % kv_heads": (kk[hs % Hkv, :r1], vv[hs % Hkv, :r1], j <= i, LM_SCALE)}
                if bool(((hs % Hkv) == (hs // G)).all()):
                    del mistakes["KV head h % kv_heads"]
                check_rows(out[base + r0:base + r1].view(-1, Hq, 128)[:, hs].transpose(0, 1), qq, kk[hs // G, :r1], vv[hs // G, :r1],
                           LM_SCALE, j <= i, mistakes, seen, f"{Hq}/{Hkv} sequence {b} rows {r0}..{r1} heads {h0}..")
    return seen


@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2)])
def test_bounds_lm_prompt(dev, ops, Hq, Hkv):
    seen = lm_bounds(ops, dev, Hq, Hkv, [PROMPT, PROMPT - 63], gen_on(dev, Hq))
    print(f"{Hq}/{Hkv} prompt of {PROMPT}: the fixture sees {sorted(seen)}")
    assert seen == {"diagonal dropped", "KV head h % kv_heads"}


def test_bounds_and_invariance_kv_prefix(dev, ops):
    """A 15,616-row prefix (whole tiles) shared by three suffixes and a 15,617-row one (a ragged prefix tile) by one: within the bound of
    [prefix | suffix] attention, and the whole-tile prefix bit-identical to the unshared launch of the concatenated rows."""
    gen = gen_on(dev, 3)
    Hq, Hkv, G = 28, 4, 7
    groups, prefix_of = [PROMPT, 300, 77, 1, PROMPT + 1, 129], [-1, 0, 0, 0, -1, 4]
    L = Layout(groups, True, prefix_of=prefix_of, device=dev)
    q, k, v = rand_heads(L.rows, Hq, dev, gen), rand_heads(L.rows, Hkv, dev, gen), rand_heads(L.rows, Hkv, dev, gen)
    st = L.start.tolist()
    k[st[5]] = (k[st[5]] * 8).bfloat16().float()          # the key right after the ragged prefix carries weight: a slip onto it shows
    qkv = lm_qkv(q, k, v)
    out = run_lm(ops, qkv, Hq, Hkv, L)
    # the unshared launch: [prefix | suffix] for the three suffixes of the whole-tile prefix
    parts = [torch.cat([qkv[:PROMPT], qkv[st[s]:st[s] + groups[s]]]) for s in (1, 2, 3)]
    Lu = Layout([p.shape[0] for p in parts], True, device=dev)
    un = run_lm(ops, torch.cat(parts).contiguous(), Hq, Hkv, Lu)
    ust = Lu.start.tolist()
    for i, s in enumerate((1, 2, 3)):
        assert_bits(out[st[s]:st[s] + groups[s]], un[ust[i] + PROMPT:ust[i] + PROMPT + groups[s]], f"suffix {s} vs unshared")
    seen = set()
    for s in (1, 2, 3, 5):
        p = prefix_of[s]
        pb, pl, n = st[p], groups[p], groups[s]
        pad = -(-pl // 128) * 128                             # the kernel's own key tiles restart after the prefix
        keys = torch.cat([torch.arange(pb, pb + pl, device=dev), torch.zeros(pad - pl, dtype=torch.long, device=dev),
                          torch.arange(st[s], st[s] + n, device=dev)])
        col = torch.arange(pad + n, device=dev)[None, :]
        i = torch.arange(n, device=dev)[:, None]
        vis = (col < pl) | ((col >= pad) & (col - pad <= i))
        past = torch.cat([keys[:pl], torch.tensor([pb + pl], device=dev), keys[pl + 1:]]) if pad > pl else None
        for h0 in range(0, Hq, G):
            hs = torch.arange(h0, h0 + G, device=dev)
            kk, vv = k[keys][:, hs // G].transpose(0, 1), v[keys][:, hs // G].transpose(0, 1)
            mistakes = {"prefix tiles masked at the suffix length": (kk, vv, ((col < min(pl, n)) | ((col >= pad) & (col - pad <= i))), LM_SCALE)}
            if past is not None:
                mistakes["one key past the prefix"] = (k[past][:, hs // G].transpose(0, 1), v[past][:, hs // G].transpose(0, 1),
                                                       vis | (col == pl), LM_SCALE)
            check_rows(out[st[s]:st[s] + n].view(n, Hq, 128)[:, hs].transpose(0, 1), q[st[s]:st[s] + n, hs].transpose(0, 1), kk, vv,
                       LM_SCALE, vis, mistakes, seen, f"suffix {s} heads {h0}..")
    print(f"kv_prefix: the fixture sees {sorted(seen)}")
    assert seen == {"prefix tiles masked at the suffix length", "one key past the prefix"}


def test_bounds_vision_frame(dev, ops):
    """A 1,000-patch frame (ragged last tile) and a 62,208-patch one, 16 heads of 80 in 128-wide slots, compact output."""
    gen = gen_on(dev, 4)
    H, groups = 16, [1000, FRAMES[0]]
    R = sum(groups)
    q, k, v = (rand_heads(R, H, dev, gen, 0.6, VIS_HD) for _ in range(3))
    out = run_vision(ops, vision_qkv(q, k, v, True), H, groups, True, False).view(R, H, VIS_HD)
    seen = set()
    for f, (a, n) in enumerate([(0, groups[0]), (groups[0], groups[1])]):
        kk, vv = k[a:a + n].transpose(0, 1)[..., :VIS_HD], v[a:a + n].transpose(0, 1)[..., :VIS_HD]
        kp, vp = k[a:a + n + 1].transpose(0, 1)[..., :VIS_HD], v[a:a + n + 1].transpose(0, 1)[..., :VIS_HD]
        for r0, r1 in sample_row_blocks(n):
            for h0 in range(0, H, 2):
                hs = slice(h0, h0 + 2)
                vis = torch.ones(r1 - r0, n, dtype=torch.bool, device=dev)
                mistakes = {"vision scale 1/sqrt(128)": (kk[hs], vv[hs], vis, LM_SCALE)}
                if f == 0:
                    mistakes["one key past len"] = (kp[hs], vp[hs], torch.ones(r1 - r0, n + 1, dtype=torch.bool, device=dev), VIS_SCALE)
                check_rows(out[a + r0:a + r1, hs].transpose(0, 1), q[a + r0:a + r1, hs, :VIS_HD].transpose(0, 1), kk[hs], vv[hs], VIS_SCALE,
                           vis, mistakes, seen, f"frame {f} rows {r0}..{r1} heads {h0}..")
    print(f"frames: the fixture sees {sorted(seen)}")
    assert seen == {"vision scale 1/sqrt(128)", "one key past len"}


def test_bounds_vision_windows(dev, ops):
    """The 2160x3840 windows two per tile, each pair tile against fp64 attention within its own window."""
    gen = gen_on(dev, 6)
    H, groups = 16, PAIR_CASES["2160x3840 odd"]
    R = sum(groups)
    q, k, v = (rand_heads(R, H, dev, gen, 0.6, VIS_HD) for _ in range(3))
    out = run_vision(ops, vision_qkv(q, k, v, True), H, groups, True, True).view(R, H, VIS_HD)
    cu = [0] + torch.tensor(groups).cumsum(0).tolist()
    n_tiles = (len(groups) + 1) // 2
    idx = torch.full((n_tiles, 128), -1, dtype=torch.long)
    win = torch.full((n_tiles, 128), -1, dtype=torch.long)
    for t in range(n_tiles):
        a, e = cu[2 * t], cu[min(2 * t + 2, len(groups))]
        idx[t, :e - a] = torch.arange(a, e)
        win[t, :cu[2 * t + 1] - a] = 0
        win[t, cu[2 * t + 1] - a:e - a] = 1
    idx, win = idx.to(dev), win.to(dev)
    ok = idx >= 0
    g = lambda x: x[idx.clamp_min(0)].permute(0, 2, 1, 3)[..., :VIS_HD]        # [tiles, H, 128, 80]
    vis = (ok[:, None, :] & ok[:, :, None] & (win[:, None, :] == win[:, :, None]))[:, None]
    seen = set()
    mistakes = {"pair mask off": (g(k), g(v), (ok[:, None, :] & ok[:, :, None])[:, None], VIS_SCALE),
                "vision scale 1/sqrt(128)": (g(k), g(v), vis, LM_SCALE)}
    ref, ref_p = masked_ref(g(q), g(k), g(v), VIS_SCALE, vis)
    got = out[idx.clamp_min(0)].permute(0, 2, 1, 3)
    rows = ok[:, None, :, None]
    tol = attn_bound(ref.nan_to_num(0.0), ref_p.nan_to_num(0.0))
    excess = torch.where(rows, (got.double() - ref).abs() - tol, -1.0)
    assert float(excess.max()) <= 0.0, f"{int((excess > 0).sum())} elements past the bound"
    for name, (k2, v2, vis2, sc) in mistakes.items():
        wrong = masked_ref(g(q), k2, v2, sc, vis2)[0]
        if bool((((wrong - ref).abs() > 4.0 * tol) & rows).any()):
            seen.add(name)
    print(f"windows: the fixture sees {sorted(seen)}")
    assert seen == set(mistakes)


# ================================================================================================ 3. invariance
def test_invariance_offsets_neighbours_batch_and_padding(dev, ops):
    """One sequence's rows are bit-identical wherever the launch puts them: fixed stride in a batch, alone (B = 1), in the batch reversed,
    packed at other row offsets after other neighbours, and with its padding rows holding +-3.0e38 (finite in bf16; their scores overflow)
    instead of zeros. NaN in padding V rows is outside the contract: P = 0 times NaN in the P.V wgmma is NaN."""
    gen = gen_on(dev, 9)
    Hq, Hkv = 28, 4
    lens, S = [1024, 897, 1, 961, 1023, 130], 1152
    L = Layout(lens, True, S=S, device=dev)
    q, k, v = rand_heads(L.rows, Hq, dev, gen), rand_heads(L.rows, Hkv, dev, gen), rand_heads(L.rows, Hkv, dev, gen)
    pad = L.seq < 0
    q[pad], k[pad], v[pad] = 0.0, 0.0, 0.0
    qkv = lm_qkv(q, k, v)
    full = run_lm(ops, qkv, Hq, Hkv, L)
    B = len(lens)
    x = qkv.view(B, S, -1)
    for b in range(B):
        one = run_lm(ops, x[b].contiguous(), Hq, Hkv, Layout([lens[b]], True, S=S, device=dev))
        assert_bits(one, full[b * S:(b + 1) * S], f"B = 1 launch of sequence {b}")
    rev = run_lm(ops, x.flip(0).reshape(B * S, -1).contiguous(), Hq, Hkv, Layout(lens[::-1], True, S=S, device=dev))
    assert_bits(rev.view(B, S, -1).flip(0).reshape(B * S, -1), full, "batch reversed")
    # packed, in reverse order, after a 77-row neighbour: every sequence at another row offset, mid-tile
    extra = lm_qkv(rand_heads(77, Hq, dev, gen), rand_heads(77, Hkv, dev, gen), rand_heads(77, Hkv, dev, gen))
    rows = [extra] + [x[b, :lens[b]] for b in reversed(range(B))]
    Lp = Layout([r.shape[0] for r in rows], True, device=dev)
    packed = run_lm(ops, torch.cat(rows).contiguous(), Hq, Hkv, Lp)
    for i, b in enumerate(reversed(range(B))):
        a = int(Lp.start[i + 1])
        assert_bits(packed[a:a + lens[b]], full[b * S:b * S + lens[b]], f"sequence {b} packed at row {a}")
    huge = qkv.clone()
    sign = torch.randint(0, 2, (int(pad.sum()), qkv.shape[1] - 64), generator=gen, device=dev).float() * 2 - 1
    huge[pad, :-64] = (sign * 3.0e38).bfloat16()
    assert bool(torch.isfinite(huge[:, :-64].float()).all())
    assert_bits(run_lm(ops, huge, Hq, Hkv, L), full, "padding rows of +-3.0e38")
    assert bool((full[pad].view(torch.int16) == 0).all())


# ================================================================================================ 4. flash decoding
def split_rule(B, Hkv, cap):
    """decode_attn_splits: two CTAs per SM, at least 16 keys per split."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min((2 * sms + B * Hkv - 1) // (B * Hkv), (cap + 15) // 16))


@pytest.mark.parametrize("G", [1, 2, 4, 5, 7, 8])
def test_decode_selector(dev, ops, G):
    """Key-code selectors over the cache, placed against each split count's own boundaries: the winner in the first split, the last live
    key, the last key of split 0 (and a split ending exactly at len), ties across split boundaries. Slots past len hold NaN. The merge
    divides O by L in IEEE fp32: bf16(sum / count)."""
    Hkv, cap = 2, 448
    Hq = G * Hkv
    for splits in sorted({1, split_rule(12, Hkv, cap), -(-cap // 16)}):
        chunk = -(-cap // splits)
        lens = sorted({1, 2, chunk - 1, chunk, chunk + 1, 2 * chunk, 2 * chunk + 1, cap - 1, cap, min(cap, 3 * chunk), 200, 333} - {0})
        lens = [n for n in lens if 1 <= n <= cap]
        gen = torch.Generator().manual_seed(G * 1000 + splits)
        q, kc, vc, want, cnt = decode_selector(lens, Hq, Hkv, cap, chunk, gen)
        B = len(lens)
        gen_len = torch.tensor([1 + (5 * b) % n for b, n in enumerate(lens)], dtype=torch.int32)
        seq_lens = torch.tensor(lens, dtype=torch.int32) - gen_len
        out, used = ops.decode_attention(q.reshape(B, -1).bfloat16().to(dev), kc.bfloat16().to(dev), vc.bfloat16().to(dev),
                                         seq_lens.to(dev), gen_len.to(dev), Hq, LM_SCALE, splits=splits)
        torch.cuda.synchronize()
        assert used == splits
        assert int(cnt.max()) >= (4 if 2 * chunk < cap else 1)
        assert_bits(out.view(B, Hq, 128).cpu(), want, f"G = {G}, {splits} splits")


def prefill_cache(ops, qkv, Hq, Hkv, T):
    dev = qkv.device
    kc = torch.full((1, Hkv, T, 128), float("nan"), dtype=torch.bfloat16, device=dev)
    vc = kc.clone()
    ops.kv_cache_write(qkv, Hq * 128, (Hq + Hkv) * 128, Hkv, T, torch.tensor([T], dtype=torch.int32, device=dev), kc, vc)
    return kc, vc


def decode_row(ops, qkv, kc, vc, t, Hq):
    """Row t's query as a decode step: the prompt's first t keys plus the input itself at slot t."""
    dev = qkv.device
    out, _ = ops.decode_attention(qkv[t:t + 1], kc, vc, torch.tensor([t], dtype=torch.int32, device=dev),
                                  torch.ones(1, dtype=torch.int32, device=dev), Hq, LM_SCALE)
    torch.cuda.synchronize()
    return out.view(Hq, 128)


PARITY_ROWS = [0, 1, 127, 128, 4095, 7825, PROMPT - 129, PROMPT - 2, PROMPT - 1]


def test_prefill_decode_parity_selector(dev, ops):
    """A 15,616-token prompt's prefill rows and decode steps over the cache written from it: bit-identical where the tie count is 1, 2 or 4
    (1 / count is exact, so O * (1 / l) and O / L agree), and the closed form everywhere. The future keys in the cache include decoys."""
    Hq, Hkv = 28, 4
    L = Layout([PROMPT], True, S=PROMPT, device=dev)
    sel = Selector(L, Hq, Hkv, 128, gen_on(dev, 21), ties=400, tie_sizes=(2, 4))
    want, cnt = sel.expected()
    qkv = lm_qkv(*sel.tensors())
    pre = run_lm(ops, qkv, Hq, Hkv, L).view(PROMPT, Hq, 128)
    assert_bits(pre, want, "prefill")
    kc, vc = prefill_cache(ops, qkv, Hq, Hkv, PROMPT)
    checked = 0
    for t in PARITY_ROWS + torch.randint(0, PROMPT, (23,), generator=torch.Generator().manual_seed(2)).tolist():
        d = decode_row(ops, qkv, kc, vc, t, Hq)
        exact = (cnt[t] == 1) | (cnt[t] == 2) | (cnt[t] == 4)
        assert_bits(d[exact], pre[t][exact], f"decode row {t}")
        checked += int(exact.sum())
    assert checked >= 0.9 * Hq * (len(PARITY_ROWS) + 23) and int(cnt.max()) >= 2


def test_prefill_decode_parity_random(dev, ops):
    """Random inputs: the prefill row and the decode step of the same query lie within the bound of the same fp64 reference."""
    gen = gen_on(dev, 22)
    Hq, Hkv, G = 28, 4, 7
    L = Layout([PROMPT], True, S=PROMPT, device=dev)
    q, k, v = rand_heads(PROMPT, Hq, dev, gen), rand_heads(PROMPT, Hkv, dev, gen), rand_heads(PROMPT, Hkv, dev, gen)
    qkv = lm_qkv(q, k, v)
    pre = run_lm(ops, qkv, Hq, Hkv, L).view(PROMPT, Hq, 128)
    kc, vc = prefill_cache(ops, qkv, Hq, Hkv, PROMPT)
    hs = torch.arange(Hq, device=dev)
    for t in PARITY_ROWS:
        d = decode_row(ops, qkv, kc, vc, t, Hq)
        kk, vv = k[:t + 1, hs // G].transpose(0, 1), v[:t + 1, hs // G].transpose(0, 1)
        vis = torch.ones(1, t + 1, dtype=torch.bool, device=dev)
        ref, ref_p = masked_ref(q[t:t + 1].transpose(0, 1), kk, vv, LM_SCALE, vis)
        assert_attn(pre[t][:, None], ref, ref_p, f"prefill row {t}")
        assert_attn(d[:, None], ref, ref_p, f"decode row {t}")

"""The selector fixtures of tests/test_gpu_attention_d128.py checked on the CPU before any GPU run: on small shapes of every launch mode
the closed-form expected output equals plain fp64 softmax attention over the same q / k / v and mask, every runner-up is far enough below
the winner that its exp2 is +0 at the launch's scale, and every decoy wins once the mask lets it through."""
import math

import pytest
import torch

from attention_ref import DECOY_MAG, LN2, Layout, Selector, bf16_ulp, decode_selector

LM_SCALE = 128 ** -0.5
VIS_SCALE = 80 ** -0.5
MIN_GAP = 150.0             # exp2 of anything below -126 is +0 (flushed); 150 leaves room for the rounding of the scaled scores


def check_selector(sel, scale):
    want, cnt = sel.expected()
    got, gap = sel.brute(scale)
    valid = sel.L.seq >= 0
    assert bool((want[~valid].view(torch.int16) == 0).all()), "padding query rows must expect +0"
    w, g = want[valid].double(), got[valid]
    assert bool(((w - g).abs() <= 0.5 * bf16_ulp(g) * (1 + 2 ** -14) + 1e-12).all()), "closed form differs from fp64 attention"
    assert float(gap[valid].min()) >= MIN_GAP, float(gap[valid].min())
    assert int(cnt[valid].max()) >= 2, "the fixture has no ties"
    # every decoy wins for its query once visible to it
    vq, vh, dk, tgt = sel.victims
    assert len(vq) > 0
    vis = sel.L.dense_visible()
    vis[vq, dk] = True
    leak, _ = sel.brute(scale, vis)
    g_of = vh // sel.G
    assert bool((sel.mag[dk, g_of] == DECOY_MAG).all())
    moved = (leak[vq, vh] - want[vq, vh].double()).abs().amax(-1)
    assert bool((moved > 0).all()), f"{int((moved == 0).sum())} of {len(vq)} decoys change nothing when unmasked"
    return want, cnt


def test_fixed_stride_causal_gqa():
    gen = torch.Generator().manual_seed(1)
    for Hq, Hkv in [(4, 2), (7, 1), (10, 2), (8, 1), (5, 5)]:
        lens = [129, 1, 200, 256, 17]
        sel = Selector(Layout(lens, True, S=256), Hq, Hkv, 128, gen, ties=6)
        check_selector(sel, LM_SCALE)


def test_wrong_kv_head_and_dropped_diagonal_change_the_output():
    """The named kernel mistakes, restated on the fixture, move some output: q head h reading KV head h % kv_heads, and a diagonal mask."""
    gen = torch.Generator().manual_seed(2)
    L = Layout([300, 77], True, S=300)
    sel = Selector(L, 8, 2, 128, gen, ties=4)
    want, _ = sel.expected()
    right, _ = sel.brute(LM_SCALE)
    q, k, v = (t.double() for t in sel.tensors())
    vis = L.dense_visible()
    wrong_head = torch.stack([torch.softmax((q[:, h] @ k[:, h % 2].t()).masked_fill(~vis, float("-inf")), -1).nan_to_num(0.0) @ v[:, h % 2]
                              for h in range(8)], 1)[..., :128]
    assert float((wrong_head - right).abs().max()) > 0.5
    r = torch.arange(L.rows)
    no_diag = vis & (r[:, None] != r[None, :])
    dropped, _ = sel.brute(LM_SCALE, no_diag)
    assert float((dropped - right).abs().max()) > 0.5


def test_varlen_and_prefix():
    gen = torch.Generator().manual_seed(3)
    sel = Selector(Layout([130, 1, 129, 64, 255], True), 4, 2, 128, gen, ties=5)
    check_selector(sel, LM_SCALE)
    # prefixes of 129 and 127 rows, suffixes over each and one sequence without a prefix
    sel = Selector(Layout([129, 50, 200, 127, 1, 90], True, prefix_of=[-1, 0, 0, -1, 3, -1]), 4, 2, 128, gen, ties=5)
    check_selector(sel, LM_SCALE)


def test_vision_windows_and_frames():
    gen = torch.Generator().manual_seed(4)
    sel = Selector(Layout([64, 64, 16, 64, 40, 4], False), 3, 3, 80, gen, ties=4)
    check_selector(sel, VIS_SCALE)
    sel = Selector(Layout([300, 129], False), 2, 2, 80, gen, ties=8)
    want, cnt = check_selector(sel, VIS_SCALE)


def test_triple_codes():
    """More key rows than pairs of 80 dimensions: triples, whose two-dimension overlaps keep the same gaps."""
    gen = torch.Generator().manual_seed(5)
    sel = Selector(Layout([2000, 1300], False), 1, 1, 80, gen, ties=4)
    assert sel.codes.shape[1] == 3
    want, cnt = sel.expected()
    got, gap = sel.brute(VIS_SCALE)
    assert float(gap.min()) >= MIN_GAP
    assert bool(((want.double() - got).abs() <= 0.5 * bf16_ulp(got) * (1 + 2 ** -14) + 1e-12).all())


@pytest.mark.parametrize("G", [1, 2, 4, 5, 7, 8])
def test_decode_selector(G):
    gen = torch.Generator().manual_seed(G)
    Hkv, cap = 2, 100
    chunk = 16
    lens = [1, 16, 17, 32, 50, 99, 100, 64, 31]
    q, kc, vc, want, cnt = decode_selector(lens, G * Hkv, Hkv, cap, chunk, gen)
    assert int(cnt.min()) >= 1 and int(cnt.max()) >= 4
    B = len(lens)
    scale = LM_SCALE
    live = torch.arange(cap)[None, :] < torch.tensor(lens)[:, None]
    k = torch.where(live[:, None, :, None], kc, 0.0).double()
    v = torch.where(live[:, None, :, None], vc, 0.0).double()
    s = torch.einsum("bhd,bhcd->bhc", q.double() * scale, k[:, torch.arange(G * Hkv) // G]).masked_fill(~live[:, None, :], float("-inf"))
    top = s.amax(-1, keepdim=True)
    gap = (top - s.masked_fill(s == top, float("-inf")).amax(-1, keepdim=True)) / LN2
    assert float(gap.min()) >= MIN_GAP
    vh = v[:, torch.arange(G * Hkv) // G]
    ref = torch.einsum("bhc,bhcd->bhd", torch.softmax(s, -1), vh)
    assert bool(((want.double() - ref).abs() <= 0.5 * bf16_ulp(ref) * (1 + 2 ** -14) + 1e-12).all())
    # a split that ends one key early drops the last key of each split: some output moves
    drop = (torch.arange(cap)[None, :] % chunk == chunk - 1) | (torch.arange(cap)[None, :] == torch.tensor(lens)[:, None] - 1)
    ref2 = torch.einsum("bhc,bhcd->bhd", torch.softmax(s.masked_fill(drop[:, None, :], float("-inf")), -1).nan_to_num(0.0), vh)
    assert float((ref2 - ref).abs().max()) > 0.5

"""Host side of the Qwen2.5-VL scoring-path kernel entry points (no GPU needed): every refused shape or argument returns its error code before
anything is launched, and a valid call reaches the launch."""
import ctypes as C

import pytest
import torch

from t2v_metrics_b200 import _lib

OK, INVALID, CUDA_ERR, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4, -5

# Fake device addresses: these checks run only where no device exists, so a check that failed to refuse could never reach a kernel; there
# a call that passes every check stops at the launch (or the tensor-map build) with VQA_ERR_CUDA.
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="argument checks run with fake device addresses, only where no device exists")
P = C.c_void_p(1 << 20)             # a 256-byte aligned fake device address


def at(offset):
    return C.c_void_p((1 << 20) + offset)


# 7B text layer: 28 query heads over 4 KV heads in one packed qkv row of 36 * 128 columns
HQ, HKV = 28, 4
LD = (HQ + 2 * HKV) * 128


@no_device
def test_attention_d128_argument_checks():
    lib = _lib.load()

    def call(qkv=P, ld=LD, rows=4 * 320, q0=0, k0=HQ * 128, v0=(HQ + HKV) * 128, out=P, ldo=HQ * 128, n_seq=4, max_len=320, S=320, Hq=HQ,
             group=HQ // HKV, cu=None, lens=P):
        return lib.vqa_op_attention_d128(qkv, ld, rows, q0, k0, v0, out, ldo, n_seq, max_len, S, Hq, group, cu, lens, 0.088, 1, None)

    assert call() == CUDA_ERR and call(lens=None) == CUDA_ERR
    assert call(rows=4 * 320 + 7) == CUDA_ERR and call(max_len=400) == CUDA_ERR
    # fixed stride: every written row inside `rows`, S >= 1, the grid covering all S rows
    assert call(rows=4 * 320 - 1) == INVALID and call(n_seq=5) == INVALID
    assert call(S=0) == INVALID and call(S=0, max_len=1) == INVALID and call(max_len=319) == INVALID
    assert call(cu=P, S=0) == CUDA_ERR                                    # variable length: S unused
    # GQA: q_heads a multiple of kv_group
    assert call(group=6) == INVALID and call(group=0) == INVALID and call(Hq=27) == INVALID
    for g in (1, 2, 4, 7, 14, 28):
        kv = HQ // g
        assert call(group=g, ld=(HQ + 2 * kv) * 128, v0=(HQ + kv) * 128) == CUDA_ERR, g
    # 8-element alignment of ld, ldo and the column offsets; 16-byte aligned pointers
    assert call(ld=LD + 4) == INVALID and call(ldo=HQ * 128 + 4) == INVALID
    for k in ("q0", "k0", "v0"):
        assert call(**{k: {"q0": 0, "k0": HQ * 128, "v0": (HQ + HKV) * 128}[k] + 4}) == INVALID, k
    assert call(qkv=at(8)) == INVALID and call(out=at(8)) == INVALID
    # every head inside its row
    assert call(v0=(HQ + HKV) * 128 + 8) == INVALID and call(ld=LD - 8) == INVALID and call(ldo=HQ * 128 - 8) == INVALID
    assert call(q0=-8) == INVALID and call(q0=9 * 128) == INVALID
    assert call(rows=0) == INVALID and call(n_seq=0) == INVALID and call(Hq=0) == INVALID
    for k in ("qkv", "out"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_attention_d128_ex_argument_checks():
    lib = _lib.load()
    H, hd = 16, 80                  # the 7B vision tower: 16 heads of 80 dims in 128-wide slots, compact output

    def call(qkv=P, ld=3 * H * 128, rows=4096, q0=0, k0=H * 128, v0=2 * H * 128, out=P, ldo=H * hd, n_seq=64, max_len=64, Hq=H, group=1, cu=P,
             kvp=None, causal=0, pair=1, ohs=hd, d_out=hd):
        return lib.vqa_op_attention_d128_ex(qkv, ld, rows, q0, k0, v0, out, ldo, n_seq, max_len, Hq, group, cu, kvp, 0.11, causal, pair, ohs, d_out,
                                            None)

    assert call() == CUDA_ERR and call(pair=0, max_len=1024) == CUDA_ERR
    assert call(pair=0, causal=1, kvp=P, ld=(HQ + 2 * HKV) * 128, Hq=HQ, group=7, k0=HQ * 128, v0=(HQ + 4) * 128, ldo=HQ * 128, ohs=128,
                d_out=128) == CUDA_ERR
    # pair_sequences: <= 64 rows, non-causal, no shared prefix
    assert call(max_len=65) == INVALID and call(causal=1) == INVALID and call(kvp=P) == INVALID
    assert call(cu=None) == INVALID and call(cu=None, pair=0) == INVALID
    # output heads: 8 <= d_out <= 128, multiples of 8, inside o_head_stride and ldo
    assert call(d_out=84) == INVALID and call(d_out=0) == INVALID and call(d_out=136, ohs=136, ldo=H * 136) == INVALID
    assert call(ohs=84) == INVALID and call(ohs=72) == INVALID and call(ldo=H * hd - 8) == INVALID
    assert call(d_out=128, ohs=128, ldo=H * 128) == CUDA_ERR
    assert call(group=3) == INVALID and call(ld=3 * H * 128 + 4) == INVALID and call(k0=H * 128 + 4) == INVALID
    assert call(v0=2 * H * 128 + 8) == INVALID and call(qkv=at(8)) == INVALID and call(out=at(8)) == INVALID


@no_device
def test_qwen_rope_argument_checks():
    lib = _lib.load()

    def call(pos=P, rows=320, axis=P, inv=P, half=64, cos=P, sin=P, x=P, ld=LD, col0=0, n_heads=HQ + HKV, hs=128, hd=128, text=1):
        return lib.vqa_op_qwen_rope(pos, rows, axis, inv, half, cos, sin, x, ld, col0, n_heads, hs, hd, text, None)

    assert call() == CUDA_ERR and call(text=0) == CUDA_ERR
    vis = dict(ld=3 * 16 * 128, n_heads=32, half=40, hd=80)                # the vision tower: q and k of 16 heads, 80 of 128 dims
    assert call(**vis, text=0) == CUDA_ERR
    assert call(**dict(vis, hd=88, half=44)) == INVALID                    # head_dim % 16
    assert call(hd=144, half=72) == INVALID                                # head_dim > head_stride
    assert call(half=32) == INVALID and call(**dict(vis, half=64)) == INVALID   # the tables must be head_dim wide
    assert call(x=at(8)) == INVALID and call(cos=at(8)) == INVALID and call(sin=at(4)) == INVALID
    assert call(ld=LD + 4) == INVALID and call(col0=4) == INVALID and call(hs=132, ld=36 * 132) == INVALID
    assert call(col0=4 * 128 + 8) == INVALID and call(n_heads=37) == INVALID and call(col0=-8) == INVALID   # heads past ld
    assert call(col0=4 * 128, n_heads=HQ + 2 * HKV - 4) == CUDA_ERR
    assert call(rows=0) == INVALID and call(n_heads=0) == INVALID and call(hd=0, half=0) == INVALID
    for k in ("pos", "axis", "inv", "cos", "sin", "x"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_gather_rows_argument_checks():
    lib = _lib.load()

    def call(src=P, dst=P, idx=P, rows=1024, group=4, D=1280):
        return lib.vqa_op_gather_rows(src, dst, idx, rows, group, D, None)

    assert call() == CUDA_ERR and call(group=1, rows=1023) == CUDA_ERR
    assert call(rows=1022) == INVALID and call(D=1284) == INVALID and call(D=0) == INVALID and call(group=0) == INVALID and call(rows=0) == INVALID
    assert call(src=at(8)) == INVALID and call(dst=at(8)) == INVALID
    for k in ("src", "dst", "idx"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_qwen_embed_argument_checks():
    lib = _lib.load()

    def call(ids=P, feat=P, lens=P, emb=P, feats=P, out=P, rows=4 * 330, S=330, D=3584):
        return lib.vqa_op_qwen_embed(ids, feat, lens, emb, feats, out, rows, S, D, None)

    assert call() == CUDA_ERR and call(rows=1001, S=1001) == CUDA_ERR          # packed rows: one sequence of all rows
    assert call(rows=4 * 330 + 1) == INVALID and call(S=0) == INVALID and call(rows=0) == INVALID
    assert call(D=3580) == INVALID and call(D=0) == INVALID
    for k in ("emb", "feats", "out"):
        assert call(**{k: at(8)}) == INVALID, k
    for k in ("ids", "feat", "lens", "emb", "feats", "out"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_token_bitmap_argument_checks():
    lib = _lib.load()

    def call(ids=P, lens=P, B=4, S=330, cu=None, kvp=None, pair=None, maxp=0, vocab=152064, bm=P):
        return lib.vqa_op_token_bitmap(ids, lens, B, S, cu, kvp, pair, maxp, vocab, bm, None)

    assert call() == CUDA_ERR
    assert call(lens=None, S=0, cu=P, kvp=P, pair=P, maxp=330) == CUDA_ERR and call(lens=None, S=0, cu=P, pair=P, maxp=330) == CUDA_ERR
    assert call(lens=None) == INVALID and call(S=0) == INVALID                  # padded rows
    assert call(cu=P, pair=None, maxp=330) == INVALID and call(cu=P, pair=P, maxp=0) == INVALID   # packed rows
    assert call(B=0) == INVALID and call(vocab=0) == INVALID and call(bm=at(2)) == INVALID
    assert call(ids=None) == INVALID and call(bm=None) == INVALID


@no_device
def test_topk_softmax_argument_checks():
    lib = _lib.load()

    def call(logits=P, ldl=152064, B=4, V=152064, T=1.0, pen=None, rp=1.0, K=5, ids=P, probs=P):
        return lib.vqa_op_topk_softmax(logits, ldl, B, V, T, pen, rp, K, ids, probs, None)

    for K in (1, 5, 8):
        assert call(K=K) == CUDA_ERR, K
    assert call(pen=P, rp=1.3) == CUDA_ERR and call(V=1000, ldl=1000, T=0.5) == CUDA_ERR and call(V=1000) == CUDA_ERR
    assert call(K=0) == INVALID and call(K=9) == INVALID and call(ldl=152063) == INVALID
    assert call(T=0.0) == INVALID and call(T=-1.0) == INVALID and call(rp=0.0) == INVALID and call(T=float("nan")) == INVALID
    assert call(B=0) == INVALID and call(V=0) == INVALID and call(logits=at(1)) == INVALID and call(pen=at(2), rp=1.3) == INVALID
    for k in ("logits", "ids", "probs"):
        assert call(**{k: None}) == INVALID, k


def lmhead_scratch_bytes(M, N):
    """lse_max and lse_sum (M x 2 partials per 128 columns each), the label logits [M] and the scores [M]: no slot shared."""
    return 4 * (2 * M * 2 * ((N + 127) // 128) + 2 * M)


@no_device
def test_lmhead_logprob_scratch_and_argument_checks():
    lib = _lib.load()
    need = C.c_size_t(0)

    def call(h=P, ldh=3584, w=P, ldw=3584, M=7, N=152064, K=3584, labels=P, T=1.0, pen=None, rp=1.0, out=P, scratch=P, nbytes=1 << 30):
        need.value = 0
        return lib.vqa_op_lmhead_logprob(h, ldh, w, ldw, M, N, K, labels, T, pen, rp, out, scratch, nbytes, C.byref(need), None)

    assert call() == CUDA_ERR and need.value == lmhead_scratch_bytes(7, 152064)
    for M, N in ((1, 1000), (64, 130), (128, 32128)):
        n = lmhead_scratch_bytes(M, N)
        assert call(M=M, N=N, nbytes=n - 1) == WORKSPACE and need.value == n
        assert call(M=M, N=N, nbytes=n) == CUDA_ERR
    assert call(scratch=None) == WORKSPACE and need.value == lmhead_scratch_bytes(7, 152064)
    assert call(T=0.5, pen=P, rp=1.3) == CUDA_ERR and call(T=2.0, pen=P, rp=0.8) == CUDA_ERR
    assert call(T=0.0) == INVALID and call(rp=0.0) == INVALID and call(rp=-1.3) == INVALID
    assert call(K=3580) == INVALID and call(ldh=3588) == INVALID and call(ldw=2048) == INVALID and call(M=0) == INVALID and call(N=0) == INVALID
    assert call(h=at(8)) == INVALID and call(w=at(8)) == INVALID and call(pen=at(2), rp=1.3) == INVALID
    for k in ("h", "w", "labels", "out"):
        assert call(**{k: None}) == INVALID, k

"""Host side of the CLIP-FlanT5 scoring-path kernel entry points (no GPU needed): every refused shape or argument returns its error code
before anything is launched, and a valid call reaches the launch."""
import ctypes as C

import pytest
import torch

from t2v_metrics_b200 import _lib

OK, INVALID, CUDA_ERR, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4, -5

# Fake device addresses: these checks run only where no device exists, so a check that failed to refuse could never reach a kernel; there
# a call that passes every check stops at the launch with VQA_ERR_CUDA.
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="argument checks run with fake device addresses, only where no device exists")
P = C.c_void_p(1 << 20)             # a 256-byte aligned fake device address


def at(offset):
    return C.c_void_p((1 << 20) + offset)


@no_device
def test_f32acc_gemm_argument_checks():
    lib = _lib.load()

    def call(A=P, lda=1024, W=P, ldw=1024, w_rows=1024, Cp=P, ldc=1024, M=577, N=1024, K=1024, bias=P, variant=0):
        return lib.vqa_op_gemm_bf16_f32acc(A, lda, W, ldw, w_rows, Cp, ldc, M, N, K, bias, variant, None)

    assert call() == CUDA_ERR and call(bias=None) == CUDA_ERR
    for v in (2561, 2562, 1281, 1282, 641, 321):
        assert call(variant=v) == CUDA_ERR, v
    assert call(variant=7) == INVALID and call(variant=2560) == INVALID
    assert call(N=1000, ldc=1004) == CUDA_ERR                     # an N tail, ldc a multiple of 4
    assert call(ldc=1020) == INVALID and call(ldc=1026) == INVALID  # narrower than N / not a multiple of 4
    assert call(N=1004, ldc=1004) == INVALID and call(K=1020) == INVALID and call(lda=1028) == INVALID and call(lda=512) == INVALID
    assert call(ldw=1028) == INVALID and call(ldw=512) == INVALID
    assert call(A=at(8)) == INVALID and call(W=at(8)) == INVALID and call(Cp=at(8)) == INVALID and call(bias=at(4)) == INVALID
    assert call(bias=at(8)) == CUDA_ERR
    for k in ("A", "W", "Cp"):
        assert call(**{k: None}) == INVALID, k
    assert call(M=0) == INVALID and call(N=0) == INVALID and call(K=0) == INVALID and call(w_rows=0) == INVALID


# The four batched launches of the absorbed cross-attention (clipt5_absorbed_cross_attention) at clip-flant5-xxl width, T = 1, S = 605.
H, DM, B, T, S = 64, 4096, 3, 1, 605
SP, TH, MD, INNER = 608, 64, 3, 64 * 64
PRODUCTION = {
    "q~ = Wk^T q":     dict(M=MD, N=DM, K=64, lda=INNER, ldw=INNER, ldc=H * DM, nb=H, a_off=(0, 64), w_off=(0, 64), c_stride=DM,
                            a_ext=(MD, INNER), w_ext=(DM, INNER), variant=2561),
    "scores":          dict(M=TH, N=SP, K=DM, lda=DM, ldw=DM, ldc=SP, nb=B, a_off=(TH, 0), w_off=(S, 0), c_stride=TH * SP,
                            a_ext=(B * TH, DM), w_ext=(B * S, DM), variant=1281),
    "ctx = P x":       dict(M=TH, N=DM, K=SP, lda=SP, ldw=SP, ldc=DM, nb=B, a_off=(TH, 0), w_off=(DM, 0), c_stride=TH * DM,
                            a_ext=(B * TH, SP), w_ext=(B * DM, SP), variant=2561),
    "out = Wv ctx":    dict(M=MD, N=64, K=DM, lda=H * DM, ldw=DM, ldc=INNER, nb=H, a_off=(0, DM), w_off=(64, 0), c_stride=64,
                            a_ext=(MD, H * DM), w_ext=(INNER, DM), variant=641),
}


def batched_call(lib, A=P, W=P, Cp=P, **over):
    s = dict(PRODUCTION["scores"])
    s.update(over)
    return lib.vqa_op_gemm_bf16_batched(A, s["lda"], W, s["ldw"], Cp, s["ldc"], s["M"], s["N"], s["K"], s["nb"], s["a_off"][0], s["a_off"][1],
                                        s["w_off"][0], s["w_off"][1], s["c_stride"], s["a_ext"][0], s["a_ext"][1], s["w_ext"][0], s["w_ext"][1],
                                        s["variant"], None)


@no_device
@pytest.mark.parametrize("name", list(PRODUCTION))
def test_batched_gemm_accepts_the_production_launches(name):
    """Including the score GEMM, whose last batch reads Sp - S encoder rows past w_rows (TMA zero fill)."""
    assert batched_call(_lib.load(), **PRODUCTION[name]) == CUDA_ERR


@no_device
def test_batched_gemm_argument_checks():
    lib = _lib.load()
    call = lambda **kw: batched_call(lib, **kw)
    assert call() == CUDA_ERR
    # every batch's first row inside the extents: the last batch starts at (nb - 1) * offset
    assert call(a_ext=(2 * TH, DM)) == INVALID and call(a_ext=(2 * TH + 1, DM)) == CUDA_ERR
    assert call(w_ext=(2 * S, DM)) == INVALID and call(w_ext=(2 * S + 1, DM)) == CUDA_ERR
    assert call(nb=4) == INVALID
    # every batch's K columns inside the extents
    q = dict(PRODUCTION["q~ = Wk^T q"])
    assert call(**q) == CUDA_ERR
    assert call(**dict(q, a_ext=(MD, INNER - 8))) == INVALID and call(**dict(q, w_ext=(DM, INNER - 8))) == INVALID
    assert call(**dict(q, a_off=(0, 72))) == INVALID and call(**dict(q, w_off=(0, 72))) == INVALID
    assert call(**dict(q, nb=H + 1)) == INVALID
    assert call(a_ext=(B * TH, DM + 8)) == INVALID and call(w_ext=(B * S, DM + 8)) == INVALID    # extents wider than the rows
    assert call(ldc=SP - 8) == INVALID and call(ldc=SP + 4) == INVALID and call(c_stride=TH * SP + 4) == INVALID
    assert call(N=SP + 4, ldc=SP + 8) == INVALID and call(K=DM - 4) == INVALID and call(lda=DM + 4) == INVALID
    assert call(a_off=(-1, 0)) == INVALID and call(w_off=(0, -8)) == INVALID and call(c_stride=-8) == INVALID
    assert call(nb=0) == INVALID and call(M=0) == INVALID and call(a_ext=(0, DM)) == INVALID
    assert call(variant=2560) == INVALID and call(variant=0) == CUDA_ERR
    assert call(A=at(8)) == INVALID and call(W=at(8)) == INVALID and call(Cp=at(8)) == INVALID
    for k in ("A", "W", "Cp"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_batched_gemm_k_tail_needs_one_operand_extent_at_k():
    """The kernel reads K in 64-column k blocks clipped only at the extents: with K % 64 != 0 the tail block of every batch adds the
    products of columns K .. roundup(K, 64), which vanish only when A's or W's extent ends at K (TMA zero fill). Refused otherwise, for
    one batch, K-offset batches and row-offset batches alike; accepted with an extent at K (the `ctx = P x` launch has K = a_cols = Sp = 608)."""
    lib = _lib.load()
    call = lambda **kw: batched_call(lib, **kw)
    q = dict(PRODUCTION["q~ = Wk^T q"], K=72, lda=72 * H, ldw=72 * H, a_off=(0, 72), w_off=(0, 72), a_ext=(MD, 72 * H), w_ext=(DM, 72 * H))
    assert call(**q) == INVALID
    assert call(**dict(q, w_off=(0, 0))) == INVALID and call(**dict(q, a_off=(0, 0))) == INVALID
    assert call(**dict(q, nb=1)) == INVALID                                   # one batch: a 128-term dot product
    assert call(**dict(q, nb=1, a_ext=(MD, 72))) == CUDA_ERR and call(**dict(q, nb=1, w_ext=(DM, 72))) == CUDA_ERR
    assert call(**dict(q, a_off=(0, 0), a_ext=(MD, 72))) == CUDA_ERR       # W offset along K, A's tail zero-filled in every batch
    assert call(**dict(q, K=128, a_off=(0, 128), w_off=(0, 128), lda=128 * H, ldw=128 * H, a_ext=(MD, 128 * H), w_ext=(DM, 128 * H))) == CUDA_ERR
    assert call(K=DM - 8) == INVALID                                          # rows-offset scores launch: columns DM - 8 .. DM would be added
    assert call(K=DM - 8, a_ext=(B * TH, DM - 8)) == CUDA_ERR and call(K=DM - 8, w_ext=(B * S, DM - 8)) == CUDA_ERR
    assert call(**PRODUCTION["ctx = P x"]) == CUDA_ERR


def cross_attn_workspace(B, T, S, H, Dm):
    """The documented mode-0 layout: xt | q~ | csc | ctx, each at the next multiple of 256 bytes."""
    r = lambda n: (n + 255) // 256 * 256
    Sp, TH = (S + 7) // 8 * 8, T * H
    return r(B * Dm * Sp * 2) + r(B * TH * Dm * 2) + r((B * TH + 256) * Sp * 2) + r(B * TH * Dm * 2)


@no_device
def test_cross_attention_argument_checks():
    lib = _lib.load()
    need = C.c_size_t(0)

    def call(q=P, x=P, sl=P, wkT=P, wkv=P, out=P, B=3, T=2, S=605, H=64, Dm=4096, mode=0, ws=P, ws_bytes=1 << 34):
        need.value = 0
        return lib.vqa_op_t5_cross_attention(q, x, sl, wkT, wkv, out, B, T, S, H, Dm, mode, 1, ws, ws_bytes, C.byref(need), None)

    assert call() == CUDA_ERR and need.value == cross_attn_workspace(3, 2, 605, 64, 4096)
    assert call(B=64, T=1, S=83) == CUDA_ERR and need.value == cross_attn_workspace(64, 1, 83, 64, 4096)
    assert call(T=33, H=4, Dm=256) == CUDA_ERR and need.value == cross_attn_workspace(3, 33, 605, 4, 256)
    assert call(mode=1) == CUDA_ERR and need.value == (3 * 605 * 2 * 64 * 64 * 2 + 255) // 256 * 256
    assert call(mode=1, wkT=None) == CUDA_ERR and call(mode=0, wkT=None) == INVALID
    assert call(mode=1, T=8) == CUDA_ERR and call(mode=1, T=9) == UNSUPPORTED and call(mode=0, T=9) == CUDA_ERR
    assert call(mode=2) == INVALID and call(mode=-1) == INVALID
    n0 = cross_attn_workspace(3, 2, 605, 64, 4096)
    assert call(ws_bytes=n0 - 1) == WORKSPACE and need.value == n0 and call(ws_bytes=n0) == CUDA_ERR
    assert call(ws=None) == WORKSPACE and call(ws=at(128)) == INVALID
    assert call(Dm=4092) == INVALID and call(B=0) == INVALID and call(T=0) == INVALID and call(S=0) == INVALID and call(H=0) == INVALID
    for k in ("q", "x", "wkT", "wkv", "out"):
        assert call(**{k: at(8)}) == INVALID, k
    for k in ("q", "x", "sl", "wkv", "out"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_attention_d64_argument_checks():
    """Every call the head-dim-64 kernel cannot serve is refused before the tensor-map build: misaligned TMA rows or output rows (the kernel's
    4-byte stores to a misaligned `out` would fault), misaligned lengths or bias entries, int32 overflow of the row, column or work-item
    arithmetic, and a bias row longer than shared memory holds next to the 2-stage K/V ring (S = 16,496 is the longest that fits)."""
    lib = _lib.load()
    I32_MAX = 2 ** 31 - 1

    def call(qkv=P, out=P, B=2, S=672, H=64, lens=P, table=P, const_from=128, round_scores=1):
        return lib.vqa_op_attention_d64(qkv, out, B, S, H, lens, table, 1.0, const_from, round_scores, None)

    assert call() == CUDA_ERR and call(round_scores=0, const_from=0) == CUDA_ERR
    assert call(lens=None) == CUDA_ERR and call(table=None) == CUDA_ERR and call(lens=None, table=None) == CUDA_ERR
    # alignment: qkv / out rows are TMA rows and 16-byte output rows, seq_lens / bias_table are read as 4-byte words
    assert call(qkv=at(8)) == INVALID and call(out=at(2)) == INVALID and call(out=at(8)) == INVALID
    assert call(qkv=at(16)) == CUDA_ERR and call(out=at(16)) == CUDA_ERR
    assert call(table=at(2)) == INVALID and call(lens=at(2)) == INVALID
    assert call(table=at(4)) == CUDA_ERR and call(lens=at(4)) == CUDA_ERR
    # the bias row: 4 stages up to S = 8,304, 3 up to 12,400, 2 up to 16,496, refused past that; without a table S is not limited by it
    for S in (8304, 8305, 12400, 12401, 16496):
        assert call(B=1, H=2, S=S) == CUDA_ERR, S
    assert call(B=1, H=2, S=16497) == INVALID and call(B=1, H=2, S=16497, const_from=0) == INVALID
    assert call(B=1, H=2, S=16497, table=None) == CUDA_ERR and call(B=1, H=2, S=1 << 20, table=None) == CUDA_ERR
    # int32 arithmetic: the qkv row of 3 * H * 64 columns, B * S rows, H * B * ceil(S / 128) work items
    h_max = I32_MAX // (3 * 64)
    assert call(B=1, S=1, H=h_max, table=None) == CUDA_ERR and call(B=1, S=1, H=h_max + 1, table=None) == INVALID
    assert call(B=1 << 16, S=(1 << 15) - 1, H=1, table=None) == CUDA_ERR and call(B=1 << 16, S=1 << 15, H=1, table=None) == INVALID
    assert call(B=(1 << 24) - 1, S=128, H=128, table=None) == CUDA_ERR and call(B=(1 << 24) - 1, S=128, H=129, table=None) == INVALID
    assert call(B=(1 << 24) - 1, S=1, H=128, table=None) == CUDA_ERR and call(B=(1 << 24) - 1, S=1, H=129, table=None) == INVALID
    assert call(B=1, S=I32_MAX, H=1, table=None) == CUDA_ERR       # ceil(S / 128) without overflowing S + 127
    # null pointers and sizes below 1
    assert call(qkv=None) == INVALID and call(out=None) == INVALID
    for kw in ("B", "S", "H"):
        assert call(**{kw: 0}) == INVALID and call(**{kw: -1}) == INVALID, kw


@no_device
def test_layernorm_f32_argument_checks():
    lib = _lib.load()

    def call(x=P, g=P, b=P, y=P, rows=1731, D=1024):
        return lib.vqa_op_layernorm_f32(x, g, b, y, rows, D, 1e-5, None)

    for D in (256, 512, 768, 1024):
        assert call(D=D) == CUDA_ERR, D
    for D in (128, 1280, 1000, 0):
        assert call(D=D) == UNSUPPORTED, D
    assert call(rows=0) == INVALID
    for k in ("x", "g", "b", "y"):
        assert call(**{k: None}) == INVALID and call(**{k: at(8)}) == INVALID, k


@no_device
def test_clip_embed_ln_argument_checks():
    lib = _lib.load()

    def call(patch=P, cls=P, pos=P, g=P, b=P, y=P, n=3, Pn=576, D=1024):
        return lib.vqa_op_clip_embed_ln(patch, cls, pos, g, b, y, n, Pn, D, 1e-5, None)

    assert call() == CUDA_ERR and call(D=256, Pn=16) == CUDA_ERR
    for D in (512, 768, 1280, 0):
        assert call(D=D) == UNSUPPORTED, D
    assert call(n=0) == INVALID and call(Pn=0) == INVALID
    for k in ("patch", "cls", "pos", "g", "b", "y"):
        assert call(**{k: None}) == INVALID and call(**{k: at(8)}) == INVALID, k

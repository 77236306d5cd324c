"""Host side of the CLIP-FlanT5 glue-kernel entry points (patch gather, multimodal splice, decoder embedding, bias table, lm_head score,
row sums of squares) and of vqa_op_norm, no GPU needed: every refused shape, null pointer or misaligned pointer returns its error code before
anything is launched, and a valid call reaches the launch."""
import ctypes as C

import pytest
import torch

from t2v_metrics_b200 import _lib

OK, INVALID, CUDA_ERR, WORKSPACE = 0, -1, -3, -4

# Fake device addresses: these checks run only where no device exists, so a check that failed to refuse could never reach a kernel; there
# a call that passes every check stops at the launch with VQA_ERR_CUDA.
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="argument checks run with fake device addresses, only where no device exists")
P = C.c_void_p(1 << 20)             # a 256-byte aligned fake device address
F32, BF16, I32 = _lib.VQA_DTYPE_F32, _lib.VQA_DTYPE_BF16, _lib.VQA_DTYPE_I32


def at(offset):
    return C.c_void_p((1 << 20) + offset)


@no_device
def test_patchify_argument_checks():
    lib = _lib.load()

    def call(pix=P, dt=F32, n=3, size=336, patch=14, kpad=640, out=P):
        return lib.vqa_op_patchify(pix, dt, n, size, patch, kpad, out, None)

    assert call() == CUDA_ERR and call(dt=BF16) == CUDA_ERR and call(size=28, kpad=592) == CUDA_ERR
    assert call(dt=I32) == INVALID and call(dt=7) == INVALID
    assert call(kpad=584) == INVALID and call(kpad=644) == INVALID and call(kpad=592) == CUDA_ERR   # >= 588 and a multiple of 8
    assert call(n=0) == INVALID and call(patch=0) == INVALID and call(size=13) == INVALID
    assert call(pix=at(2)) == INVALID and call(pix=at(2), dt=BF16) == CUDA_ERR and call(pix=at(1), dt=BF16) == INVALID
    assert call(out=at(8)) == INVALID
    for k in ("pix", "out"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_splice_embed_argument_checks():
    lib = _lib.load()

    def call(ids=P, lens=P, index=P, shared=P, feats=P, ldf=4096, off=1, rows=577, out=P, sl=P, B=64, L=96, Pn=576, D=4096, tok=-200):
        return lib.vqa_op_splice_embed(ids, lens, index, shared, feats, ldf, off, rows, out, sl, B, L, Pn, D, tok, None)

    assert call() == CUDA_ERR and call(index=None) == CUDA_ERR
    assert call(B=3, L=12, Pn=16, rows=17, D=256, ldf=256) == CUDA_ERR        # the tiny config
    assert call(off=0, rows=576) == CUDA_ERR and call(ldf=4104) == CUDA_ERR
    assert call(off=2) == INVALID and call(rows=576) == INVALID and call(off=-1) == INVALID   # P feature rows must fit in the block
    assert call(ldf=4092) == INVALID and call(ldf=2048) == INVALID and call(D=4092, ldf=4096) == INVALID
    assert call(B=0) == INVALID and call(L=0) == INVALID and call(Pn=0) == INVALID and call(D=0) == INVALID
    for k in ("shared", "feats", "out"):
        assert call(**{k: at(8)}) == INVALID, k
    for k in ("ids", "lens", "index", "sl"):
        assert call(**{k: at(2)}) == INVALID, k
    for k in ("ids", "lens", "shared", "feats", "out", "sl"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_decoder_embed_argument_checks():
    lib = _lib.load()

    def call(labels=P, shared=P, out=P, B=64, T=2, D=4096, start=0, pad=0):
        return lib.vqa_op_decoder_embed(labels, shared, out, B, T, D, start, pad, None)

    assert call() == CUDA_ERR and call(T=256, D=256) == CUDA_ERR
    assert call(labels=None, T=1) == CUDA_ERR and call(labels=None, T=2) == INVALID      # labels NULL only for the start token
    assert call(B=0) == INVALID and call(T=0) == INVALID and call(D=0) == INVALID and call(D=4092) == INVALID
    assert call(start=-1) == INVALID and call(pad=-100) == INVALID
    assert call(labels=at(2)) == INVALID and call(shared=at(8)) == INVALID and call(out=at(8)) == INVALID
    for k in ("shared", "out"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_bias_table_argument_checks():
    lib = _lib.load()

    def call(rel=P, lut=P, maxd=128, table=P, H=64, S=672):
        return lib.vqa_op_t5_bias_table(rel, lut, maxd, table, H, S, None)

    assert call() == CUDA_ERR and call(S=1) == CUDA_ERR and call(rel=at(2)) == CUDA_ERR
    assert call(H=0) == INVALID and call(S=0) == INVALID and call(maxd=0) == INVALID
    assert call(rel=at(1)) == INVALID and call(lut=at(2)) == INVALID and call(table=at(2)) == INVALID
    for k in ("rel", "lut", "table"):
        assert call(**{k: None}) == INVALID, k


def lmhead_scratch_bytes(M, N):
    """lse_max and lse_sum [M, 2 * ceil(N / 128)] each, the label logits [M] and the (unused) scores [M], in floats."""
    parts = 2 * ((N + 127) // 128)
    return 4 * (2 * M * parts + 2 * M)


@no_device
def test_lmhead_score_argument_checks():
    lib = _lib.load()
    need = C.c_size_t(0)

    def call(h=P, ldh=4096, w=P, ldw=4096, B=64, T=2, N=32128, K=4096, labels=P, scores=P, logp=P, scratch=P, nbytes=1 << 34):
        need.value = 0
        return lib.vqa_op_lmhead_score(h, ldh, w, ldw, B, T, N, K, labels, scores, logp, scratch, nbytes, C.byref(need), None)

    assert call() == CUDA_ERR and need.value == lmhead_scratch_bytes(128, 32128)
    assert call(logp=None) == CUDA_ERR and call(B=3, T=33, N=1000, K=256, ldh=256, ldw=256) == CUDA_ERR
    assert need.value == lmhead_scratch_bytes(99, 1000)
    n0 = lmhead_scratch_bytes(128, 32128)
    assert call(nbytes=n0 - 1) == WORKSPACE and need.value == n0 and call(nbytes=n0) == CUDA_ERR
    assert call(scratch=None) == WORKSPACE and call(scratch=at(2)) == WORKSPACE
    assert call(K=4092) == INVALID and call(ldh=4092) == INVALID and call(ldw=2048) == INVALID
    assert call(B=0) == INVALID and call(T=0) == INVALID and call(N=0) == INVALID and call(K=0) == INVALID
    assert call(h=at(8)) == INVALID and call(w=at(8)) == INVALID
    for k in ("labels", "scores", "logp"):
        assert call(**{k: at(2)}) == INVALID, k
    for k in ("h", "w", "labels", "scores"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_row_ssq_argument_checks():
    lib = _lib.load()

    def call(x=P, ssq=P, rows=64 * 672, D=4096, stride=128):
        return lib.vqa_op_row_ssq(x, ssq, rows, D, stride, None)

    assert call() == CUDA_ERR and call(D=256, stride=1) == CUDA_ERR
    assert call(rows=0) == INVALID and call(D=0) == INVALID and call(D=4092) == INVALID and call(stride=0) == INVALID
    assert call(x=at(8)) == INVALID and call(ssq=at(2)) == INVALID
    for k in ("x", "ssq"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_rmsnorm_argument_checks():
    """Before these checks vqa_op_norm refused null pointers only: rows = 0 returned OK, and a misaligned pointer reached the 16-byte loads."""
    lib = _lib.load()

    def call(x=P, g=P, y=P, rows=1000, D=4096):
        return lib.vqa_op_norm(x, g, y, rows, D, 1e-6, None)

    for D in (256, 512, 1024, 1280, 2048, 3584, 4096, 4104, 5120, 8192, 8):
        assert call(D=D) == CUDA_ERR, D
    for D in (0, -256, 4100, 8200):
        assert call(D=D) == INVALID, D
    assert call(rows=0) == INVALID and call(rows=-1) == INVALID
    for k in ("x", "g", "y"):
        assert call(**{k: at(8)}) == INVALID and call(**{k: None}) == INVALID, k

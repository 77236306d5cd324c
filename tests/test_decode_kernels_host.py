"""Host side of the decode-loop kernel entry points (no GPU needed): the engine's T5 relative-position bucket table against transformers,
and the argument checks of the kernel-level entry points, which must refuse a bad call before anything is launched."""
import ctypes as C

import pytest
import torch

from t2v_metrics_b200 import _lib
from t2v_metrics_b200.engine import ops

OK, INVALID, CUDA_ERR, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4, -5


@pytest.mark.parametrize("num_buckets,max_distance", [(32, 128), (32, 64), (16, 32), (64, 256)])
@pytest.mark.parametrize("bidirectional", [True, False])
def test_bucket_table_matches_hf(bidirectional, num_buckets, max_distance):
    from transformers.models.t5.modeling_t5 import T5Attention
    got = ops.t5_bucket_lut(bidirectional, num_buckets, max_distance)
    rel = torch.arange(-max_distance, max_distance + 1)
    ref = T5Attention._relative_position_bucket(rel, bidirectional=bidirectional, num_buckets=num_buckets, max_distance=max_distance)
    assert torch.equal(got.long(), ref)
    # beyond the table the buckets saturate, which is what lets the kernels clamp rel to [-max_distance, max_distance]
    far = torch.tensor([-10 * max_distance, 10 * max_distance])
    assert torch.equal(T5Attention._relative_position_bucket(far, bidirectional=bidirectional, num_buckets=num_buckets, max_distance=max_distance),
                       ref[[0, -1]])


def test_bucket_table_rejects_degenerate_sizes():
    lib = _lib.load()
    out = (C.c_int32 * 1025)()
    assert lib.vqa_t5_bucket_lut(0, 2, 128, out) == INVALID
    assert lib.vqa_t5_bucket_lut(0, 32, 16, out) == INVALID         # max_distance inside the exact range: log of a ratio <= 1
    assert lib.vqa_t5_bucket_lut(0, 32, 128, None) == INVALID
    assert lib.vqa_t5_bucket_lut(0, 32, 128, out) == OK


# The argument checks below hand the library fake device addresses. They run only where no device exists, so a check that failed to
# refuse could never reach a kernel; there a call that passes every check stops at the launch with VQA_ERR_CUDA.
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="argument checks run with fake device addresses, only where no device exists")
P = C.c_void_p(1 << 20)             # a 16-byte aligned fake device address


def at(offset):
    return C.c_void_p((1 << 20) + offset)


@no_device
def test_decode_attention_argument_checks():
    lib = _lib.load()
    used = C.c_int32(-1)

    def call(q=P, ldq=36 * 128, kc=P, vc=P, cap=64, B=2, hq=28, hkv=4, splits=0, ws=P, ws_bytes=1 << 30, out=P, ldo=28 * 128, sl=P, gl=P):
        return lib.vqa_op_decode_attention_d128(q, ldq, kc, vc, cap, sl, gl, B, hq, hkv, 0.088, splits, ws, ws_bytes, C.byref(used), out, ldo,
                                                None)

    assert call() == CUDA_ERR and used.value == min((2 * 132 + 7) // 8, (64 + 15) // 16)     # valid: reaches the launch; the rule's splits
    for hq, hkv in [(3, 1), (6, 1), (12, 2), (36, 4), (9, 1)]:                                   # G = 3, 6, 6, 9, 9
        assert call(hq=hq, hkv=hkv, ldq=(hq + 2 * hkv) * 128, ldo=hq * 128) == UNSUPPORTED, (hq, hkv)
    assert call(hq=28, hkv=3) == INVALID                                                       # q_heads not a multiple of kv_heads
    assert call(splits=65) == INVALID and call(splits=64) == CUDA_ERR                           # more splits than slots
    assert call(splits=-1) == INVALID
    need = 2 * 28 * 16 * 130 * 4
    assert call(splits=16, ws_bytes=need - 4) == WORKSPACE and call(splits=16, ws_bytes=need) == CUDA_ERR
    assert call(ws=None) == WORKSPACE
    assert call(ldq=36 * 128 + 2) == INVALID and call(ldo=28 * 128 + 2) == INVALID
    assert call(ldq=27 * 128) == INVALID and call(ldo=27 * 128) == INVALID                     # strides that do not cover the q heads
    assert call(q=at(4)) == INVALID and call(kc=at(2)) == INVALID and call(vc=at(4)) == INVALID and call(out=at(1)) == INVALID
    for k in ("q", "kc", "vc", "out", "sl", "gl"):
        assert call(**{k: None}) == INVALID, k
    assert call(B=0) == INVALID and call(cap=0) == INVALID


@no_device
def test_kv_cache_write_argument_checks():
    lib = _lib.load()

    def call(qkv=P, ld=36 * 128, k0=28 * 128, v0=32 * 128, hkv=4, B=3, S=10, sl=P, gl=None, kc=P, vc=P, cap=16):
        return lib.vqa_op_kv_cache_write(qkv, ld, k0, v0, hkv, B, S, sl, gl, kc, vc, cap, None)

    assert call() == CUDA_ERR and call(S=1, gl=P) == CUDA_ERR
    assert call(S=2, gl=P) == INVALID                     # decode mode takes one row per sequence
    assert call(S=17) == INVALID                          # padded rows beyond the cache
    assert call(ld=36 * 128 - 8) == INVALID               # V heads past the row
    assert call(ld=36 * 128 + 4) == INVALID and call(k0=28 * 128 + 4) == INVALID and call(v0=32 * 128 - 4) == INVALID
    assert call(qkv=at(8)) == INVALID and call(kc=at(8)) == INVALID and call(vc=at(2)) == INVALID
    for k in ("qkv", "sl", "kc", "vc"):
        assert call(**{k: None}) == INVALID, k


@no_device
def test_greedy_select_argument_checks():
    lib = _lib.load()

    def call(logits=P, B=2, V=1001, pen=None, penalty=1.0, eos=P, n_eos=1, max_new=8, first=None, pos3=None, **state):
        s = dict(tokens=P, lengths=P, done=P, n_done=P, all_done=P, next_ids=P)
        s.update(state)
        return lib.vqa_op_greedy_select(logits, B, V, pen, penalty, eos, n_eos, max_new, first, s["tokens"], s["lengths"], s["done"],
                                        s["n_done"], s["all_done"], s["next_ids"], pos3, None)

    assert call() == CUDA_ERR and call(first=P, pos3=P) == CUDA_ERR and call(eos=None, n_eos=0) == CUDA_ERR
    assert call(first=P) == INVALID and call(pos3=P) == INVALID
    assert call(eos=None) == INVALID and call(n_eos=-1) == INVALID
    assert call(penalty=0.0) == INVALID and call(penalty=float("nan")) == INVALID
    assert call(B=0) == INVALID and call(V=0) == INVALID and call(max_new=0) == INVALID
    for k in ("tokens", "lengths", "done", "n_done", "all_done", "next_ids"):
        assert call(**{k: None}) == INVALID, k
    assert call(logits=None) == INVALID


@no_device
def test_t5_self_attention_argument_checks():
    lib = _lib.load()

    def scoring(qkv=P, out=P, rel=P, lut=P, md=128, B=2, T=17, H=32):
        return lib.vqa_op_t5_decoder_self_attn(qkv, out, rel, lut, md, B, T, H, 1, None)

    def cached(qkv=P, kc=P, vc=P, cap=2048, lengths=P, out=P, rel=P, lut=P, md=128, B=2, H=32):
        return lib.vqa_op_t5_decode_self_attn(qkv, kc, vc, cap, lengths, out, rel, lut, md, B, H, 1, None)

    assert scoring() == CUDA_ERR and scoring(T=256) == CUDA_ERR
    assert scoring(T=257) == INVALID and scoring(T=0) == INVALID and scoring(md=0) == INVALID and scoring(H=0) == INVALID
    assert scoring(qkv=at(2)) == INVALID and scoring(out=at(2)) == INVALID
    for k in ("qkv", "out", "rel", "lut"):
        assert scoring(**{k: None}) == INVALID, k
    assert cached() == CUDA_ERR
    assert cached(cap=2049) == INVALID and cached(cap=0) == INVALID and cached(B=0) == INVALID
    assert cached(qkv=at(4)) == INVALID and cached(kc=at(8)) == INVALID and cached(vc=at(8)) == INVALID
    for k in ("qkv", "kc", "vc", "lengths", "out", "rel", "lut"):
        assert cached(**{k: None}) == INVALID, k


@no_device
@pytest.mark.parametrize("epilogue", [3, 6])
def test_gated_gemm_rejects_a_half_width_off_the_store_grid(epilogue):
    """A gated epilogue stores its N / 2 columns 8 at a time: N / 2 % 8 != 0 would write past every output row, and an up block that
    ends below w_rows would read rows that are not there. Both entry points refuse these shapes."""
    lib = _lib.load()

    def plain(N, w_rows, off):
        return lib.vqa_op_gemm_bf16(P, 512, P, 512, w_rows, P, 4096, 7, N, 512, None, None, 0, epilogue, off, 0, None)

    def normfuse(N, w_rows, off):
        return lib.vqa_op_gemm_bf16_normfuse(P, 512, P, 512, w_rows, P, 4096, 7, N, 512, None, 0, epilogue, off, P, None, 4, 512, 1e-6, None,
                                             None)

    for fn in (plain, normfuse):
        assert fn(2 * 3456, 2 * 3456, 3456) == CUDA_ERR                 # the padded vision MLP: accepted, stops at the launch
        assert fn(2 * 3420, 2 * 3420, 3420) == INVALID                  # the unpadded one: 3420 % 8 == 4
        assert fn(2 * 3456, 2 * 3456 - 8, 3456) == INVALID              # up block past w_rows
        assert fn(2 * 3456, 4 * 3456, 3456 * 3) == CUDA_ERR and fn(2 * 3456, 4 * 3456, 3456 * 3 + 8) == INVALID
        assert fn(2 * 3456, 2 * 3456, -8) == INVALID

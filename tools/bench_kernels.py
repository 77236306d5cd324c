#!/usr/bin/env python
"""Kernel-level measurements through the C ABI (run on the GPU box).

  python tools/bench_kernels.py attn [--dump DIR]   # head_dim-64 attention: T5 encoder shape and CLIP shape, both rounding modes,
                                                    # CUDA-event timing; --dump writes the outputs (raw bf16) to DIR
  python tools/bench_kernels.py gemm-time [--dump DIR]   # the T5-encoder and CLIP-tower GEMM shapes under a list of tile schedules,
                                                # CUDA-event timing; --dump writes each shape's output (raw bytes) to DIR
  python tools/bench_kernels.py gemm-ncu        # same launches once each, in a fixed order, for `ncu --metrics dram__bytes_*`
  python tools/bench_kernels.py gemm-list       # prints that order (shape, group_rows, chunk_rows) as JSON
  python tools/bench_kernels.py attn128 [--model qwen2.5-vl-3b]   # head_dim-128 attention at that model's heads (default the 7B)
  SHAPES=qwen3b_qkv,qwen3b_o,qwen3b_gate_up,qwen3b_down python tools/bench_kernels.py gemm-time   # the 3B's prefill GEMMs
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def time_ms(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def attn(dump_dir=None):
    """Both rounding modes at each shape. useful: 4 * 64 * H * sum(len_b^2) FLOP; tiles128: the same with every sequence padded to whole
    128-row tiles (what a kernel that runs every query and key tile in full executes). dump_dir: the outputs as raw bf16 bytes, so that
    two builds can be compared byte for byte."""
    import numpy as np
    from t2v_metrics_b200.engine import ops
    out = {}
    for name, (B, S, H, bias, scale) in dict(t5_enc=(64, 672, 64, True, 1.0), t5_enc_ragged=(64, 672, 64, True, 1.0),
                                             clip=(64, 577, 16, False, 0.125)).items():
        torch.manual_seed(0)
        qkv = (torch.randn(B * S, 3 * H * 64, device="cuda") * (0.5 if bias else 1.0)).bfloat16()
        table = None
        if bias:
            rel = torch.arange(-(S - 1), S, device="cuda").clamp(-128, 128) + 128
            table = (torch.randn(H, 257, device="cuda")).bfloat16().float()[:, rel].contiguous()
        lens = torch.randint(639, 673, (B,), device="cuda", dtype=torch.int32) if "ragged" in name else None
        L = lens.double().cpu() if lens is not None else torch.full((B,), float(S), dtype=torch.float64)
        useful = 4.0 * 64 * H * float((L * L).sum())
        tiles = 4.0 * 64 * H * float(((torch.ceil(L / 128) * 128) ** 2).sum())
        for rnd in (False, True):
            fn = lambda: ops.attention(qkv, B, S, H, seq_lens=lens, bias_table=table, scale=scale, bias_const_from=128 if bias else 0,
                                       round_scores=rnd)
            ms = time_ms(fn)
            o = fn()
            torch.cuda.synchronize()
            key = f"{name}_round{int(rnd)}"
            out[key] = dict(ms=round(ms, 4), tflops_useful=round(useful / ms / 1e9, 1), tflops_tiles128=round(tiles / ms / 1e9, 1),
                            checksum=float(o.float().abs().sum()))
            if dump_dir:
                os.makedirs(dump_dir, exist_ok=True)
                np.save(os.path.join(dump_dir, key + ".npy"), o.view(torch.int16).cpu().numpy())
    print(json.dumps(dict(kernel="attn64_ws_kernel", **out)))


def _t5_attn_inputs(B=64, S=672, H=64):
    torch.manual_seed(0)
    qkv = (torch.randn(B * S, 3 * H * 64, device="cuda") * 0.5).bfloat16()
    rel = torch.arange(-(S - 1), S, device="cuda").clamp(-128, 128) + 128
    table = (torch.randn(H, 257, device="cuda")).bfloat16().float()[:, rel].contiguous()
    return qkv, table


def attn_one():
    """one launch of the production attention kernel at the T5-encoder shape (target of `ncu --set full`)."""
    from t2v_metrics_b200.engine import ops
    qkv, table = _t5_attn_inputs()
    for _ in range(3):
        ops.attention(qkv, 64, 672, 64, bias_table=table, scale=1.0, bias_const_from=128, round_scores=True)
    torch.cuda.synchronize()


def attn128(model="qwen2.5-vl-7b"):
    """head_dim-128 attention at a Qwen2.5-VL size's shapes: causal GQA prefill (B=32, S=320; 7B 28/4 heads, 3B 16/2), vision windows (64
    tokens) and whole frames."""
    import ctypes as C
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _ptr, _stream_ptr, _check
    lib = _lib.load()
    torch.manual_seed(0)
    res = {}

    def run(qkv, out_cols, n_seq, max_len, S, Hq, group, cu, scale, causal, q0, k0, v0):
        out = torch.empty(qkv.shape[0], out_cols, dtype=torch.bfloat16, device="cuda")
        fn = lambda: _check(lib.vqa_op_attention_d128(_ptr(qkv), qkv.shape[1], qkv.shape[0], q0, k0, v0, _ptr(out), out_cols, n_seq, max_len, S, Hq,
                                                       group, _ptr(cu), None, float(scale), 1 if causal else 0, _stream_ptr(qkv.device)), None, "d128")
        return time_ms(fn), float(out.float().abs().sum())
    from t2v_metrics_b200.config import QWEN25VL_MODELS
    cfg = QWEN25VL_MODELS[model]["config"]()
    B, S, Hq, Hkv = 32, 320, cfg.heads, cfg.kv_heads
    qkv = (torch.randn(B * S, (Hq + 2 * Hkv) * 128, device="cuda") * 0.5).bfloat16()
    ms, cs = run(qkv, Hq * 128, B, S, S, Hq, Hq // Hkv, None, 128 ** -0.5, True, 0, Hq * 128, (Hq + Hkv) * 128)
    res["llm_causal"] = dict(ms=round(ms, 4), tflops=round(2.0 * B * Hq * S * S * 128 / ms / 1e9, 1), checksum=cs)
    L, Hv = 32 * 1024, 16
    x = torch.zeros(L, 3, Hv, 128, device="cuda")
    x[..., :80] = torch.randn(L, 3, Hv, 80, device="cuda") * 0.5
    vq = x.reshape(L, 3 * Hv * 128).bfloat16()
    for name, wlen in (("vis_window64", 64), ("vis_frame1024", 1024)):
        cu = torch.arange(0, L + 1, wlen, dtype=torch.int32, device="cuda")
        ms, cs = run(vq, Hv * 128, L // wlen, wlen, 0, Hv, 1, cu, 80 ** -0.5, False, 0, Hv * 128, 2 * Hv * 128)
        res[name] = dict(ms=round(ms, 4), tflops_padded=round(4.0 * L * wlen * Hv * 128 / ms / 1e9, 1), checksum=cs)
    print(json.dumps(dict(kernel="attn_wgmma_kernel d128", model=model, q_heads=Hq, kv_heads=Hkv, **res)))


SHAPES = dict(   # name: (M, N, K, epilogue, residual, bias)   residual: None, "bf16" (in the output's place) or "f32" (fp32 stream, in place)
    # clip-flant5-xxl encoder layer at B=64, S=672
    qkv=(43008, 12288, 4096, "store", None, False),
    o=(43008, 4096, 4096, "store", "bf16", False),
    wi=(43008, 20480, 4096, "gated_gelu", None, False),
    wo=(43008, 4096, 10240, "store", "bf16", False),
    # o with twice the K: 2 t(o) - t(o_k8192) is the fixed cost per tile (epilogue, pipeline ramp) that the main loop does not amortise
    o_k8192=(43008, 4096, 8192, "store", "bf16", False),
    # CLIP ViT-L/14-336 layer at 64 images x 577 tokens
    clip_qkv=(36928, 3072, 1024, "store", None, True),
    clip_out=(36928, 1024, 1024, "store", "f32", True),
    clip_fc1=(36928, 4096, 1024, "quick_gelu", None, True),
    clip_fc2=(36928, 1024, 4096, "store", "f32", True),
    # Qwen2.5-VL-3B decoder layer at B=32 prompts of 320 tokens (448x448 image + 64 text ids)
    qwen3b_qkv=(10240, 2560, 2048, "store", None, True),
    qwen3b_o=(10240, 2048, 2048, "store", "bf16", False),
    qwen3b_gate_up=(10240, 22016, 2048, "gated_silu", None, False),
    qwen3b_down=(10240, 2048, 11008, "store", "bf16", False),
)
SCHEDULES = [(0, 0), (4096, -1), (1024, -1), (512, 2048), (512, 4096), (1024, 3072), (1024, 4096), (1024, 6144), (2048, 4096), (1024, 8192),
             (2048, 2048), (512, 6144)]


def gemm(mode, dump_dir=None):
    """dump_dir: each shape's output after its last schedule, as raw bytes (bf16 or fp32), so that two builds can be compared byte for byte.
    The in-place residual shapes restore their residual before every launch, so the dumped output is one GEMM's result."""
    import numpy as np
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import ops
    lib = _lib.load()
    torch.manual_seed(0)
    rows = []
    only = os.environ.get("SHAPES", "").split(",") if os.environ.get("SHAPES") else list(SHAPES)
    scheds = [tuple(int(x) for x in s.split(":")) for s in os.environ["SCHEDS"].split(",")] if os.environ.get("SCHEDS") else SCHEDULES
    ballast = None
    if os.environ.get("BALLAST_GB"):      # mimic the footprint of the real step (weights + workspace) around the operands
        ballast = torch.empty(int(os.environ["BALLAST_GB"]) << 30, dtype=torch.uint8, device="cuda").fill_(1)
    for name in only:
        M, N, K, epi, res, has_bias = SHAPES[name]
        a = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
        w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
        if os.environ.get("ZERO_OPERANDS"):
            a.zero_(); w.zero_()
        bias = (torch.randn(N, device="cuda") * 0.1).bfloat16() if has_bias else None
        n_out = N // 2 if epi.startswith("gated") else N
        if res == "f32":
            c = torch.randn(M, n_out, device="cuda")
            fn = lambda: ops.gemm_f32acc(a, w, c, bias=bias)
        else:
            c = torch.empty(M, n_out, dtype=torch.bfloat16, device="cuda")
            r = torch.randn(M, n_out, device="cuda").bfloat16() if res == "bf16" else None
            fn = lambda: ops.gemm(a, w, bias=bias, residual=r, epilogue=epi, out=c, gate_up_offset=N // 2 if epi.startswith("gated") else 0)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for (g, ch) in scheds:
            lib.vqa_set_gemm_schedule(g, ch)
            if mode == "ncu":
                flush.zero_()      # start every measured launch from a cold L2
                fn()
                torch.cuda.synchronize()
            else:
                ms = time_ms(fn, iters=10, warm=2)
                rows.append(dict(shape=name, group_rows=g, chunk_rows=ch, ms=round(ms, 4), tflops=round(2.0 * M * N * K / ms / 1e9, 1)))
        if dump_dir:
            if res == "f32":   # one accumulation into a fresh copy of the seeded stream
                torch.manual_seed(1)
                c.copy_(torch.randn(M, n_out, device="cuda"))
            fn()
            torch.cuda.synchronize()
            os.makedirs(dump_dir, exist_ok=True)
            np.save(os.path.join(dump_dir, f"gemm_{name}.npy"), c.view(torch.int32 if c.dtype == torch.float32 else torch.int16).cpu().numpy())
        lib.vqa_set_gemm_schedule(0, 0)
        del a, w, c
    if mode != "ncu":
        print(json.dumps(rows))


if __name__ == "__main__":
    cmd = sys.argv[1]
    if cmd == "attn":
        attn(sys.argv[sys.argv.index("--dump") + 1] if "--dump" in sys.argv else None)
    elif cmd == "attn-one":
        attn_one()
    elif cmd == "attn128":
        attn128(sys.argv[sys.argv.index("--model") + 1] if "--model" in sys.argv else "qwen2.5-vl-7b")
    elif cmd == "gemm-time":
        gemm("time", sys.argv[sys.argv.index("--dump") + 1] if "--dump" in sys.argv else None)
    elif cmd == "gemm-ncu":
        gemm("ncu")
    elif cmd == "gemm-list":
        only = os.environ.get("SHAPES", "").split(",") if os.environ.get("SHAPES") else list(SHAPES)
        print(json.dumps([dict(shape=n, group_rows=g, chunk_rows=c) for n in only for (g, c) in SCHEDULES]))

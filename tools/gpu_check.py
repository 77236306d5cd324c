"""Bring-up checks on a GPU (one sub-test per process so a hung kernel cannot take the others down).

usage: python tools/gpu_check.py <test> [args...]   -> appends one JSON line to $VQA_CHECK_DIR/check.jsonl (default check_out/)
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

OUT = os.environ.get("VQA_CHECK_DIR") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "check_out")
os.makedirs(OUT, exist_ok=True)


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    with open(os.path.join(OUT, "check.jsonl"), "a") as f:
        f.write(line + "\n")


def ref_gemm(a, w, bias=None, residual=None, epilogue="store", gate_off=0):
    acc = a.float() @ w.float().t()
    if epilogue == "gated_gelu":
        g = acc[:, :gate_off].bfloat16().float()
        u = acc[:, gate_off:].bfloat16().float()
        h = torch.nn.functional.gelu(g, approximate="tanh").bfloat16().float()
        return (h * u).bfloat16()
    if bias is not None:
        acc = acc + bias.float()
    y = acc.bfloat16().float()
    if epilogue == "quick_gelu":
        y = y * torch.sigmoid(1.702 * y)
    elif epilogue == "gelu":
        y = torch.nn.functional.gelu(y)
    elif epilogue == "relu":
        y = torch.relu(y)
    if residual is not None:
        y = y + residual.float()
    return y.bfloat16()


def err(x, y):
    d = (x.float() - y.float()).abs()
    return float(d.max()), float(d.mean()), float(y.float().abs().mean())


def t_gemm(variant, M, N, K, epilogue="store", use_bias=0, use_res=0):
    from t2v_metrics_b200.engine import ops
    variant, M, N, K, use_bias, use_res = int(variant), int(M), int(N), int(K), int(use_bias), int(use_res)
    torch.manual_seed(0)
    dev = "cuda:0"
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=dev) * (K ** -0.5)).bfloat16()
    bias = (torch.randn(N, device=dev) * 0.1).bfloat16() if use_bias else None
    n_out = N // 2 if epilogue == "gated_gelu" else N
    res = torch.randn(M, n_out, device=dev).bfloat16() if use_res else None
    t0 = time.time()
    c = ops.gemm(a, w, bias=bias, residual=res, epilogue=epilogue, variant=variant, gate_up_offset=N // 2)
    torch.cuda.synchronize()
    ref = ref_gemm(a, w, bias, res, epilogue, N // 2)
    mx, mean, scale = err(c, ref)
    # count badly wrong elements
    bad = int(((c.float() - ref.float()).abs() > 0.05 + 0.02 * ref.float().abs()).sum())
    emit(test="gemm", variant=variant, M=M, N=N, K=K, epilogue=epilogue, bias=use_bias, res=use_res, max_err=mx,
         mean_err=mean, ref_scale=scale, bad=bad, total=c.numel(), ok=bool(bad == 0), secs=round(time.time() - t0, 3))


def t_gemm_perf(variant, M, N, K, epilogue="store"):
    from t2v_metrics_b200.engine import ops
    variant, M, N, K = int(variant), int(M), int(N), int(K)
    dev = "cuda:0"
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=dev) * (K ** -0.5)).bfloat16()
    n_out = N // 2 if epilogue == "gated_gelu" else N
    out = torch.empty(M, n_out, dtype=torch.bfloat16, device=dev)
    for _ in range(3):
        ops.gemm(a, w, epilogue=epilogue, variant=variant, out=out, gate_up_offset=N // 2)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = 10
    ev0.record()
    for _ in range(iters):
        ops.gemm(a, w, epilogue=epilogue, variant=variant, out=out, gate_up_offset=N // 2)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / iters
    tf = 2.0 * M * N * K / ms / 1e9
    # cuBLAS (torch.matmul) on the same shape for context
    for _ in range(3):
        torch.matmul(a, w.t())
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(iters):
        torch.matmul(a, w.t())
    ev1.record()
    torch.cuda.synchronize()
    ms_ref = ev0.elapsed_time(ev1) / iters
    emit(test="gemm_perf", variant=variant, M=M, N=N, K=K, epilogue=epilogue, ms=ms, tflops=tf,
         cublas_ms=ms_ref, cublas_tflops=2.0 * M * N * K / ms_ref / 1e9)


def t_gemm_once(variant, M, N, K, epilogue="store", reps=3):
    """A few launches of one GEMM shape (run under ncu --metrics dram__bytes... to read its DRAM traffic)."""
    from t2v_metrics_b200.engine import ops
    variant, M, N, K, reps = int(variant), int(M), int(N), int(K), int(reps)
    dev = "cuda:0"
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=dev) * (K ** -0.5)).bfloat16()
    n_out = N // 2 if epilogue == "gated_gelu" else N
    out = torch.empty(M, n_out, dtype=torch.bfloat16, device=dev)
    for _ in range(reps):
        ops.gemm(a, w, epilogue=epilogue, variant=variant, out=out, gate_up_offset=N // 2)
    torch.cuda.synchronize()
    emit(test="gemm_once", M=M, N=N, K=K, epilogue=epilogue, group_rows=os.environ.get("VQA_GEMM_GROUP_ROWS", "default"))


def t_norm():
    from t2v_metrics_b200.engine import ops
    dev = "cuda:0"
    torch.manual_seed(0)
    for D in (4096, 2048, 256):
        x = torch.randn(777, D, device=dev).bfloat16()
        g = (1 + 0.1 * torch.randn(D, device=dev)).bfloat16()
        y = ops.norm(x, g, 1e-6)
        var = x.float().pow(2).mean(-1, keepdim=True)
        ref = (g.float() * (x.float() * torch.rsqrt(var + 1e-6)).bfloat16().float()).bfloat16()
        mx, mean, sc = err(y, ref)
        emit(test="rmsnorm", D=D, max_err=mx, mean_err=mean, ok=bool(mx < 0.05))


def t_norm_perf(rows=43008, D=4096):
    from t2v_metrics_b200.engine import ops
    rows, D = int(rows), int(D)
    x = torch.randn(rows, D, device="cuda:0").bfloat16()
    g = torch.ones(D, device="cuda:0").bfloat16()
    for _ in range(3):
        ops.norm(x, g, 1e-6)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(20):
        ops.norm(x, g, 1e-6)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / 20
    emit(test="norm_perf", rows=rows, D=D, ms=ms, gbps=4.0 * rows * D / ms / 1e6)


def t_attention():
    from t2v_metrics_b200.engine import ops
    dev = "cuda:0"
    torch.manual_seed(0)
    for (B, S, H, use_bias, ragged, scale) in [(2, 100, 4, 1, 1, 1.0), (3, 577, 16, 0, 0, 0.125), (2, 672, 8, 1, 1, 1.0)]:
        qkv = (torch.randn(B * S, 3 * H * 64, device=dev) * 0.5).bfloat16()
        lens = torch.full((B,), S, dtype=torch.int32, device=dev)
        if ragged:
            lens = torch.randint(S // 2, S + 1, (B,), device=dev, dtype=torch.int32)
        table = (torch.randn(H, 2 * S - 1, device=dev) * 0.5).bfloat16().float().contiguous() if use_bias else None
        out = ops.attention(qkv, B, S, H, seq_lens=lens if ragged else None, bias_table=table, scale=scale,
                            round_scores=False)
        torch.cuda.synchronize()
        q, k, v = qkv.float().view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
        sc = torch.matmul(q, k.transpose(-1, -2)) * scale
        if use_bias:
            idx = (torch.arange(S, device=dev)[None, :] - torch.arange(S, device=dev)[:, None]) + S - 1
            sc = sc + table[:, idx][None]
        kmask = torch.arange(S, device=dev)[None, :] < lens[:, None]
        sc = sc.masked_fill(~kmask[:, None, None, :], float("-inf"))
        p = torch.softmax(sc, dim=-1)
        ref = torch.matmul(p, v).permute(0, 2, 1, 3).reshape(B * S, H * 64)
        qmask = kmask.reshape(B * S)
        mx, mean, scl = err(out[qmask], ref[qmask])
        emit(test="attention", B=B, S=S, H=H, bias=use_bias, ragged=ragged, max_err=mx, mean_err=mean, ref_scale=scl,
             ok=bool(mx < 0.03))


def t_attention_perf(B=64, S=672, H=64, use_bias=1):
    from t2v_metrics_b200.engine import ops
    B, S, H, use_bias = int(B), int(S), int(H), int(use_bias)
    dev = "cuda:0"
    qkv = (torch.randn(B * S, 3 * H * 64, device=dev) * 0.5).bfloat16()
    dist = int(os.environ.get("VQA_BIAS_DIST", "128"))
    rel = torch.arange(-(S - 1), S, device=dev).clamp(-dist, dist) + dist
    table = (torch.randn(H, 2 * dist + 1, device=dev) * 0.5)[:, rel].contiguous() if use_bias else None
    scale = 1.0 if use_bias else 0.125
    for _ in range(3):
        ops.attention(qkv, B, S, H, bias_table=table, scale=scale)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(10):
        ops.attention(qkv, B, S, H, bias_table=table, scale=scale)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / 10
    emit(test="attention_perf", B=B, S=S, H=H, bias=use_bias, ms=ms, tflops=4.0 * B * H * S * S * 64 / ms / 1e9,
         mma_sync=os.environ.get("VQA_ATTN_MMA_SYNC", "0"))


def t_preprocess_perf(n=64, size=512, out=336):
    """Device pre-processing kernel alone: device-resident uint8 sources, HBM roofline = (source bytes + output bytes) / time;
    plus the CPU (PIL) path on the host for the same images."""
    import time
    from PIL import Image
    from oracle import clipt5_oracle as orc
    from t2v_metrics_b200.engine import clip_preprocess_u8
    n, size, out = int(n), int(size), int(out)
    dev = "cuda:0"
    raw = torch.randint(0, 256, (n, size, size, 3), dtype=torch.uint8)
    d_raw = raw.to(dev)
    dst = torch.empty(n, 3, out, out, dtype=torch.float32, device=dev)
    for _ in range(3):
        clip_preprocess_u8(d_raw, out, dev, out=dst)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(20):
        clip_preprocess_u8(d_raw, out, dev, out=dst)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / 20
    t0 = time.perf_counter()
    m = min(n, 8)
    ref = torch.stack([orc.clip_preprocess(Image.fromarray(raw[i].numpy()), out) for i in range(m)])
    cpu_ms_per_image = (time.perf_counter() - t0) * 1000 / m
    exact = bool(torch.equal(dst[:m].cpu(), ref))
    by = raw.numel() + dst.numel() * 4
    emit(test="preprocess_perf", n=n, size=size, out=out, ms=ms, us_per_image=1000 * ms / n, gbps=by / ms / 1e6, bytes=by,
         cpu_pil_ms_per_image=cpu_ms_per_image, bit_exact=exact)


def t_lmhead():
    from t2v_metrics_b200.engine import ops
    dev = "cuda:0"
    torch.manual_seed(0)
    for (M, N, K) in [(128, 32128, 512), (6, 1000, 256)]:
        h = torch.randn(M, K, device=dev).bfloat16()
        w = (torch.randn(N, K, device=dev) * K ** -0.5 * 3).bfloat16()
        labels = torch.randint(0, N, (M,), device=dev, dtype=torch.int32)
        lp = ops.lmhead_logprob(h, w, labels)
        torch.cuda.synchronize()
        logits = (h.float() @ w.float().t()).bfloat16().float()
        ref = torch.log_softmax(logits, -1).gather(-1, labels.long()[:, None])[:, 0]
        mx, mean, scl = err(lp, ref)
        emit(test="lmhead", M=M, N=N, K=K, max_err=mx, mean_err=mean, ok=bool(mx < 0.02))


def t_pipeline(kind="tiny", batch=3):
    """Full CLIP-FlanT5 forward vs the oracle (fp32 and bf16-emulating) on a small config."""
    from oracle import clipt5_oracle as orc
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.engine import ClipT5Engine
    import dataclasses
    batch = int(batch)
    if kind == "tiny":
        ocfg = orc.ClipT5Config.tiny()
        L = 12
    elif kind == "mid":
        ocfg = orc.ClipT5Config.tiny(image_size=112, vit_hidden=1024, vit_heads=16, vit_mlp=1024, vit_layers=3, d_model=512,
                                     n_heads=8, d_ff=1024, enc_layers=2, dec_layers=2, vocab=2048)
        L = 24
    else:
        raise SystemExit("unknown kind")
    cfg = ClipT5Config(**dataclasses.asdict(ocfg))
    labels_ids = (37 % ocfg.vocab, 1)
    sd = orc.make_synthetic_state_dict(ocfg, seed=0, label_ids=labels_ids)
    inp = orc.make_synthetic_inputs(ocfg, batch, L, seed=1, ragged=True, label_ids=labels_ids)
    orc.calibrate_lm_head(sd, ocfg, inp)
    t0 = time.time()
    ref32 = orc.clipt5_score(sd, ocfg, inp["pixels"], inp["input_ids"], inp["text_lens"], inp["labels"], mode="fp32",
                             return_all=True)
    ref16 = orc.clipt5_score(sd, ocfg, inp["pixels"], inp["input_ids"], inp["text_lens"], inp["labels"], mode="bf16",
                             return_all=True)
    t_or = time.time() - t0
    dev = "cuda:0"
    eng = ClipT5Engine(cfg, dev, cross_attention_mode=os.environ.get("VQA_CROSS", "absorbed"))
    eng.load_state_dict(sd)
    scores, logp = eng.score_tensors(inp["pixels"].to(dev), inp["input_ids"].to(dev, torch.int32),
                                     inp["text_lens"].to(dev, torch.int32), inp["labels"].to(dev, torch.int32),
                                     return_logprobs=True)
    torch.cuda.synchronize()
    s = scores.cpu()
    emit(test="pipeline", kind=kind, gemm_simt=os.environ.get("VQA_GEMM_SIMT", "0"), cross=os.environ.get("VQA_CROSS", "absorbed"),
         attn_mma_sync=os.environ.get("VQA_ATTN_MMA_SYNC", "0"),
         variant=os.environ.get("VQA_GEMM_VARIANT", "auto"),
         scores=[round(float(x), 5) for x in s], ref_fp32=[round(float(x), 5) for x in ref32["scores"]],
         ref_bf16=[round(float(x), 5) for x in ref16["scores"]],
         logp=[[round(float(v), 4) for v in r] for r in logp.cpu()],
         ref_logp32=[[round(float(v), 4) for v in r] for r in ref32["logprobs"]],
         ref_logp16=[[round(float(v), 4) for v in r] for r in ref16["logprobs"]],
         max_err_vs_fp32=float((s - ref32["scores"]).abs().max()), max_err_vs_bf16=float((s - ref16["scores"]).abs().max()),
         bf16_vs_fp32=float((ref16["scores"] - ref32["scores"]).abs().max()), launches=eng.last_launch_count(),
         oracle_secs=round(t_or, 2))


def t_pytest(*args):
    """Run a pytest selection inside this (timeout-guarded) process."""
    import pytest as _pt
    rc = _pt.main(["-q", "-s", "-x", "-m", "gpu", *args])
    emit(test="pytest", args=list(args), ok=bool(rc == 0), rc=int(rc))


if __name__ == "__main__":
    name = sys.argv[1]
    fn = globals()["t_" + name]
    try:
        fn(*sys.argv[2:])
    except Exception as e:  # noqa
        import traceback
        emit(test=name, args=sys.argv[2:], ok=False, error=repr(e), tb=traceback.format_exc()[-1500:])
        sys.exit(1)

"""Single-prefill VQAScore throughput on one H100 for a Qwen2.5-VL size (--model): synthetic weights drawn on the device (tied for the 3B),
B prompts of a 448x448 image (256 vision tokens) + 64 text ids (S = 320), one engine call (QwenVLEngine.score_tensors) per step, timed
with CUDA events after warm-up. One JSON line: pairs/s, ms per step, launches, the per-category device time of one profiled step
(attention, GEMM, ...) and the GPU name, power limit and SM clock read in the same run.

  python tools/bench_score_qwen.py [--model qwen2.5-vl-3b] [--batch 32] [--steps 20] [--out results.jsonl]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch

from oracle import qwen25vl_oracle as qo
from bench_generate import gpu_identity
from bench_video_score import sm_clocks
from qwen_bench_model import add_model_arg, engine, model_config, synthetic_weights


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    add_model_arg(ap)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_score_qwen.py measures on a CUDA device; there is none")
    from t2v_metrics_b200 import qwen_host
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    cfg, ecfg = model_config(a.model)
    eng = engine(ecfg, synthetic_weights(cfg, ecfg, dev), dev)
    B = a.batch
    inp = qo.make_synthetic_inputs(cfg, B, (448, 448), 64, seed=1)
    grids = [tuple(map(int, g)) for g in inp["grid_thw"]]
    idx = qwen_host.build_batch_indices([x.tolist() for x in inp["input_ids"]], grids, list(range(B)), cfg.image_token_id,
                                        cfg.spatial_merge_size, cfg.tokens_per_second, video_token_id=cfg.video_token_id)
    d = {k: v.to(dev) for k, v in idx.items() if torch.is_tensor(v)}
    pix = inp["pixel_patches"].to(dev)
    ans = torch.tensor(inp["answer_ids"], dtype=torch.int32, device=dev)
    step = lambda: eng.score_tensors(pix, grids, d["input_ids"], d["seq_lens"], d["feat_index"], d["position_ids"], ans)
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        out = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    assert bool(torch.isfinite(out).all())
    launches = eng.last_launch_count()
    eng.set_profile(True)
    step()
    torch.cuda.synchronize()
    prof = eng.read_profile()
    eng.set_profile(False)
    line = dict(workload=f"{a.model} VQAScore, one prefill per step", gpu=gpu, power_limit=power, sm_clock=sm_clocks(), batch=B,
                image=448, text_tokens=64, seq_len=int(d["input_ids"].shape[1]), steps=a.steps, ms_per_step=round(ms, 3),
                pairs_per_s=round(B / (ms * 1e-3), 1), launches=launches,
                device_ms_by_category={k: round(v[0], 3) for k, v in prof.items()})
    print(json.dumps(line), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

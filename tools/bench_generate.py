"""Greedy generation on one H100: Qwen2.5-VL width (--model, default qwen2.5-vl-7b) with synthetic weights drawn on the device, 448x448
images and 64 text tokens per prompt, B in {1, 8, 32}, 128 new tokens with no EOS ids so every run decodes the same number of steps. One JSON line per batch size:
prefill ms, median / spread of the decode step (CUDA events around each graph replay), generated tokens/s, launches per step, algorithmic
bytes per step (every language-model weight read once + the K/V rows the step attends to) and the whole-step rate they give against the
3.35 TB/s HBM3 data-sheet figure, per-category device time of one profiled step, and the GPU name and power limit read in the same run.

The baseline is the reference's loop: HF Qwen2_5_VLForConditionalGeneration.generate(do_sample=False) in bf16 with sdpa, one sample at a
time, min_new_tokens = max_new_tokens, on the same GPU and weights (its rate does not depend on B: it is measured once, on --hf-samples).

The decode GEMMs split their K range (splitk_slices); run with VQA_GEMM_SPLITK=0 to time the step without the split.

  python tools/bench_generate.py [--model qwen2.5-vl-3b] [--batches 1,8,32] [--new 128] [--no-hf] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from oracle import qwen25vl_oracle as qo
from qwen_bench_model import add_model_arg, engine, hf_model, model_config, synthetic_weights

HBM_PEAK = 3.35e12


def gpu_identity():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                               timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def weight_bytes(cfg):
    D, qkv = cfg.hidden, (cfg.heads + 2 * cfg.kv_heads) * cfg.head_dim
    per_layer = qkv * D + qkv + D * cfg.heads * cfg.head_dim + 2 * cfg.mlp * D + D * cfg.mlp + 2 * D
    return 2.0 * (cfg.layers * per_layer + cfg.vocab * D + D)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--text", type=int, default=64)
    ap.add_argument("--image", type=int, default=448)
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--hf-samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    add_model_arg(ap)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_generate.py measures on a CUDA device; there is none")
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    cfg, ecfg = model_config(a.model)
    N = a.new
    sd = synthetic_weights(cfg, ecfg, dev)
    eng = engine(ecfg, sd, dev)
    W = weight_bytes(cfg)
    lines = []
    for B in [int(x) for x in a.batches.split(",")]:
        inp = qo.make_synthetic_inputs(cfg, B, (a.image, a.image), a.text, seed=1)
        prompts = [x.tolist() for x in inp["input_ids"]]
        pix = inp["pixel_patches"].to(dev)
        eng.generate_prompts(pix, inp["grid_thw"], prompts, N, ())          # warm-up: loads modules, captures the step graph
        st = eng.generate_begin(pix, inp["grid_thw"], prompts, N, ())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        pre = []
        for _ in range(3):
            e0.record()
            st["prefill"]()
            e1.record()
            torch.cuda.synchronize()
            pre.append(e0.elapsed_time(e1))
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(N - 1)]
        t0 = time.perf_counter()
        for s, e in evs:
            s.record()
            st["graph"].replay()
            e.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        steps = torch.tensor([s.elapsed_time(e) for s, e in evs])
        assert bool((st["lengths"].cpu() == N).all())
        st["prefill"]()
        eng.generate_step(st)
        launches = eng.last_launch_count()
        eng.set_profile(True)
        eng.generate_step(st)
        torch.cuda.synchronize()
        prof = eng.read_profile()
        eng.set_profile(False)
        S_avg = sum(len(p) for p in prompts) / B
        kv = 2.0 * cfg.layers * B * cfg.kv_heads * cfg.head_dim * 2 * (S_avg + N / 2)      # K and V rows a step attends to, mean over the steps
        med = float(steps.median())
        line = dict(workload=f"{a.model} greedy generate", gpu=gpu, power_limit=power, batch=B, image=a.image, text_tokens=a.text,
                    prompt_tokens=S_avg, new_tokens=N, splitk=os.environ.get("VQA_GEMM_SPLITK", "1") != "0",
                    prefill_ms=round(min(pre), 3), step_ms_median=round(med, 4), step_ms_p10=round(float(steps.quantile(0.1)), 4),
                    step_ms_p90=round(float(steps.quantile(0.9)), 4), decode_tokens_per_s=round(B * (N - 1) / wall, 1),
                    launches_per_step=launches, step_bytes=W + kv, step_weight_bytes=W, step_kv_bytes=kv,
                    whole_step_GBps=round((W + kv) / (med * 1e-3) / 1e9, 1), whole_step_share_of_hbm_peak=round((W + kv) / (med * 1e-3) / HBM_PEAK, 3),
                    step_device_ms_by_category={k: round(v[0], 4) for k, v in prof.items()},
                    step_scopes_by_category={k: v[2] for k, v in prof.items()})
        print(json.dumps(line), flush=True)
        lines.append(line)
        del st
    del eng
    torch.cuda.empty_cache()
    if not a.no_hf:
        model = hf_model(cfg, ecfg, sd, dev)
        inp = qo.make_synthetic_inputs(cfg, a.hf_samples, (a.image, a.image), a.text, seed=1)
        P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]

        def run(b, n):
            ids = inp["input_ids"][b].to(dev)
            with torch.no_grad():
                return model.generate(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long, device=dev),
                                      pixel_values=inp["pixel_patches"][b * P:(b + 1) * P].to(dev, torch.bfloat16),
                                      image_grid_thw=torch.tensor([list(inp["grid_thw"][b])], device=dev),
                                      mm_token_type_ids=(ids == cfg.image_token_id).long()[None], max_new_tokens=n, min_new_tokens=n,
                                      do_sample=False, eos_token_id=None, pad_token_id=0)
        run(0, 4)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in range(a.hf_samples):
            run(b, N)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        line = dict(workload="HF generate(do_sample=False) bf16 sdpa, one sample at a time", gpu=gpu, power_limit=power, samples=a.hf_samples,
                    image=a.image, text_tokens=a.text, new_tokens=N, seconds=round(dt, 3), tokens_per_s=round(a.hf_samples * N / dt, 1))
        print(json.dumps(line), flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

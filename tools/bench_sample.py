"""Sampled against greedy generation on one H100: Qwen2.5-VL 7B and 3B widths with synthetic weights drawn on the device, 448x448 images
and 64 text tokens per prompt, B in {1, 8, 32}, 128 new tokens with no EOS ids. Three step types share one generation workspace and are
timed alternately in one process, each round a fresh prefill then N - 1 graph replays under CUDA events:
  greedy                               generate(do_sample=False)
  sampled T 0.7 / top_k 50 / top_p 0.9  the reference's generate(temperature=0.7) with transformers' default top_k
  sampled T 0.7 / top_k 0 / top_p 0.9   a nucleus over the full vocabulary (top_k off)
One JSON line per (model, batch, step type): median and p10-p90 of the replayed steps over all rounds, launches per step, and the
device time of the selection kernel itself in one eager step under torch.profiler; every line carries the GPU name and power limit
read in the same run.

  python tools/bench_sample.py [--models qwen2.5-vl-7b,qwen2.5-vl-3b] [--batches 1,8,32] [--new 128] [--rounds 3] [--out results.jsonl]
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
from qwen_bench_model import engine, model_config, synthetic_weights

STEP_TYPES = {"greedy": None, "sample T0.7 k50 p0.9": (0.7, 50, 0.9), "sample T0.7 k0 p0.9": (0.7, 0, 0.9)}


def select_kernel_ms(eng, st, name: str) -> float:
    """Device time of the kernel named `name` in one eager decode step of st, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    st["prefill"]()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.generate_step(st)
        torch.cuda.synchronize()
    times = [e.device_time_total for e in prof.key_averages() if name in e.key]
    return round(sum(times) / 1e3, 4) if times else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="qwen2.5-vl-7b,qwen2.5-vl-3b")
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--text", type=int, default=64)
    ap.add_argument("--image", type=int, default=448)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample.py measures on a CUDA device; there is none")
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    N = a.new
    lines = []
    for model in a.models.split(","):
        cfg, ecfg = model_config(model)
        sd = synthetic_weights(cfg, ecfg, dev)
        eng = engine(ecfg, sd, dev)
        for B in [int(x) for x in a.batches.split(",")]:
            inp = qo.make_synthetic_inputs(cfg, B, (a.image, a.image), a.text, seed=1)
            prompts = [x.tolist() for x in inp["input_ids"]]
            pix = inp["pixel_patches"].to(dev)
            states = {}
            for kind, smp in STEP_TYPES.items():
                sample = None if smp is None else dict(seeds=list(range(B)), temperature=smp[0], top_k=smp[1], top_p=smp[2])
                st = eng.generate_begin(pix, inp["grid_thw"], prompts, N, (), sample=sample)
                eng._decode_loop(st, True, N)                    # warm-up: loads modules, captures the step graph
                states[kind] = st
            steps = {kind: [] for kind in STEP_TYPES}
            for _ in range(a.rounds):
                for kind, st in states.items():
                    st["prefill"]()
                    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(N - 1)]
                    for s, e in evs:
                        s.record()
                        st["graph"].replay()
                        e.record()
                    torch.cuda.synchronize()
                    assert bool((st["lengths"].cpu() == N).all())
                    steps[kind] += [s.elapsed_time(e) for s, e in evs]
            greedy_med = float(torch.tensor(steps["greedy"]).median())
            for kind, st in states.items():
                st["prefill"]()
                eng.generate_step(st)
                launches = eng.last_launch_count()
                t = torch.tensor(steps[kind])
                med = float(t.median())
                kernel = "greedy_select_kernel" if STEP_TYPES[kind] is None else "sample_select_kernel"
                line = dict(workload=f"{model} generate step", step_type=kind, gpu=gpu, power_limit=power, batch=B, image=a.image,
                            text_tokens=a.text, new_tokens=N, rounds=a.rounds, step_ms_median=round(med, 4),
                            step_ms_p10=round(float(t.quantile(0.1)), 4), step_ms_p90=round(float(t.quantile(0.9)), 4),
                            vs_greedy_median=round(med / greedy_med - 1.0, 4), launches_per_step=launches,
                            select_kernel=kernel, select_kernel_ms=select_kernel_ms(eng, st, kernel))
                print(json.dumps(line), flush=True)
                lines.append(line)
            del states
        del eng, sd
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

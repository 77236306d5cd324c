"""Sampled against greedy CLIP-FlanT5 generation on one H100: clip-flant5-xxl width with synthetic weights drawn on the device, 336x336
images and 32 text ids per prompt, no EOS ids so every run decodes the same number of steps.

Steps: B in {1, 8, 32, 64}, three step types sharing one generation workspace, timed alternately in one process, each round a fresh
prefill then N - 1 graph replays under CUDA events:
  greedy                               generate(do_sample=False)
  sampled T 0.7 / top_k 50 / top_p 0.9  generate(temperature=0.7) with transformers' default top_k
  sampled T 0.7 / top_k 0 / top_p 0.9   a nucleus over the full vocabulary (top_k off)
One JSON line per (batch, step type): median and p10-p90 of the replayed steps over all rounds, launches per step, and the device time
of the selection kernel (V = 32128) in one eager step under torch.profiler.

Prefill: 8 prompts x 8 draws each with encoder sharing (8 encoded prompts expanded to 64 sequences) against 64 distinct prompts, the
same 64-sequence sampled generation otherwise; CUDA events around each prefill, alternating, median over --prefill-reps. Every line
carries the GPU name and power limit read in the same run.

  python tools/bench_sample_clipt5.py [--batches 1,8,32,64] [--new 64] [--rounds 3] [--prefill-reps 5] [--out results.jsonl]
"""
import argparse
import dataclasses
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch

from oracle import clipt5_oracle as orc
from bench_generate import gpu_identity
from bench_sample import select_kernel_ms

STEP_TYPES = {"greedy": None, "sample T0.7 k50 p0.9": (0.7, 50, 0.9), "sample T0.7 k0 p0.9": (0.7, 0, 0.9)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,64")
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--text", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prefill-reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_clipt5.py measures on a CUDA device; there is none")
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.engine import ClipT5Engine
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    cfg = orc.ClipT5Config.xxl()
    N = a.new
    sd = orc.make_synthetic_state_dict(cfg, seed=0, device=dev, gen_device=dev)
    eng = ClipT5Engine(ClipT5Config(**dataclasses.asdict(cfg)), dev)
    eng.load_state_dict(sd)
    del sd
    lines = []
    i32 = lambda t: t.to(dev, torch.int32).contiguous()

    def emit(line):
        line = dict(gpu=gpu, power_limit=power, **line)
        print(json.dumps(line), flush=True)
        lines.append(line)

    for B in [int(x) for x in a.batches.split(",")]:
        inp = orc.make_synthetic_inputs(cfg, B, a.text, seed=1)
        px, ids, lens = inp["pixels"].to(dev).contiguous(), i32(inp["input_ids"]), i32(inp["text_lens"])
        states = {}
        for kind, smp in STEP_TYPES.items():
            sample = None if smp is None else dict(seeds=list(range(B)), temperature=smp[0], top_k=smp[1], top_p=smp[2])
            st = eng.generate_begin(px, ids, lens, N, (), sample=sample)
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
            emit(dict(workload="clip-flant5-xxl generate step", step_type=kind, batch=B, text_tokens=a.text, new_tokens=N, rounds=a.rounds,
                      step_ms_median=round(med, 4), step_ms_p10=round(float(t.quantile(0.1)), 4), step_ms_p90=round(float(t.quantile(0.9)), 4),
                      vs_greedy_median=round(med / greedy_med - 1.0, 4), launches_per_step=launches, select_kernel=kernel,
                      select_kernel_ms=select_kernel_ms(eng, st, kernel)))
        del states

    # prefill of 64 sampled sequences: 8 prompts x 8 draws with sharing, against 64 distinct prompts
    B, P = 64, 8
    inp = orc.make_synthetic_inputs(cfg, B, a.text, seed=2)
    px, ids, lens = inp["pixels"].to(dev).contiguous(), i32(inp["input_ids"]), i32(inp["text_lens"])
    smp = dict(seeds=list(range(B)), temperature=0.7, top_k=50, top_p=0.9)
    pidx = torch.tensor(list(range(P)) + [b % P for b in range(P, B)], dtype=torch.int32, device=dev)
    runs = {"shared 8 prompts x 8 draws": eng.generate_begin(px[:P], ids[:P], lens[:P], N, (), sample=smp, prompt_index=pidx)["prefill"],
            "64 distinct prompts": eng.generate_begin(px, ids, lens, N, (), sample=smp)["prefill"]}
    counts = {}
    for kind, fn in runs.items():
        fn()
        counts[kind] = eng.last_launch_count()
    torch.cuda.synchronize()
    times = {kind: [] for kind in runs}
    for _ in range(a.prefill_reps):
        for kind, fn in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1))
    for kind, t in times.items():
        t = torch.tensor(t)
        emit(dict(workload="clip-flant5-xxl sampled prefill", prefill=kind, batch=B, text_tokens=a.text, reps=a.prefill_reps,
                  prefill_ms_median=round(float(t.median()), 3), prefill_ms_min=round(float(t.min()), 3), prefill_ms_max=round(float(t.max()), 3),
                  launches=counts[kind]))
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

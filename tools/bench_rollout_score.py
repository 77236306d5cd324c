"""Scoring over a greedy rollout on one H100: Qwen2.5-VL width (--model, default qwen2.5-vl-7b) with synthetic weights drawn on the device, 448x448 images and 64 text
tokens per prompt, B in {1, 8, 32}, k in {8, 64} new tokens with no EOS ids so every run decodes k steps. One JSON line per (B, k):
the scored prefill, the median / p10 / p90 of the scored decode step (CUDA events around each graph replay), the plain generate step of
the same shape measured the same way (the cost of the answer log-probability kernel is the difference), launches per step of both, and
pairs/s of a whole scored rollout followed by the reference's step selection on the host (engine.rollout_scores +
qwen_host.rollout_answer_score: what Qwen2VLModel.forward(max_new_tokens=k) runs after image decoding and tokenisation), with the GPU name
and power limit read in the same run.

The baseline is the reference's loop: HF Qwen2_5_VLForConditionalGeneration.generate(do_sample=False, output_scores=True) in bf16 with
sdpa, one sample at a time, min_new_tokens = max_new_tokens, on the same GPU and weights (measured on --hf-samples samples per k).

  python tools/bench_rollout_score.py [--model qwen2.5-vl-3b] [--batches 1,8,32] [--new 8,64] [--no-hf] [--out results.jsonl]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch

from oracle import qwen25vl_oracle as qo
from qwen_bench_model import add_model_arg, engine, hf_model, model_config, synthetic_weights
from bench_generate import gpu_identity

ANSWER = [9454, 11, 432, 1558]          # a four-token answer


def step_times(eng, st, n):
    """CUDA-event times of n graph replays of the state's step after a fresh prefill (captures the graph first if needed)."""
    st["prefill"]()
    if st["graph"] is None:
        eng.generate_step(st)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            eng.generate_step(st)
        st["graph"] = graph
        st["prefill"]()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for s, e in evs:
        s.record()
        st["graph"].replay()
        e.record()
    torch.cuda.synchronize()
    return torch.tensor([s.elapsed_time(e) for s, e in evs])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--new", default="8,64")
    ap.add_argument("--text", type=int, default=64)
    ap.add_argument("--image", type=int, default=448)
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--hf-samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    add_model_arg(ap)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rollout_score.py measures on a CUDA device; there is none")
    from t2v_metrics_b200 import qwen_host
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    cfg, ecfg = model_config(a.model)
    sd = synthetic_weights(cfg, ecfg, dev)
    eng = engine(ecfg, sd, dev)
    news = [int(x) for x in a.new.split(",")]
    lines = []
    for B in [int(x) for x in a.batches.split(",")]:
        inp = qo.make_synthetic_inputs(cfg, B, (a.image, a.image), a.text, seed=1)
        prompts = [x.tolist() for x in inp["input_ids"]]
        pix = inp["pixel_patches"].to(dev)
        answers = [ANSWER] * B
        for N in news:
            score = dict(answer_ids=answers, temperature=1.0, top_k=0)
            eng.rollout_scores(pix, inp["grid_thw"], prompts, answers, N, ())        # warm-up: loads modules, captures the step graph
            eng.generate_prompts(pix, inp["grid_thw"], prompts, N, ())
            st = eng.generate_begin(pix, inp["grid_thw"], prompts, N, (), score=score)
            plain = eng.generate_begin(pix, inp["grid_thw"], prompts, N, ())
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            pre = []
            for _ in range(3):
                e0.record()
                st["prefill"]()
                e1.record()
                torch.cuda.synchronize()
                pre.append(e0.elapsed_time(e1))
            reps = max(1, 64 // (N - 1))          # at least 63 timed steps per kind, alternating scored and plain
            scored, base = [], []
            for _ in range(reps):
                scored.append(step_times(eng, st, N - 1))
                base.append(step_times(eng, plain, N - 1))
            scored, base = torch.cat(scored), torch.cat(base)
            st["prefill"]()
            eng.generate_step(st)
            launches = eng.last_launch_count()
            eng.generate_step(plain)
            plain_launches = eng.last_launch_count()
            special = set()
            runs = 3
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(runs):
                r = eng.rollout_scores(pix, inp["grid_thw"], prompts, answers, N, ())
                scores = [qwen_host.rollout_answer_score(r["tokens"][b], r["logp"][b], answers[b], special, "forward")["score"] for b in range(B)]
            wall = (time.perf_counter() - t0) / runs
            assert all(len(t) == N for t in r["tokens"]) and len(scores) == B
            med, pmed = float(scored.median()), float(base.median())
            line = dict(workload=f"{a.model} scored greedy rollout", gpu=gpu, power_limit=power, batch=B, image=a.image, text_tokens=a.text,
                        prompt_tokens=sum(len(p) for p in prompts) / B, new_tokens=N, answer_tokens=len(ANSWER), timed_steps=int(scored.numel()),
                        prefill_ms=round(min(pre), 3), step_ms_median=round(med, 4), step_ms_p10=round(float(scored.quantile(0.1)), 4),
                        step_ms_p90=round(float(scored.quantile(0.9)), 4), generate_step_ms_median=round(pmed, 4),
                        generate_step_ms_p10=round(float(base.quantile(0.1)), 4), generate_step_ms_p90=round(float(base.quantile(0.9)), 4),
                        step_overhead_ms=round(med - pmed, 4), launches_per_step=launches, generate_launches_per_step=plain_launches,
                        rollout_seconds=round(wall, 4), pairs_per_s=round(B / wall, 2))
            print(json.dumps(line), flush=True)
            lines.append(line)
            del st, plain
    del eng
    torch.cuda.empty_cache()
    if not a.no_hf:
        model = hf_model(cfg, ecfg, sd, dev)
        inp = qo.make_synthetic_inputs(cfg, a.hf_samples, (a.image, a.image), a.text, seed=1)
        P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]

        def run(b, n):
            ids = inp["input_ids"][b].to(dev)
            with torch.no_grad():
                out = model.generate(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long, device=dev),
                                     pixel_values=inp["pixel_patches"][b * P:(b + 1) * P].to(dev, torch.bfloat16),
                                     image_grid_thw=torch.tensor([list(inp["grid_thw"][b])], device=dev),
                                     mm_token_type_ids=(ids == cfg.image_token_id).long()[None], max_new_tokens=n, min_new_tokens=n,
                                     do_sample=False, temperature=1.0, eos_token_id=None, pad_token_id=0, output_scores=True,
                                     return_dict_in_generate=True)
                probs = [torch.softmax(s[0].float(), -1)[ANSWER[i]].item() for i, s in enumerate(out.scores[-len(ANSWER):])]
            return probs
        run(0, 4)
        for N in news:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for b in range(a.hf_samples):
                run(b, N)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            line = dict(workload="HF generate(do_sample=False, output_scores=True) bf16 sdpa, one sample at a time", gpu=gpu, power_limit=power,
                        samples=a.hf_samples, image=a.image, text_tokens=a.text, new_tokens=N, seconds=round(dt, 3),
                        pairs_per_s=round(a.hf_samples / dt, 3))
            print(json.dumps(line), flush=True)
            lines.append(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

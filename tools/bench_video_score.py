"""Video scoring on one H100: Qwen2.5-VL width (--model, default qwen2.5-vl-7b) with synthetic weights drawn on the device, decoded uint8 frame stacks on the host
(8 frames of 448x448 = 1024 video tokens, 32 frames of 336x336 = 2304 video tokens), two videos per call with 1 or 8 texts each, scored
with k = 1 (one prefill, QwenVLEngine.score_prompts) and k = 4 (a scored greedy rollout, QwenVLEngine.rollout_scores). One JSON line per
(shape, texts, k): the device pre-processing of the call's stacks (qwen_preprocess_video_u8: pinned staging, H2D, one kernel), the
scoring call, and pairs/s of both together, each the best of a few runs timed with CUDA events; the GPU name and power limit are read in
the same run.

The baseline is the reference's loop on the same GPU and weights: per pair, the frames pre-processed on the CPU
(qwen_utils.qwen_video_to_patches, the restated qwen_vl_utils + processor path) and HF Qwen2_5_VLForConditionalGeneration in bf16 with
sdpa: one forward for k = 1, generate(do_sample=False, output_scores=True, max_new_tokens=4) for k = 4.

  python tools/bench_video_score.py [--model qwen2.5-vl-3b] [--no-hf] [--hf-samples 2] [--out results.jsonl]
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
import numpy as np
import torch

from oracle import qwen25vl_oracle as qo
from qwen_bench_model import add_model_arg, engine, hf_model, model_config, synthetic_weights
from bench_generate import gpu_identity

SHAPES = [(8, 448), (32, 336)]          # (frames, side)
ANSWER = [9454, 11, 432, 1558]
VIDEOS = 2


def stacks(frames, side, n, seed=0):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.integers(0, 256, (frames, side, side, 3), dtype=np.uint8)) for _ in range(n)]


def prompts_for(cfg, grids, texts, seed=1):
    """Chat-like prompts: 4 prefix ids, the video-token run, 24 text ids per text."""
    g = torch.Generator().manual_seed(seed)
    out, idx = [], []
    for v, (t, h, w) in enumerate(grids):
        for _ in range(texts):
            out.append([5, 6, 7, 8] + [cfg.video_token_id] * (t * h * w // 4) + torch.randint(0, 30000, (24,), generator=g).tolist())
            idx.append(v)
    return out, idx


def sm_clocks():
    """Current and maximum SM clock (read-only query), read right after the timed work."""
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def best_ms(fn, runs=3):
    times = []
    for _ in range(runs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return min(times), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--hf-samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    add_model_arg(ap)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_video_score.py measures on a CUDA device; there is none")
    from t2v_metrics_b200.engine import qwen_preprocess_video_u8
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    cfg, ecfg = model_config(a.model)
    sd = synthetic_weights(cfg, ecfg, dev)
    eng = engine(ecfg, sd, dev)
    spg_of = lambda n: [cfg.temporal_patch_size / 24] * n
    lines = []
    for frames, side in SHAPES:
        vids = stacks(frames, side, VIDEOS)
        pre = lambda: qwen_preprocess_video_u8(vids, dev, max_pixels=16384 * 28 * 28)
        pre()
        pre_ms, (patches, grids) = best_ms(pre)
        for texts in (1, 8):
            prompts, idx = prompts_for(cfg, grids, texts)
            for k in (1, 4):
                if k == 1:
                    call = lambda: eng.score_prompts(patches, grids, prompts, [ANSWER[0]] * len(prompts), image_of_sample=idx,
                                                     second_per_grid_ts=spg_of(VIDEOS))
                else:
                    call = lambda: eng.rollout_scores(patches, grids, prompts, [ANSWER] * len(prompts), k, (), image_of_sample=idx,
                                                      second_per_grid_ts=spg_of(VIDEOS))
                call()
                score_ms, _ = best_ms(call)
                line = dict(workload=f"{a.model} video scoring from host uint8 frame stacks", gpu=gpu, power_limit=power, frames=frames,
                            side=side, videos=VIDEOS, texts_per_video=texts, pairs=len(prompts), video_tokens=grids[0][0] * grids[0][1] * grids[0][2] // 4,
                            prompt_tokens=len(prompts[0]), k=k, preprocess_ms=round(pre_ms, 3),
                            **{"prefill_ms" if k == 1 else "rollout_ms": round(score_ms, 3)},
                            pairs_per_s=round(len(prompts) / ((pre_ms + score_ms) / 1e3), 2), sm_clock=sm_clocks())
                print(json.dumps(line), flush=True)
                lines.append(line)
    del eng
    torch.cuda.empty_cache()
    if not a.no_hf:
        from t2v_metrics_b200.models.vqascore_models.qwen_utils import qwen_video_to_patches
        model = hf_model(cfg, ecfg, sd, dev)
        for frames, side in SHAPES:
            vids = stacks(frames, side, a.hf_samples)
            for k in (1, 4):
                def one(v):
                    px, grid = qwen_video_to_patches(v.numpy(), max_pixels=16384 * 28 * 28)
                    (ids,), _ = prompts_for(cfg, [grid], 1)
                    ids = torch.tensor(ids, device=dev)
                    kw = dict(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long, device=dev),
                              pixel_values_videos=px.to(dev, torch.bfloat16), video_grid_thw=torch.tensor([list(grid)], device=dev),
                              second_per_grid_ts=torch.tensor([cfg.temporal_patch_size / 24], device=dev),
                              mm_token_type_ids=torch.where(ids == cfg.video_token_id, 2, 0)[None])
                    with torch.no_grad():
                        if k == 1:
                            return torch.softmax(model(**kw).logits[0, -1].float(), -1)[ANSWER[0]].item()
                        out = model.generate(**kw, max_new_tokens=k, min_new_tokens=k, do_sample=False, temperature=1.0, eos_token_id=None,
                                             pad_token_id=0, output_scores=True, return_dict_in_generate=True)
                        return [torch.softmax(s[0].float(), -1)[ANSWER[i]].item() for i, s in enumerate(out.scores)]
                one(vids[0])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for v in vids:
                    one(v)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                line = dict(workload="HF bf16 sdpa, one pair at a time, CPU pre-processing of the same frames", gpu=gpu, power_limit=power,
                            frames=frames, side=side, samples=a.hf_samples, k=k, seconds=round(dt, 3), pairs_per_s=round(a.hf_samples / dt, 3))
                print(json.dumps(line), flush=True)
                lines.append(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

"""Video-file scoring on one H100: a synthesized 640x360, 24 fps, 21 s clip (504 frames, the shape of the reference README's baby.mp4,
MJPG in .avi, written to a temporary directory), Qwen2.5-VL width (--model, default qwen2.5-vl-7b) with synthetic weights drawn on the
device. For fps 8.0 (168 frames) and "dynamic" (qwen_vl_utils' 2.0: 42 frames), each resized to 280x504 under the 360*420 pixel budget, one JSON line per (fps, B):
  decode_ms      OpenCV decoding of the sampled frames (qwen_utils.OpenCVVideoReader: counting by decoding, then the frames), host clock
  preprocess_ms  engine.qwen_preprocess_video_file_u8 on the decoded frames (pinned staging, H2D, one kernel per slice), CUDA events
  score_ms       QwenVLEngine.score_prompts for B texts on the clip (one prefill of B prompts of the video tokens + 24 text ids)
each the best of a few runs; the GPU name and power limit are read in the same run.

  python tools/bench_video_file_score.py [--model qwen2.5-vl-3b] [--out results.jsonl]
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

from bench_generate import gpu_identity
from bench_video_score import best_ms, prompts_for
from qwen_bench_model import add_model_arg, engine, model_config, synthetic_weights


def write_clip(path, frames=504, h=360, w=640, fps=24.0):
    """Moving colour gradients with a little noise, frame by frame (the clip is never held in memory as a whole)."""
    import cv2
    rng = np.random.default_rng(0)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    wr = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), fps, (w, h))
    for f in range(frames):
        img = np.stack([128 + 100 * np.sin(x / 40 + f / 9), 128 + 100 * np.cos(y / 30 - f / 13), 128 + 90 * np.sin((x + y) / 50 + f / 5)], -1)
        wr.write(np.clip(img + rng.normal(0, 6, img.shape), 0, 255).astype(np.uint8))
    wr.release()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    add_model_arg(ap)
    args = ap.parse_args()
    from t2v_metrics_b200.engine import qwen_preprocess_video_file_u8
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import VIDEO_FILE_MAX_PIXELS
    from t2v_metrics_b200.models.vqascore_models.qwen_utils import OpenCVVideoReader, qwen_video_file_plan
    dev = torch.device("cuda:0")
    cfg, ecfg = model_config(args.model)
    sd = synthetic_weights(cfg, ecfg, dev)
    eng = engine(ecfg, sd, dev)
    del sd
    name, power = gpu_identity()
    ident = dict(model=args.model, gpu=name, power_limit=power)
    lines = []
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "clip.avi")
        write_clip(path)
        for fps in (8.0, "dynamic"):
            decode = []
            for _ in range(3):
                t0 = time.perf_counter()
                total, avg_fps, get = OpenCVVideoReader().open(path)
                idx, _, size = qwen_video_file_plan(total, avg_fps, 360, 640, fps=None if fps == "dynamic" else fps,
                                                    max_pixels=VIDEO_FILE_MAX_PIXELS)
                frames = torch.from_numpy(get(idx))
                decode.append((time.perf_counter() - t0) * 1e3)
            pre = lambda: qwen_preprocess_video_file_u8(frames, size, dev, patch=cfg.patch_size, temporal_patch=cfg.temporal_patch_size,
                                                        merge=cfg.spatial_merge_size)
            pre_ms, (patches, grid) = best_ms(pre, runs=5)
            for B in (1, 8):
                prompts, image_of = prompts_for(cfg, [grid], B)
                call = lambda: eng.score_prompts(patches, [grid], prompts, [9454] * B, image_of_sample=image_of,
                                                 second_per_grid_ts=[cfg.temporal_patch_size / 24])
                score_ms, _ = best_ms(call, runs=3)
                rec = dict(fps=fps, frames=len(idx), size=list(size), grid_thw=list(grid), video_tokens=grid[0] * grid[1] * grid[2] // 4,
                           texts=B, decode_ms=round(min(decode), 1), preprocess_ms=round(pre_ms, 2), score_ms=round(score_ms, 1),
                           pairs_per_s=round(B / (score_ms / 1e3), 2), **ident)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in lines)


if __name__ == "__main__":
    main()

"""CLIP-FlanT5 video scoring by frame concatenation on one GPU, stage by stage. Synthesizes 21 s clips (24 fps) at 640x360 and
1280x720 as MJPG .avi and mp4v .mp4 (seek cost differs by codec) in a temporary directory, then for num_frames 8 / 16 and N = 1 / 8
texts per video prints one JSON line with, separately:
  extract_ms   frame extraction (container count, seeks) plus the per-frame JPEG round trips (host clock)
  canvas_ms    the canvas JPEG encode plus PIL's decode of it (host clock)
  resize_ms    H2D copy plus the device resize of the canvas to 336x336 (host clock around the call and a synchronise), and
  resize_dev_ms  the same window in CUDA events
  score_ms     the engine's scoring of the N pairs from the device pixels (CUDA events)
  pairs_per_s  N over the whole plugin call forward([video] * N, texts, num_frames) (host clock, synchronised)
at clip-flant5-xxl width with synthetic weights and a stand-in tokenizer, medians of --reps runs after a warm-up, with the GPU name
and power limit read in the same run. --stills prints one line instead: clip_preprocess_u8 on 64 x 512^2 and 64 x 640x400 host images
(median of CUDA-event times over --reps calls), for comparing builds of the library (VQA_B200_LIB).

  python tools/bench_clipt5_video.py [--stills] [--reps 5]
"""
import argparse
import dataclasses
import json
import os
import statistics
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

from oracle import clipt5_oracle as orc
from bench_generate import gpu_identity


def synth_clip(path, fourcc, w, h, seconds=21, fps=24):
    import cv2
    wr = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*fourcc), fps, (w, h))
    assert wr.isOpened(), fourcc
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([x * 255 // (w - 1), y * 255 // (h - 1), (x + y) % 256], -1).astype(np.uint8)
    for i in range(seconds * fps):
        f = base.copy()
        s = (i * 7) % (w - h // 4)
        f[h // 3: h // 3 + h // 4, s:s + h // 4] = (0, 0, 255)
        wr.write(f)
    wr.release()


def host_ms(fn, reps):
    times, out = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(times), out


def event_ms(fn, reps):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def stills(dev, reps, ident):
    from t2v_metrics_b200.engine import clip_preprocess_u8
    g = torch.Generator().manual_seed(0)
    line = dict(bench="clipt5_stills", lib=os.environ.get("VQA_B200_LIB", "default"), **ident)
    for name, (h, w) in (("512x512", (512, 512)), ("640x400", (400, 640))):
        imgs = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for _ in range(64)]
        for _ in range(3):
            clip_preprocess_u8(imgs, 336, dev)
        torch.cuda.synchronize()
        line[f"ms_64x{name}"] = round(event_ms(lambda: clip_preprocess_u8(imgs, 336, dev), reps), 4)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stills", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clipt5_video.py measures on a CUDA device; there is none")
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    ident = dict(gpu=gpu, power_limit=power)
    if a.stills:
        return stills(dev, a.reps, ident)

    import t2v_metrics_b200 as t2v
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.engine import clip_preprocess_u8_sliced
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import default_question_template, format_question, format_answer
    from t2v_metrics_b200.models.vqascore_models.mm_utils import concat_frames_rgb, video_frames_bgr

    class Tok:
        pad_token_id = 0

        def __call__(self, chunk):
            return types.SimpleNamespace(input_ids=[3 + (sum(map(ord, w)) % 30000) for w in chunk.split()] + [1])

    cfg = orc.ClipT5Config.xxl()
    sd = orc.make_synthetic_state_dict(cfg, seed=0, device=dev, gen_device=dev)
    scorer = t2v.VQAScore(model="clip-flant5-xxl", device="cuda", cache_dir=tempfile.mkdtemp(), tokenizer=Tok(), state_dict=sd,
                          config=ClipT5Config(**dataclasses.asdict(cfg)))
    model = scorer.model
    del sd
    texts8 = [f"a red square moving across a gradient, caption number {i}" for i in range(8)]
    with tempfile.TemporaryDirectory() as tmp:
        for (w, h) in ((640, 360), (1280, 720)):
            for fourcc, ext in (("MJPG", "avi"), ("mp4v", "mp4")):
                path = os.path.join(tmp, f"clip_{w}x{h}.{ext}")
                synth_clip(path, fourcc, w, h)
                for nf in (8, 16):
                    for n in (1, 8):
                        texts = texts8[:n]
                        model.forward([path] * n, texts, num_frames=nf)           # warm-up (graphs, modules, allocator)
                        torch.cuda.synchronize()
                        t_ext, frames = host_ms(lambda: video_frames_bgr(path, nf), a.reps)
                        t_can, canvas = host_ms(lambda: concat_frames_rgb(frames), a.reps)
                        src = torch.from_numpy(canvas)
                        t_rs, pixels = host_ms(lambda: clip_preprocess_u8_sliced([src], cfg.image_size, dev), a.reps)
                        t_rs_dev = event_ms(lambda: clip_preprocess_u8_sliced([src], cfg.image_size, dev), a.reps)
                        qs = [format_question(default_question_template.format(t)) for t in texts]
                        ids, lens, labels = model._tokenize(qs, [format_answer("Yes")] * n)
                        idx = torch.zeros(n, dtype=torch.int32, device=dev) if n > 1 else None
                        args = (pixels, ids.to(dev), lens.to(dev), labels.to(dev))
                        t_score = event_ms(lambda: model.engine.score_tensors(*args, image_index=idx), a.reps)
                        t_call, _ = host_ms(lambda: model.forward([path] * n, texts, num_frames=nf), a.reps)
                        print(json.dumps(dict(bench="clipt5_video", clip=f"{w}x{h}", codec=fourcc, seconds=21, fps=24, num_frames=nf,
                                              texts=n, canvas=f"{canvas.shape[1]}x{canvas.shape[0]}", extract_ms=round(t_ext, 3),
                                              canvas_ms=round(t_can, 3), resize_ms=round(t_rs, 3), resize_dev_ms=round(t_rs_dev, 3),
                                              score_ms=round(t_score, 3), call_ms=round(t_call, 3),
                                              pairs_per_s=round(n / (t_call / 1e3), 2), **ident)), flush=True)


if __name__ == "__main__":
    main()

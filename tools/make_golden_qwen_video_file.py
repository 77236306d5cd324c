"""Generate tests/golden/qwen_video_file_tiny.pt: a small synthesized video FILE and what the REAL transformers
Qwen2_5_VLForConditionalGeneration (fp32, the tiny config and seeded weights of tools/make_golden_qwen.py) scores on it, fed the way the
reference feeds a file: qwen_vl_utils fetch_video samples frames at `fps` and resizes them with torchvision's antialiased bicubic
(restated in qwen_utils.qwen_video_file_plan / qwen_video_file_to_patches), and the installed Qwen2VLVideoProcessor runs with
do_resize=False. Frames are decoded by qwen_utils.OpenCVVideoReader.

The clip: 12 frames of 64x96 at 12 fps (1 s), moving colour gradients, MJPG in .avi; its bytes are stored. For fps 8.0 and "dynamic"
(2.0) the golden holds the sampled indices, the resized size, the grid and second_per_grid_ts, and for the default question about TEXT: the last-position logits and answer probability; for fps 8.0 also the greedy `generate` ids of 8 steps from the raw text and
the per-step answer probabilities of a 4-step rollout of the scoring prompt, with the top-1 / top-2 margins. The patches are not
stored: min_pixels makes every frame at least 128 * 28 * 28 pixels, 2.6 MB of levels for the 8 frames even losslessly packed, and
tests/test_qwen_video_file_host.py rebuilds them from the clip.

  python tools/make_golden_qwen_video_file.py
"""
import dataclasses
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch
from transformers import Qwen2VLVideoProcessor

from oracle import qwen25vl_oracle as qo
from test_qwen_host import hf_model, TINY
from test_qwen_video_host import CharTokenizer
from test_qwen_video_file_host import smooth_frames, write_clip
from make_golden_qwen import sd_checksum
from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import VIDEO_FILE_MAX_PIXELS
from t2v_metrics_b200.models.vqascore_models.qwen_utils import (OpenCVVideoReader, build_prompt_ids, default_answer_template,
                                                                default_question_template, qwen_video_file_plan, qwen_video_file_to_patches)

GOLD = os.path.join(ROOT, "tests", "golden")
FRAMES, H, W, CLIP_FPS = 12, 64, 96, 12.0
TEXT = "a red car"
GEN_STEPS, ROLLOUT_STEPS = 8, 4


@torch.no_grad()
def main():
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m = hf_model(cfg)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    tok = CharTokenizer()
    unit = cfg.spatial_merge_size ** 2
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "clip.avi")
        write_clip(path, smooth_frames(FRAMES, H, W, seed=3), CLIP_FPS)
        clip = open(path, "rb").read()
        total, avg_fps, get = OpenCVVideoReader().open(path)
        decoded = get(list(range(total)))
    blob = dict(config=dataclasses.asdict(cfg), weights_seed=0, weights_sha256=sd_checksum(sd), clip=clip, clip_ext=".avi", text=TEXT,
                gen_steps=GEN_STEPS, rollout_steps=ROLLOUT_STEPS, runs={})
    answer = tok.encode(default_answer_template, add_special_tokens=False)
    margins = lambda o: torch.stack([s[0].float().topk(2).values for s in o.scores]).diff(dim=-1)[:, 0].neg()
    for fps in (8.0, "dynamic"):
        idx, _, size = qwen_video_file_plan(total, avg_fps, H, W, fps=None if fps == "dynamic" else fps, max_pixels=VIDEO_FILE_MAX_PIXELS)
        resized, _, _ = qwen_video_file_to_patches(decoded[idx], size)
        pv = Qwen2VLVideoProcessor()(videos=[resized.permute(0, 3, 1, 2).float()], do_resize=False, return_metadata=True,
                                     return_tensors="pt", fps=8.0 if fps == "dynamic" else fps)
        grid = [int(v) for v in pv["video_grid_thw"][0]]
        spg = cfg.temporal_patch_size / pv["video_metadata"][0].sampled_fps      # processing_qwen2_5_vl.py:103-113
        px = pv["pixel_values_videos"].float()
        ntok = grid[0] * grid[1] * grid[2] // unit
        vis = dict(pixel_values_videos=px, video_grid_thw=torch.tensor([grid]), second_per_grid_ts=torch.tensor([spg]))

        def run(ids):
            ids = torch.tensor(ids)[None]
            return dict(input_ids=ids, attention_mask=torch.ones_like(ids), mm_token_type_ids=torch.where(ids == cfg.video_token_id, 2, 0), **vis)

        score_ids = build_prompt_ids(tok, default_question_template.format(TEXT), ntok, cfg.video_token_id)
        logits = m(**run(score_ids)).logits[0, -1].float().clone()
        r = dict(indices=idx, size=list(size), grid_thw=grid, second_per_grid_ts=spg, score_prompt=score_ids, answer_ids=answer,
                 logits=logits, probs=float(torch.softmax(logits, -1)[answer[0]]))
        if fps == 8.0:
            gen_ids = build_prompt_ids(tok, TEXT, ntok, cfg.video_token_id)
            g = m.generate(**run(gen_ids), max_new_tokens=GEN_STEPS, do_sample=False, repetition_penalty=1.0, pad_token_id=0,
                           output_scores=True, return_dict_in_generate=True)
            ro = m.generate(**run(score_ids), max_new_tokens=ROLLOUT_STEPS, do_sample=False, repetition_penalty=1.0, pad_token_id=0,
                            output_scores=True, return_dict_in_generate=True)
            rscores = torch.stack([s[0].float() for s in ro.scores])
            r.update(generate_prompt=gen_ids, generate_ids=g.sequences[0, len(gen_ids):].tolist(), generate_margins=margins(g),
                     rollout_ids=ro.sequences[0, len(score_ids):].tolist(), rollout_probs=torch.softmax(rscores, -1)[:, answer].clone(),
                     rollout_margins=margins(ro))
        blob["runs"][str(fps)] = r
        print(f"fps {fps}: {len(idx)} frames {idx} size {size} grid {grid} spg {spg:.6f} P {r['probs']:.6f}")
    out = os.path.join(GOLD, "qwen_video_file_tiny.pt")
    torch.save(blob, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB; clip", len(clip) // 1024, "KiB")


if __name__ == "__main__":
    main()

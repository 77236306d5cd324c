"""Generate tests/golden/qwen_video_tiny.pt from the REAL transformers Qwen2_5_VLForConditionalGeneration in fp32 (committed with this
script), fed by the installed Qwen2VLVideoProcessor the way the reference's decoder-free video path feeds it: a 4-D .npy frame stack becomes
a list of PIL frames (qwen2vl_model.py:145-153), qwen_vl_utils `fetch_video` resizes each frame like a still image and pads the count to
an even number with the last frame (restated in qwen_utils.qwen_video_to_patches), and the processor runs with do_resize=False. The tiny
config and seeded weights of tools/make_golden_qwen.py. Three uint8 stacks: 4 frames of 56x84, 5 frames of 84x112 (an odd count) and
2 frames of 50x90 (resized to 56x84). Prompt i is the default question about TEXTS[i] over stack i, tokenised by the stand-in
tokenizer of tests/test_qwen_video_host.py. Stored per stack: the frames, the processor's patches (losslessly, as the uint8 level of every element and the processor's
fp32 value of each (channel, level): tests/test_qwen_video_host.load_video_golden rebuilds them bit for bit), grid and second_per_grid_ts; per
prompt: the last-position logits and answer probabilities, plain and after repetition penalty 1.3 / temperature 0.5, the greedy
`generate` ids of 8 steps from the raw text, and the per-step answer probabilities of a 4-step `generate(output_scores=True)` rollout
from the scoring prompt, with the top-1 / top-2 margin of every step.

  python tools/make_golden_qwen_video.py
"""
import dataclasses
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch
from PIL import Image
from transformers import Qwen2VLVideoProcessor
from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor

from oracle import qwen25vl_oracle as qo
from test_qwen_host import hf_model, TINY
from make_golden_qwen import sd_checksum
from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import QWEN_VL_UTILS_MIN_PIXELS, QWEN_VL_UTILS_MAX_PIXELS
from t2v_metrics_b200.models.vqascore_models.qwen_utils import (build_prompt_ids, default_question_template, default_answer_template,
                                                                smart_resize)
from test_qwen_video_host import CharTokenizer

GOLD = os.path.join(ROOT, "tests", "golden")
STACKS = [(4, 56, 84), (5, 84, 112), (2, 50, 90)]       # (frames, h, w)
TEXTS = ["a red car", "two dogs", "a blue sky"]
GEN_STEPS, ROLLOUT_STEPS = 8, 4


def make_frames(n, h, w, seed):
    """Smooth moving gradients plus noise: frames that differ from each other, so a wrong frame order is visible."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    out = []
    for f in range(n):
        base = np.stack([(x * 7 + f * 40) % 256, (y * 5 + f * 25) % 256, ((x + y) * 3 + f * 60) % 256], -1)
        out.append(np.clip(base + rng.integers(-30, 31, (h, w, 3)), 0, 255))
    return np.stack(out).astype(np.uint8)


def patch_levels(frames, temporal=2, patch=14, merge=2):
    """The uint8 level behind every element of the processor's patch rows: the fetched frames in Qwen2VLVideoProcessor's layout
    (video_processing_qwen2_vl.py:245-272) -> [t*gh*gw, 3*temporal*patch*patch] uint8."""
    x = torch.from_numpy(np.stack([np.asarray(f, dtype=np.uint8) for f in frames])).permute(0, 3, 1, 2)
    x = torch.cat([x, x[-1:].expand(-x.shape[0] % temporal, -1, -1, -1)])
    gt, gh, gw = x.shape[0] // temporal, x.shape[2] // patch, x.shape[3] // patch
    x = x.reshape(gt, temporal, 3, gh // merge, merge, patch, gw // merge, merge, patch).permute(0, 3, 6, 4, 7, 2, 1, 5, 8)
    return x.reshape(gt * gh * gw, -1).contiguous()


def compress_patches(px, levels):
    """The processor's fp32 patches as (uint8 levels, fp32 value table [3, 256]): its rescale + normalise maps each (channel, level) to one
    value, so table[channel, level] gives every element back bit for bit (checked here); a quarter of the bytes."""
    chan = torch.arange(px.shape[1]) // (px.shape[1] // 3)
    table = torch.full((3, 256), float("nan"))
    table[chan.expand_as(levels), levels.long()] = px
    assert torch.equal(table[chan.expand_as(levels), levels.long()], px), "the processor's values are not a function of (channel, level)"
    return table


def fetch_video_frames(frames):
    """qwen_vl_utils 0.0.8 fetch_video, list branch: fetch_image on every frame (smart_resize(factor 28) + PIL resize, BICUBIC by default),
    then the count padded to a multiple of FRAME_FACTOR = 2 with the last frame."""
    out = []
    for f in frames:
        im = Image.fromarray(f.astype("uint8"), "RGB")
        rh, rw = smart_resize(im.height, im.width, 28, QWEN_VL_UTILS_MIN_PIXELS, QWEN_VL_UTILS_MAX_PIXELS)
        out.append(im.resize((rw, rh), resample=Image.BICUBIC))
    out += [out[-1]] * (-len(out) % 2)
    return out


@torch.no_grad()
def main():
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m = hf_model(cfg)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    tok = CharTokenizer()
    vp = Qwen2VLVideoProcessor()
    unit = cfg.spatial_merge_size ** 2
    blob = dict(config=dataclasses.asdict(cfg), weights_seed=0, weights_sha256=sd_checksum(sd), texts=TEXTS, gen_steps=GEN_STEPS,
                rollout_steps=ROLLOUT_STEPS, stacks=[])
    pen = RepetitionPenaltyLogitsProcessor(1.3)
    for i, ((n, h, w), text) in enumerate(zip(STACKS, TEXTS)):
        frames = make_frames(n, h, w, seed=100 + i)
        pv = vp(videos=[fetch_video_frames(frames)], do_resize=False, return_metadata=True, return_tensors="pt")
        grid = [int(v) for v in pv["video_grid_thw"][0]]
        spg = cfg.temporal_patch_size / pv["video_metadata"][0].sampled_fps      # processing_qwen2_5_vl.py:103-113
        fetched = fetch_video_frames(frames)
        px = pv["pixel_values_videos"].float()
        levels = patch_levels(fetched)
        table = compress_patches(px, levels)
        ntok = grid[0] * grid[1] * grid[2] // unit
        vis = dict(pixel_values_videos=px, video_grid_thw=torch.tensor([grid]), second_per_grid_ts=torch.tensor([spg]))

        def run(ids):
            ids = torch.tensor(ids)[None]
            return dict(input_ids=ids, attention_mask=torch.ones_like(ids), mm_token_type_ids=torch.where(ids == cfg.video_token_id, 2, 0), **vis)

        score_ids = build_prompt_ids(tok, default_question_template.format(text), ntok, cfg.video_token_id)
        answer = tok.encode(default_answer_template, add_special_tokens=False)
        logits = m(**run(score_ids)).logits[0, -1].float().clone()
        probs = float(torch.softmax(logits, -1)[answer[0]])
        probs_pen = float(torch.softmax(pen(torch.tensor([score_ids]), logits[None].clone())[0] / 0.5, -1)[answer[0]])
        gen_ids = build_prompt_ids(tok, text, ntok, cfg.video_token_id)
        g = m.generate(**run(gen_ids), max_new_tokens=GEN_STEPS, do_sample=False, repetition_penalty=1.0, pad_token_id=0, output_scores=True,
                       return_dict_in_generate=True)
        r = m.generate(**run(score_ids), max_new_tokens=ROLLOUT_STEPS, do_sample=False, repetition_penalty=1.0, pad_token_id=0,
                       output_scores=True, return_dict_in_generate=True)
        margins = lambda o: torch.stack([s[0].float().topk(2).values for s in o.scores]).diff(dim=-1)[:, 0].neg()
        rscores = torch.stack([s[0].float() for s in r.scores])
        blob["stacks"].append(dict(
            frames=torch.from_numpy(frames), patch_levels=levels, patch_table=table, grid_thw=grid, second_per_grid_ts=spg, score_prompt=score_ids, answer_ids=answer,
            logits=logits, probs=probs, probs_penalty_1p3_T_0p5=probs_pen,
            generate_prompt=gen_ids, generate_ids=g.sequences[0, len(gen_ids):].tolist(), generate_margins=margins(g),
            rollout_ids=r.sequences[0, len(score_ids):].tolist(), rollout_probs=torch.softmax(rscores, -1)[:, answer].clone(),
            rollout_margins=margins(r)))
        s = blob["stacks"][-1]
        print(f"stack {i}: grid {grid} spg {spg:.6f} P {probs:.6f} penalised {probs_pen:.6f} generate {s['generate_ids']} "
              f"(min margin {float(s['generate_margins'].min()):.4f}) rollout {s['rollout_ids']} (min margin {float(s['rollout_margins'].min()):.4f})")
    path = os.path.join(GOLD, "qwen_video_tiny.pt")
    torch.save(blob, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

"""Generate tests/golden/qwen_generate_tiny.pt from the REAL transformers Qwen2_5_VLForConditionalGeneration.generate(do_sample=False) in
fp32 (committed with this script). The tiny config and seeded weights of tools/make_golden_qwen.py; the inputs (seeds picked for
top-1 / top-2 margins above 0.1 over several steps: random tiny weights give flat logits) are regenerated from their
seeds by the tests (make_synthetic_inputs) and pinned by a checksum, so the file holds ids and margins only. Cases:
  * images:   3 prompts over 2 images (grid 1x6x4), ragged text, repetition penalty 1.0 and 1.3, no EOS
  * video:    2 prompts, each its own 2-temporal-patch clip (grid 2x4x6), second_per_grid 2.0, penalty 1.0 and 1.3, no EOS
  * eos:      the images prompts with EOS ids = {a token prompt 2 emits mid-way without EOS, an id never emitted}: prompt 2 stops on it
Each entry stores HF's generated ids per prompt and, per step, the fp32 margin between the top two processed scores (output_scores).

  python tools/make_golden_qwen_generate.py
"""
import dataclasses
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from oracle import qwen25vl_oracle as qo
from test_qwen_host import hf_model, TINY
from make_golden_qwen import sd_checksum

GOLD = os.path.join(ROOT, "tests", "golden")
MAX_NEW = 16
CASES = dict(images=dict(batch=3, hw=(84, 56), text_len=12, seed=5, ragged=True, n_images=2, frames=1, spg=None),
             video=dict(batch=2, hw=(56, 84), text_len=10, seed=4, ragged=True, n_images=None, frames=2, spg=[2.0, 2.0]))


def case_inputs(cfg, spec):
    return qo.make_synthetic_inputs(cfg, spec["batch"], spec["hw"], spec["text_len"], seed=spec["seed"], ragged=spec["ragged"],
                                    n_images=spec["n_images"], frames=spec["frames"])


def inputs_checksum(inp):
    h = hashlib.sha256()
    h.update(inp["pixel_patches"].contiguous().numpy().tobytes())
    for ids in inp["input_ids"]:
        h.update(ids.to(torch.int64).numpy().tobytes())
    return h.hexdigest()


@torch.no_grad()
def hf_generate(m, cfg, inp, spg, max_new, penalty, eos_ids):
    """generate(do_sample=False) per prompt, as the reference runs it (qwen2vl_model.py:495-563). Returns (ids, margins) per prompt."""
    t, gh, gw = inp["grid_thw"][0]
    P = t * gh * gw
    video = t > 1
    out_ids, out_margins = [], []
    for b, ids in enumerate(inp["input_ids"]):
        img = inp["image_of_sample"][b] if inp["image_of_sample"] is not None else b
        px = inp["pixel_patches"][img * P:(img + 1) * P]
        grid = torch.tensor([list(inp["grid_thw"][img])])
        kw = dict(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long))
        if video:
            kw.update(pixel_values_videos=px, video_grid_thw=grid, second_per_grid_ts=torch.tensor([spg[img]]),
                      mm_token_type_ids=torch.where(ids == cfg.video_token_id, 2, 0)[None])
        else:
            kw.update(pixel_values=px, image_grid_thw=grid, mm_token_type_ids=(ids == cfg.image_token_id).long()[None])
        out = m.generate(**kw, max_new_tokens=max_new, do_sample=False, repetition_penalty=penalty, eos_token_id=list(eos_ids) or None,
                         pad_token_id=0, output_scores=True, return_dict_in_generate=True)
        gen = out.sequences[0, len(ids):].tolist()
        top2 = torch.stack([s[0].float().topk(2).values for s in out.scores])
        out_ids.append(gen)
        out_margins.append((top2[:, 0] - top2[:, 1]).clone())
    return out_ids, out_margins


def main():
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m = hf_model(cfg)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    blob = dict(config=dataclasses.asdict(cfg), weights_seed=0, weights_sha256=sd_checksum(sd), max_new_tokens=MAX_NEW, cases={})
    for name, spec in CASES.items():
        inp = case_inputs(cfg, spec)
        for pen in (1.0, 1.3):
            ids, margins = hf_generate(m, cfg, inp, spec["spg"], MAX_NEW, pen, ())
            blob["cases"][f"{name}_pen{pen}"] = dict(inputs=spec, inputs_sha256=inputs_checksum(inp), penalty=pen, eos_ids=[], ids=ids,
                                                      margins=margins)
    base = blob["cases"]["images_pen1.0"]["ids"]
    stop = base[2][5]
    never = next(t for t in range(cfg.vocab) if all(t not in x for x in base))
    spec = CASES["images"]
    inp = case_inputs(cfg, spec)
    ids, margins = hf_generate(m, cfg, inp, None, MAX_NEW, 1.0, (stop, never))
    assert len(ids[2]) < MAX_NEW and ids[2][-1] == stop
    blob["cases"]["eos"] = dict(inputs=spec, inputs_sha256=inputs_checksum(inp), penalty=1.0, eos_ids=[stop, never], ids=ids, margins=margins)
    path = os.path.join(GOLD, "qwen_generate_tiny.pt")
    torch.save(blob, path)
    for name, c in blob["cases"].items():
        print(name, c["ids"], "min margin", [round(float(x.min()), 4) for x in c["margins"]])
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

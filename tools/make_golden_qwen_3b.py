"""Generate tests/golden/qwen_tied_gqa8_tiny.pt from the REAL transformers Qwen2_5_VLForConditionalGeneration in fp32 with
tie_word_embeddings=True and Qwen2.5-VL-3B's attention layout (16 query heads over 2 K/V heads of 128, so 8 query heads per K/V head)
at two layers (committed with this script). The tied weights (tests/qwen_tied.py) are regenerated from their seed by the tests and pinned
by a checksum; the inputs are stored. Two input sets, each scored four ways as the reference does:
  * images: 4 prompts over 2 still images of 84x56 pixels (grid 1x6x4), ragged text
  * video:  3 prompts, each its own 2-temporal-patch frame stack of 56x84 (grid 2x4x6), second_per_grid 2.0
and per set:
  * score: fp32 last-position logits, softmax(logits)[answer], and the same after RepetitionPenaltyLogitsProcessor(1.3) and T = 0.5
  * trace: top-5 ids and probabilities of softmax(logits) (forward_with_trace)
  * generate: 8 greedy tokens of generate(do_sample=False, repetition_penalty=1.3) and the top-1 / top-2 margin of every step
  * rollout: generate(max_new_tokens=4, output_scores=True), p[s, j] = softmax(scores[s])[answer j] (forward(max_new_tokens=4))

  python tools/make_golden_qwen_3b.py
"""
import dataclasses
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor

from oracle import qwen25vl_oracle as qo
from qwen_tied import TINY_GQA8, build_hf_qwen_tied, sd_checksum, tied_state_dict

GOLD = os.path.join(ROOT, "tests", "golden")
GEN_NEW, GEN_PENALTY = 8, 1.3
ROLL_NEW = 4
ROLL_ANSWERS = {"images": [[11, 250], [42], [5, 7, 9], [300]], "video": [[11], [42, 7], [5]]}


def hf_kwargs(cfg, inp, b, spg):
    t, gh, gw = inp["grid_thw"][0]
    P = t * gh * gw
    img = inp["image_of_sample"][b] if inp["image_of_sample"] is not None else b
    ids = inp["input_ids"][b]
    px = inp["pixel_patches"][img * P:(img + 1) * P]
    grid = torch.tensor([list(inp["grid_thw"][img])])
    kw = dict(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long))
    if t > 1:
        kw.update(pixel_values_videos=px, video_grid_thw=grid, second_per_grid_ts=torch.tensor([spg[img]]),
                  mm_token_type_ids=torch.where(ids == cfg.video_token_id, 2, 0)[None])
    else:
        kw.update(pixel_values=px, image_grid_thw=grid, mm_token_type_ids=(ids == cfg.image_token_id).long()[None])
    return kw


@torch.no_grad()
def hf_set(m, cfg, inp, spg, answers):
    logits = torch.stack([m(**hf_kwargs(cfg, inp, b, spg)).logits[0, -1].float() for b in range(len(inp["input_ids"]))])
    ans = torch.tensor(inp["answer_ids"])
    probs = torch.softmax(logits, -1)
    proc = RepetitionPenaltyLogitsProcessor(1.3)
    pen = torch.stack([torch.softmax(proc(ids[None], logits[b][None].clone())[0] / 0.5, -1)[ans[b]] for b, ids in enumerate(inp["input_ids"])])
    top = torch.topk(probs, 5, dim=-1)
    out = dict(logits=logits, probs=probs[torch.arange(len(ans)), ans], probs_penalty_1p3_T_0p5=pen, top5_ids=top.indices.to(torch.int32),
               top5_probs=top.values, gen_ids=[], gen_margins=[], roll_ids=[], roll_p=[])
    for b in range(len(inp["input_ids"])):
        g = m.generate(**hf_kwargs(cfg, inp, b, spg), max_new_tokens=GEN_NEW, do_sample=False, repetition_penalty=GEN_PENALTY,
                       eos_token_id=None, pad_token_id=0, output_scores=True, return_dict_in_generate=True)
        top2 = torch.stack([s[0].float().topk(2).values for s in g.scores])
        out["gen_ids"].append(g.sequences[0, len(inp["input_ids"][b]):].tolist())
        out["gen_margins"].append((top2[:, 0] - top2[:, 1]).clone())
        r = m.generate(**hf_kwargs(cfg, inp, b, spg), max_new_tokens=ROLL_NEW, do_sample=False, temperature=1.0, eos_token_id=None,
                       pad_token_id=0, output_scores=True, return_dict_in_generate=True)
        sc = torch.stack([s[0].float() for s in r.scores])
        out["roll_ids"].append(r.sequences[0, len(inp["input_ids"][b]):].tolist())
        out["roll_p"].append(torch.softmax(sc, -1)[:, answers[b]].clone())
    return out


def main():
    cfg = qo.Qwen25VLConfig.tiny(**TINY_GQA8)
    sd = tied_state_dict(cfg, seed=0)
    m = build_hf_qwen_tied(cfg, sd)
    blob = dict(config=dataclasses.asdict(cfg), weights_seed=0, weights_sha256=sd_checksum(sd), gen_new_tokens=GEN_NEW,
                gen_penalty=GEN_PENALTY, rollout_new_tokens=ROLL_NEW, cases={})
    img = qo.make_synthetic_inputs(cfg, 4, (84, 56), 12, seed=1, ragged=True, n_images=2)
    img["answer_ids"][0] = int(img["input_ids"][0][-1])       # an answer id in its own prompt: the penalty moves the label logit too
    vid = qo.make_synthetic_inputs(cfg, 3, (56, 84), 10, seed=2, ragged=True, frames=2)
    for name, inp, spg in (("images", img, None), ("video", vid, [2.0, 2.0, 2.0])):
        blob["cases"][name] = dict(inputs=inp, second_per_grid_ts=spg, rollout_answers=ROLL_ANSWERS[name],
                                   hf=hf_set(m, cfg, inp, spg, ROLL_ANSWERS[name]))
    path = os.path.join(GOLD, "qwen_tied_gqa8_tiny.pt")
    torch.save(blob, path)
    for name, c in blob["cases"].items():
        h = c["hf"]
        print(name, "probs", [round(float(x), 5) for x in h["probs"]], "gen", h["gen_ids"],
              "min margins", [round(float(x.min()), 4) for x in h["gen_margins"]])
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

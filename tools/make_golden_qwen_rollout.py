"""Generate tests/golden/qwen_rollout_tiny.pt from the REAL transformers Qwen2_5_VLForConditionalGeneration.generate(do_sample=False,
output_scores=True) in fp32 (committed with this script): what the reference's Qwen2VLModel.forward / forward_with_trace read for
max_new_tokens > 1 (qwen2vl_model.py:160-167, :223-231). The tiny config, seeded weights and the "images" inputs of
tools/make_golden_qwen_generate.py (3 prompts over 2 images, ragged text; regenerated from their seeds by the tests and pinned by a
checksum). Cases:
  * pen1.0:      repetition penalty 1.0, temperature 1.0, no EOS
  * pen1.3_T0.7: repetition penalty 1.3, temperature 0.7, no EOS
  * eos:         penalty 1.0, temperature 1.3, EOS ids = {a token prompt 2 emits mid-way without EOS, an id never emitted}
Each case stores, per prompt: HF's generated ids, answer ids, p [L, n] = softmax(scores[s] / T)[answer id], the top-5 ids and
probabilities [L, 5] of softmax(scores[s] / T), and the fp32 margin between the top two processed scores of each step.

  python tools/make_golden_qwen_rollout.py
"""
import dataclasses
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch

from oracle import qwen25vl_oracle as qo
from test_qwen_host import hf_model, TINY
from make_golden_qwen import sd_checksum
from make_golden_qwen_generate import CASES, case_inputs, inputs_checksum

GOLD = os.path.join(ROOT, "tests", "golden")
MAX_NEW = 12
ANSWERS = [[11, 250, 3], [42, 7], [5]]      # one, two and three-token answers


@torch.no_grad()
def hf_rollout(m, cfg, inp, max_new, penalty, temperature, eos_ids, answers):
    """generate(do_sample=False, output_scores=True) per prompt, as the reference runs it. Returns per prompt (ids, p, top5 ids, top5
    probabilities, margins)."""
    t, gh, gw = inp["grid_thw"][0]
    P = t * gh * gw
    out = dict(ids=[], p=[], top5_ids=[], top5_probs=[], margins=[])
    for b, ids in enumerate(inp["input_ids"]):
        img = inp["image_of_sample"][b] if inp["image_of_sample"] is not None else b
        o = m.generate(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long), pixel_values=inp["pixel_patches"][img * P:(img + 1) * P],
                       image_grid_thw=torch.tensor([list(inp["grid_thw"][img])]), mm_token_type_ids=(ids == cfg.image_token_id).long()[None],
                       max_new_tokens=max_new, do_sample=False, temperature=1.0, repetition_penalty=penalty, eos_token_id=list(eos_ids) or None,
                       pad_token_id=0, output_scores=True, return_dict_in_generate=True)
        scores = torch.stack([s[0].float() for s in o.scores])
        probs = torch.softmax(scores / temperature, dim=-1)
        top = torch.topk(probs, 5, dim=-1)
        top2 = scores.topk(2, dim=-1).values
        out["ids"].append(o.sequences[0, len(ids):].tolist())
        out["p"].append(probs[:, answers[b]].clone())
        out["top5_ids"].append(top.indices.to(torch.int32).clone())
        out["top5_probs"].append(top.values.clone())
        out["margins"].append((top2[:, 0] - top2[:, 1]).clone())
    return out


def main():
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m = hf_model(cfg)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    blob = dict(config=dataclasses.asdict(cfg), weights_seed=0, weights_sha256=sd_checksum(sd), max_new_tokens=MAX_NEW, cases={})
    spec = CASES["images"]
    inp = case_inputs(cfg, spec)
    common = dict(inputs=spec, inputs_sha256=inputs_checksum(inp), answer_ids=ANSWERS)
    for name, pen, temp in (("pen1.0", 1.0, 1.0), ("pen1.3_T0.7", 1.3, 0.7)):
        r = hf_rollout(m, cfg, inp, MAX_NEW, pen, temp, (), ANSWERS)
        blob["cases"][name] = dict(common, penalty=pen, temperature=temp, eos_ids=[], **r)
    base = blob["cases"]["pen1.0"]["ids"]
    stop = base[2][4]
    never = next(t for t in range(cfg.vocab) if all(t not in x for x in base))
    r = hf_rollout(m, cfg, inp, MAX_NEW, 1.0, 1.3, (stop, never), ANSWERS)
    assert len(r["ids"][2]) < MAX_NEW and r["ids"][2][-1] == stop
    blob["cases"]["eos"] = dict(common, penalty=1.0, temperature=1.3, eos_ids=[stop, never], **r)
    path = os.path.join(GOLD, "qwen_rollout_tiny.pt")
    torch.save(blob, path)
    for name, c in blob["cases"].items():
        print(name, c["ids"], "min margin", [round(float(x.min()), 4) for x in c["margins"]])
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

"""Generate tests/golden/clipt5_generate_tiny.pt from the REAL transformers T5ForConditionalGeneration.generate(inputs_embeds=<spliced
prompt>, attention_mask=<its mask>, do_sample=False, num_beams=1) in fp32 (committed with this script). The tiny CLIP-FlanT5 config and
seeded weights of oracle/clipt5_oracle.py (checked against a stored checksum); the inputs -- 3 ragged prompts over 2 images, the first
image shared by prompts 0 and 2 -- are regenerated from their seed by the tests (make_synthetic_inputs) and pinned by a checksum, so the
file holds ids and margins only. Cases:
  * free: no EOS ids, every prompt runs to max_new_tokens
  * eos:  EOS ids = {a token prompt 1 emits mid-way in the free run, an id never emitted}: prompt 1 stops on it, the others run on
Each entry stores HF's generated ids per prompt and, per step, the fp32 margin between the top two scores (output_scores).

  python tools/make_golden_clipt5_generate.py
"""
import copy
import dataclasses
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from oracle import clipt5_oracle as orc
from oracle import clipt5_generate as cg
from oracle.hf_reference import build_hf_modules

GOLD = os.path.join(ROOT, "tests", "golden")
MAX_NEW = 16
WEIGHTS_SEED = 0
INPUTS = dict(batch=3, text_len=14, seed=3, ragged=True, n_images=2)


def case_inputs(cfg, spec=INPUTS):
    return orc.make_synthetic_inputs(cfg, spec["batch"], spec["text_len"], seed=spec["seed"], ragged=spec["ragged"], n_images=spec["n_images"])


def inputs_checksum(inp):
    h = hashlib.sha256()
    for k in ("pixels", "input_ids", "text_lens", "image_index"):
        h.update(inp[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def hf_t5(cfg, sd):
    """The fp32 transformers T5ForConditionalGeneration carrying `sd` (the vision tower and projector are the oracle's)."""
    _, _, t5 = build_hf_modules(cfg, {k: v.float() for k, v in sd.items()})
    return t5


@torch.no_grad()
def hf_generate(t5, embeds, mask, max_new, eos_ids):
    """generate(do_sample=False, num_beams=1) over the batch. Returns (ids, margins) per prompt: the generated ids up to and including
    the first EOS id, and the top-1 / top-2 margin of HF's scores at each of those steps."""
    gc = copy.deepcopy(t5.generation_config)
    gc.eos_token_id = list(eos_ids) or None
    gc.max_new_tokens, gc.max_length, gc.min_length = max_new, None, 0
    gc.do_sample, gc.num_beams = False, 1
    gc.output_scores, gc.return_dict_in_generate = True, True
    out = t5.generate(inputs_embeds=embeds, attention_mask=mask.long(), generation_config=gc)
    seq = out.sequences[:, 1:]                                  # drop decoder_start_id
    top2 = torch.stack([s.float().topk(2, dim=-1).values for s in out.scores], dim=1)      # [B, steps, 2]
    ids, margins = [], []
    for b in range(seq.shape[0]):
        row = seq[b].tolist()
        n = next((i + 1 for i, t in enumerate(row) if t in eos_ids), len(row))
        ids.append(row[:n])
        margins.append((top2[b, :n, 0] - top2[b, :n, 1]).clone())
    return ids, margins


def main():
    cfg = orc.ClipT5Config.tiny()
    sd = orc.make_synthetic_state_dict(cfg, seed=WEIGHTS_SEED)
    t5 = hf_t5(cfg, sd)
    inp = case_inputs(cfg)
    embeds, mask, _ = cg.encode_prompts(sd, cfg, inp["pixels"], inp["input_ids"], inp["text_lens"], inp["image_index"])
    blob = dict(config=dataclasses.asdict(cfg), weights_seed=WEIGHTS_SEED, weights_sha256=orc.state_dict_sha256(sd), max_new_tokens=MAX_NEW,
                inputs=INPUTS, inputs_sha256=inputs_checksum(inp), cases={})
    ids, margins = hf_generate(t5, embeds, mask, MAX_NEW, [])
    blob["cases"]["free"] = dict(eos_ids=[], ids=ids, margins=margins)
    stop = ids[1][5]
    never = next(t for t in range(cfg.vocab) if all(t not in x for x in ids))
    eos_ids, eos_margins = hf_generate(t5, embeds, mask, MAX_NEW, [stop, never])
    assert len(eos_ids[1]) < MAX_NEW and eos_ids[1][-1] == stop
    blob["cases"]["eos"] = dict(eos_ids=[stop, never], ids=eos_ids, margins=eos_margins)
    path = os.path.join(GOLD, "clipt5_generate_tiny.pt")
    torch.save(blob, path)
    for name, c in blob["cases"].items():
        print(name, c["ids"], "min margin", [round(float(x.min()), 4) for x in c["margins"]])
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()

"""Host restatement of CLIP-FlanT5 sampled generation for the tests: a sampled decode of the tiny model on top of
oracle/clipt5_generate.py's decoder logits, with the token drawn by tests/sample_ref.py's fp64 warpers and Gumbel-max draw."""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch

from sample_ref import draw, warp_row


@torch.no_grad()
def clipt5_sample(sd, cfg, pixels, input_ids: torch.Tensor, text_lens: torch.Tensor, max_new_tokens: int, seeds: Sequence[int],
                  temperature: float, top_k: int, top_p: float, eos_ids: Sequence[int] = (), image_index=None, mode: str = "fp32"):
    """T5 generate(do_sample=True) of each prompt on its own, as oracle/clipt5_generate.clipt5_generate decodes greedily (the decoder rerun
    over [start] + the tokens so far, its last-row fp32 logits; in mode "bf16" those are the bf16-rounded lm_head output the engine
    draws from), with the token drawn by warp_row / draw under seeds[b] at step t. No repetition penalty (FlanT5's generation config has
    none). Returns dict(tokens, margins: per step the draw's gap, boundary: per step the distance of the nearest kept-set boundary mass
    from 1 - top_p)."""
    from oracle.clipt5_generate import encode_prompts
    from oracle.clipt5_oracle import t5_decoder_logits
    _, mask, enc = encode_prompts(sd, cfg, pixels, input_ids, text_lens, image_index, mode)
    eos = set(int(e) for e in eos_ids)
    out = dict(tokens=[], margins=[], boundary=[])
    for b in range(input_ids.shape[0]):
        gen, margins, bounds = [], [], []
        for t in range(max_new_tokens):
            labels = torch.tensor([gen + [0]], dtype=torch.long)          # shift_right feeds [start] + gen; the last label is unused
            s = t5_decoder_logits(sd, enc[b:b + 1], mask[b:b + 1], labels, cfg, mode)[0, -1].float().numpy().astype(np.float32)
            if temperature != 1.0:
                s = (s / np.float32(temperature)).astype(np.float32)
            s = np.where(s == 0, np.float32(0), s).astype(np.float32)
            kept, cum, thr = warp_row(s, top_k, top_p)
            tok, gap = draw(s, kept, int(seeds[b]), t)
            fin = np.isfinite(cum)
            bounds.append(float(np.abs(cum[fin] - thr).min()) if top_p < 1.0 else np.inf)
            margins.append(gap)
            gen.append(tok)
            if tok in eos:
                break
        out["tokens"].append(gen)
        out["margins"].append(margins)
        out["boundary"].append(bounds)
    return out

"""CPU oracle for CLIP-FlanT5 greedy generation -- TEST INFRASTRUCTURE, NOT THE PRODUCT.

Plain-PyTorch restatement (fp32 or bf16-rounding-emulating) of HF `T5ForConditionalGeneration.generate(inputs_embeds=<spliced prompt>,
attention_mask=<its mask>, do_sample=False, num_beams=1)` on top of oracle/clipt5_oracle.py: the vision tower, projector, splice and
encoder of the scoring oracle, then greedy search from decoder_start_id. The decoder is causal, so the logits of step t are those of
`t5_decoder_logits` over the tokens generated so far (recomputed over the whole prefix instead of kept in a K/V cache). No logits
processors. Pinned against the real `generate` in tests/test_clipt5_generate_host.py.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from .clipt5_oracle import ClipT5Config, clip_vision_features, mm_projector, splice_multimodal, t5_decoder_logits, t5_encoder


@torch.no_grad()
def encode_prompts(sd: Dict[str, torch.Tensor], cfg: ClipT5Config, pixels: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor,
                   image_index: Optional[torch.Tensor] = None, mode: str = "fp32"):
    """Spliced embeddings [B, S, D], their mask [B, S] and the encoder output [B, S, D] of a padded prompt batch (as clipt5_score)."""
    feats = clip_vision_features(sd, pixels, cfg, mode)
    proj = mm_projector(sd, feats, mode)
    embeds, mask = splice_multimodal(sd, input_ids, text_lens, proj, image_index, mode)
    return embeds, mask, t5_encoder(sd, embeds, mask, cfg, mode)


@torch.no_grad()
def clipt5_generate(sd: Dict[str, torch.Tensor], cfg: ClipT5Config, pixels: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor,
                    max_new_tokens: int, eos_ids: Sequence[int] = (), image_index: Optional[torch.Tensor] = None, mode: str = "fp32",
                    forced: Optional[List[List[int]]] = None):
    """Greedy decoding of each prompt of the batch: the scores of step t are the fp32-cast last-row logits of the decoder run over
    [start] + the t tokens chosen before; the token is their arg-max (lowest id on ties); a sample stops after an EOS id or
    max_new_tokens tokens. With `forced` (one token list per sample) the given tokens are fed instead of the arg-max (teacher forcing).
    Returns dict(tokens: List[List[int]], scores: List[Tensor [steps, vocab]] the fp32 scores of every step)."""
    _, mask, enc = encode_prompts(sd, cfg, pixels, input_ids, text_lens, image_index, mode)
    eos = set(int(e) for e in eos_ids)
    out_tokens, out_scores = [], []
    for b in range(input_ids.shape[0]):
        gen, scores = [], []
        n_steps = max_new_tokens if forced is None else min(max_new_tokens, len(forced[b]))
        for t in range(n_steps):
            labels = torch.tensor([gen + [0]], dtype=torch.long)          # shift_right feeds [start] + gen; the last label is unused
            s = t5_decoder_logits(sd, enc[b:b + 1], mask[b:b + 1], labels, cfg, mode)[0, -1].float()
            scores.append(s)
            tok = int(torch.argmax(s)) if forced is None else int(forced[b][t])
            gen.append(tok)
            if forced is None and tok in eos:
                break
        out_tokens.append(gen)
        out_scores.append(torch.stack(scores))
    return dict(tokens=out_tokens, scores=out_scores)

"""CPU oracle for Qwen2.5-VL greedy generation -- TEST INFRASTRUCTURE, NOT THE PRODUCT.

Plain-PyTorch restatement (fp32 or bf16-rounding-emulating) of what the reference's Qwen2VLModel.generate runs
(t2v_metrics/models/vqascore_models/qwen2vl_model.py:495-563: per sample, `generate(**inputs, max_new_tokens=N, do_sample=False)`)
on top of transformers 5.5.0: the prefill of oracle/qwen25vl_oracle.py into a K/V cache, then one position at a time
(modeling_qwen2_5_vl.py:1576-1612 _prepare_position_ids_for_generation), greedy search with the repetition-penalty processor
(generation/utils.py). Pinned against the real `Qwen2_5_VLForConditionalGeneration.generate` in tests/test_qwen_generate_host.py.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from .clipt5_oracle import _Num
from .qwen25vl_oracle import Qwen25VLConfig, mrope_position_ids, rms_norm, rotate_half, vision_tower


def text_step_cached(sd, embeds: torch.Tensor, position_ids: torch.Tensor, cfg: Qwen25VLConfig, cache: List[list], mode="fp32",
                     prefix="model.language_model.") -> torch.Tensor:
    """text_last_logits over `n` new rows that follow the rows already in `cache` (one [k, v] pair per layer, post-rope, as HF's
    DynamicCache holds them; empty list = prefill). Appends the new rows' K/V to the cache. Returns the fp32 logits of the last new row."""
    num = _Num(mode)
    g = lambda k: sd[prefix + k].float()
    n = embeds.shape[0]
    Hq, Hkv, hd = cfg.heads, cfg.kv_heads, cfg.head_dim
    inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float) / hd))
    freqs = position_ids[:, :, None].float() * inv_freq[None, None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    cos3, sin3 = num.r(emb.cos()), num.r(emb.sin())
    sec = list(cfg.mrope_section) * 2
    cos = torch.cat([m[i % 3] for i, m in enumerate(cos3.split(sec, dim=-1))], dim=-1)[:, None, :]
    sin = torch.cat([m[i % 3] for i, m in enumerate(sin3.split(sec, dim=-1))], dim=-1)[:, None, :]
    past = cache[0][0].shape[0] if cache else 0
    allowed = torch.arange(past + n)[None, :] <= (past + torch.arange(n))[:, None]
    neg = torch.finfo(torch.bfloat16 if num.bf16 else torch.float32).min
    x = embeds
    for l in range(cfg.layers):
        p = f"layers.{l}."
        y = rms_norm(x, g(p + "input_layernorm.weight"), cfg.rms_eps, num)
        q = num.linear(y, g(p + "self_attn.q_proj.weight"), g(p + "self_attn.q_proj.bias")).view(n, Hq, hd)
        k = num.linear(y, g(p + "self_attn.k_proj.weight"), g(p + "self_attn.k_proj.bias")).view(n, Hkv, hd)
        v = num.linear(y, g(p + "self_attn.v_proj.weight"), g(p + "self_attn.v_proj.bias")).view(n, Hkv, hd)
        q = num.r(q * cos + rotate_half(q) * sin)
        k = num.r(k * cos + rotate_half(k) * sin)
        if len(cache) <= l:
            cache.append([k, v])
        else:
            cache[l] = [torch.cat([cache[l][0], k]), torch.cat([cache[l][1], v])]
        k, v = cache[l]
        rep = Hq // Hkv
        kk = k.repeat_interleave(rep, dim=1).transpose(0, 1)
        vv = v.repeat_interleave(rep, dim=1).transpose(0, 1)
        att = num.r(torch.matmul(q.transpose(0, 1), kk.transpose(1, 2)) * hd ** -0.5)
        att = num.r(att + torch.where(allowed, 0.0, neg)[None])
        att = num.r(torch.softmax(att.float(), dim=-1))
        o = num.r(torch.matmul(att, vv)).transpose(0, 1).reshape(n, Hq * hd)
        x = num.r(x + num.linear(o, g(p + "self_attn.o_proj.weight")))
        y = rms_norm(x, g(p + "post_attention_layernorm.weight"), cfg.rms_eps, num)
        gate = num.linear(y, g(p + "mlp.gate_proj.weight"))
        up = num.linear(y, g(p + "mlp.up_proj.weight"))
        x = num.r(x + num.linear(num.r(num.r(F.silu(gate)) * up), g(p + "mlp.down_proj.weight")))
    h = rms_norm(x[-1:], g("norm.weight"), cfg.rms_eps, num)
    return num.linear(h, sd["lm_head.weight"])[0].float()


def process_logits(logits: torch.Tensor, seen_ids: torch.Tensor, repetition_penalty: float = 1.0) -> torch.Tensor:
    """The fp32 scores greedy decoding arg-maxes: RepetitionPenaltyLogitsProcessor over every id seen so far (prompt + generated)."""
    s = logits.float().clone()
    if repetition_penalty != 1.0:
        idx = torch.unique(seen_ids)
        v = s[idx]
        s[idx] = torch.where(v < 0, v * repetition_penalty, v / repetition_penalty)
    return s


@torch.no_grad()
def qwen25vl_generate(sd: Dict[str, torch.Tensor], cfg: Qwen25VLConfig, pixel_patches: torch.Tensor, grid_thw: Sequence[Sequence[int]],
                      input_ids: List[torch.Tensor], max_new_tokens: int, eos_ids: Sequence[int] = (), image_of_sample=None, mode: str = "fp32",
                      repetition_penalty: float = 1.0, second_per_grid_ts: Optional[Sequence[float]] = None, forced: Optional[List[List[int]]] = None):
    """HF generate(do_sample=False) for each sample on its own: prefill into a K/V cache, then one position at a time. Generated token t
    sits at (position of the last prompt token) + 1 + t on all three mRoPE axes (generate advances the prompt's last position ids by one
    per step; with a vision run whose temporal index exceeds the text positions this is below max(prompt positions) + 1); the scores are the bf16 (or fp32) last-row logits in fp32 after the
    repetition penalty over prompt + generated ids; the token is their arg-max (lowest id on ties); a sample stops after an EOS id or
    max_new_tokens tokens. With `forced` (one token list per sample) the given tokens are fed instead of the arg-max (teacher forcing).
    Returns dict(tokens: List[List[int]], scores: List[Tensor [steps, vocab]] the processed fp32 scores of every step)."""
    num = _Num(mode)
    feats = vision_tower(sd, pixel_patches, grid_thw, cfg, mode)
    unit = cfg.spatial_merge_size ** 2
    offs = [0]
    for t, h, w in grid_thw:
        offs.append(offs[-1] + t * h * w // unit)
    embed_w = num.r(sd["model.language_model.embed_tokens.weight"].float())
    eos = set(int(e) for e in eos_ids)
    out_tokens, out_scores = [], []
    for b, ids in enumerate(input_ids):
        img = image_of_sample[b] if image_of_sample is not None else b
        e = embed_w[ids].clone()
        mask = (ids == cfg.image_token_id) | (ids == cfg.video_token_id)
        e[mask] = num.r(feats[offs[img]:offs[img + 1]])
        pos = mrope_position_ids(ids, [grid_thw[img]], cfg, None if second_per_grid_ts is None else [second_per_grid_ts[img]])
        assert bool((pos[:, -1] == pos[0, -1]).all()), "the prompt must end with a text token"
        first = int(pos[0, -1]) + 1
        cache: List[list] = []
        logits = text_step_cached(sd, e, pos, cfg, cache, mode)
        gen, scores = [], []
        n_steps = max_new_tokens if forced is None else min(max_new_tokens, len(forced[b]))
        for t in range(n_steps):
            s = process_logits(logits, torch.cat([ids.long(), torch.tensor(gen, dtype=torch.long)]), repetition_penalty)
            scores.append(s)
            tok = int(torch.argmax(s)) if forced is None else int(forced[b][t])
            gen.append(tok)
            if (forced is None and tok in eos) or t + 1 == n_steps:
                break
            logits = text_step_cached(sd, embed_w[tok][None], torch.full((3, 1), first + t, dtype=torch.long), cfg, cache, mode)
        out_tokens.append(gen)
        out_scores.append(torch.stack(scores))
    return dict(tokens=out_tokens, scores=out_scores)

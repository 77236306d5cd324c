"""Host restatement of the sampled token selection (sample_select_kernel) for the tests: HF's processors for generate(do_sample=True) in
fp64 on the kernel's fp32 processed scores, the documented tie rule at the top-p cut, Philox4x32-10 in numpy and the Gumbel-max draw,
and a sampled cached decode of the tiny model on top of oracle/qwen25vl_generate.py's language-model step."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

PHILOX_M0, PHILOX_M1, PHILOX_W0, PHILOX_W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox4x32_10(ctr: np.ndarray, key: Sequence[int]) -> np.ndarray:
    """Philox4x32-10 of counters ctr uint32 [..., 4] under key (k0, k1) -> uint32 [..., 4] (Random123's philox4x32 with 10 rounds)."""
    c = [ctr[..., i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0] & 0xFFFFFFFF), np.uint64(key[1] & 0xFFFFFFFF)
    mask = np.uint64(0xFFFFFFFF)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(PHILOX_W0)) & mask, (k1 + np.uint64(PHILOX_W1)) & mask
        p0, p1 = np.uint64(PHILOX_M0) * c[0], np.uint64(PHILOX_M1) * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & mask, p1 >> np.uint64(32), p1 & mask
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, -1).astype(np.uint32)


def gumbel(seed: int, step: int, V: int) -> np.ndarray:
    """g_n = -log(-log u_n) in fp64 for ids n < V: u_n = ((bits >> 8) + 0.5) 2^-24 from lane n & 3 of Philox4x32-10, key = the 64-bit seed
    (low word first), counter (n >> 2, step, 0, 0). Every u is exact in fp64."""
    G = (V + 3) // 4
    ctr = np.zeros((G, 4), dtype=np.uint32)
    ctr[:, 0] = np.arange(G, dtype=np.uint32)
    ctr[:, 1] = step
    bits = philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)).reshape(-1)[:V]
    u = ((bits >> 8).astype(np.float64) + 0.5) * 2.0 ** -24
    return -np.log(-np.log(u))


def processed_scores(logits_bf16: torch.Tensor, bitmap: Optional[torch.Tensor], penalty: float, temperature: float) -> np.ndarray:
    """The kernel's fp32 scores [B, V]: bf16 -> fp32 -> repetition penalty on the bitmap's ids -> / temperature (IEEE fp32, none at 1),
    -0 as +0, saturated to [-FLT_MAX, FLT_MAX] with NaN at -FLT_MAX. numpy's float32 operations round as the kernel's do, so these are
    the kernel's values bit for bit."""
    x = logits_bf16.float().cpu().numpy().astype(np.float32)
    if bitmap is not None and penalty != 1.0:
        V = x.shape[1]
        words = bitmap.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        ids = np.arange(V)
        hit = ((words[:, ids // 32] >> (ids % 32)) & 1).astype(bool)
        pen = np.float32(penalty)
        x = np.where(hit, np.where(x < 0, x * pen, x / pen), x).astype(np.float32)
    if temperature != 1.0:
        with np.errstate(over="ignore"):
            x = (x / np.float32(temperature)).astype(np.float32)
    # the kernel saturates an overflowing score (and a NaN, to the bottom), where HF's softmax would give NaN
    fmax = np.finfo(np.float32).max
    x = np.where(np.isnan(x), -fmax, np.clip(x, -fmax, fmax)).astype(np.float32)
    return np.where(x == 0, np.float32(0), x).astype(np.float32)


def warp_row(x: np.ndarray, top_k: int, top_p: float):
    """HF's TopK then TopP warpers on one row of fp32 scores, restated in fp64 with the documented tie rule (ascending (score, id): lower
    ids of the group at the cut go first). Returns (kept bool [V], cum float64 [V]: each kept-by-top-k id's cumulative probability in
    that ascending order (inf for ids top-k removed), fp32(1 - top_p) as HF compares against it)."""
    V = x.shape[0]
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        kth = np.sort(x)[::-1][top_k - 1]
        keep = x >= kth
    xd = x.astype(np.float64)
    p = np.where(keep, np.exp(xd - xd[keep].max()), 0.0)
    p /= p.sum()
    order = np.lexsort((np.arange(V), xd))       # ascending score, then ascending id
    cum = np.full(V, np.inf)
    cum[order] = np.cumsum(p[order])
    cum[~keep] = np.inf
    thr = float(np.float32(1.0 - top_p))
    kept = keep.copy()
    if top_p < 1.0:
        kept &= ~(cum <= thr)
        kept[order[-1]] = True
    return kept, cum, thr


def draw(x: np.ndarray, kept: np.ndarray, seed: int, step: int):
    """The Gumbel-max draw over the kept ids in fp64 -> (token, gap between the best and second-best perturbed scores)."""
    xd = x.astype(np.float64)
    v = np.where(kept, (xd - xd.max()) + gumbel(seed, step, x.shape[0]), -np.inf)
    top2 = np.sort(v)[-2:] if kept.sum() > 1 else np.array([-np.inf, v.max()])
    return int(np.argmax(v)), float(top2[1] - top2[0])


@torch.no_grad()
def qwen25vl_sample(sd, cfg, pixel_patches, grid_thw, input_ids: List[torch.Tensor], max_new_tokens: int, seeds: Sequence[int],
                    temperature: float, top_k: int, top_p: float, eos_ids: Sequence[int] = (), image_of_sample=None, mode: str = "fp32",
                    repetition_penalty: float = 1.0, second_per_grid_ts=None):
    """generate(do_sample=True) of each sample on its own, as oracle/qwen25vl_generate.qwen25vl_generate decodes greedily, with the
    token drawn by warp_row / draw under seeds[b] at step t. The scores are the last-row logits rounded to bf16 (the engine's lm_head
    output) in mode "bf16", fp32 otherwise. Returns dict(tokens, margins: per step the draw's gap, boundary: per step the distance of
    the nearest kept-set boundary mass from 1 - top_p)."""
    from oracle.qwen25vl_generate import process_logits, text_step_cached
    from oracle.qwen25vl_oracle import mrope_position_ids, vision_tower
    from oracle.clipt5_oracle import _Num
    num = _Num(mode)
    feats = vision_tower(sd, pixel_patches, grid_thw, cfg, mode)
    unit = cfg.spatial_merge_size ** 2
    offs = [0]
    for t, h, w in grid_thw:
        offs.append(offs[-1] + t * h * w // unit)
    embed_w = num.r(sd["model.language_model.embed_tokens.weight"].float())
    eos = set(int(e) for e in eos_ids)
    out = dict(tokens=[], margins=[], boundary=[])
    for b, ids in enumerate(input_ids):
        img = image_of_sample[b] if image_of_sample is not None else b
        e = embed_w[ids].clone()
        mask = (ids == cfg.image_token_id) | (ids == cfg.video_token_id)
        e[mask] = num.r(feats[offs[img]:offs[img + 1]])
        pos = mrope_position_ids(ids, [grid_thw[img]], cfg, None if second_per_grid_ts is None else [second_per_grid_ts[img]])
        first = int(pos[0, -1]) + 1
        cache: list = []
        logits = text_step_cached(sd, e, pos, cfg, cache, mode)
        gen, margins, bounds = [], [], []
        for t in range(max_new_tokens):
            s = process_logits(logits, torch.cat([ids.long(), torch.tensor(gen, dtype=torch.long)]), repetition_penalty).numpy()
            if temperature != 1.0:
                s = (s.astype(np.float32) / np.float32(temperature)).astype(np.float32)
            s = np.where(s == 0, np.float32(0), s).astype(np.float32)
            kept, cum, thr = warp_row(s, top_k, top_p)
            tok, gap = draw(s, kept, int(seeds[b]), t)
            fin = np.isfinite(cum)
            bounds.append(float(np.abs(cum[fin] - thr).min()) if top_p < 1.0 else np.inf)
            margins.append(gap)
            gen.append(tok)
            if tok in eos or t + 1 == max_new_tokens:
                break
            logits = text_step_cached(sd, embed_w[tok][None], torch.full((3, 1), first + t, dtype=torch.long), cfg, cache, mode)
        out["tokens"].append(gen)
        out["margins"].append(margins)
        out["boundary"].append(bounds)
    return out

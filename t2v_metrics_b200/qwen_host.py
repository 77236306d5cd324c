"""Host-side index logic of the Qwen2.5-VL path (pure integer work, cached per grid shape by the engine).

Mirrors, bit for bit, what the reference computes in Python inside transformers before any kernel runs:
  * rot_pos_emb            modeling_qwen2_5_vl.py:382-409  -> (h, w) index of every patch, merge-block order
  * get_window_index       :411-451                         -> window order of 2x2 patch groups + cumulative window lengths
  * get_rope_index         :1024-1133 (+ get_vision_position_ids :981-1022) -> (t, h, w) mRoPE position ids
  * rotary frequency tables :119-131 (vision), :568-585 (text), mrope sections :650-662
tests/test_qwen_host.py checks every function against the transformers implementation.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F


def vision_rot_pos_ids(grid_thw: Sequence[Sequence[int]], merge: int) -> torch.Tensor:
    out = []
    for t, h, w in grid_thw:
        hp = torch.arange(h).unsqueeze(1).expand(-1, w).reshape(h // merge, merge, w // merge, merge).permute(0, 2, 1, 3).flatten()
        wp = torch.arange(w).unsqueeze(0).expand(h, -1).reshape(h // merge, merge, w // merge, merge).permute(0, 2, 1, 3).flatten()
        out.append(torch.stack([hp, wp], dim=-1).repeat(t, 1))
    return torch.cat(out, dim=0)


def vision_window_index(grid_thw: Sequence[Sequence[int]], merge: int, window_size: int, patch_size: int):
    """Returns (window_index [n_groups], cu_window_seqlens (patches, duplicates removed), cu_frame_seqlens).

    This is a TRANSCRIPTION of `Qwen2_5_VisionTransformerPretrainedModel.get_window_index` (transformers 5.5.0
    models/qwen2_5_vl/modeling_qwen2_5_vl.py:411-451) -- same `F.pad(..., -100)`, same reshape / permute chain -- because the index arrays
    must match the installed transformers bit for bit (tested as such in tests/test_qwen_host.py); `vision_rot_pos_ids` above likewise
    follows `rot_pos_emb` (:382-409). Third-party index logic, not reference code."""
    unit = merge * merge
    vw = window_size // merge // patch_size
    window_index, cu_win, base = [], [0], 0
    for t, h, w in grid_thw:
        gh, gw = h // merge, w // merge
        index = torch.arange(t * gh * gw).reshape(t, gh, gw)
        pad_h, pad_w = vw - gh % vw, vw - gw % vw
        nh, nw = (gh + pad_h) // vw, (gw + pad_w) // vw
        padded = F.pad(index, (0, pad_w, 0, pad_h), "constant", -100)
        padded = padded.reshape(t, nh, vw, nw, vw).permute(0, 1, 3, 2, 4).reshape(t, nh * nw, vw, vw)
        seqlens = (padded != -100).sum([2, 3]).reshape(-1)
        flat = padded.reshape(-1)
        window_index.append(flat[flat != -100] + base)
        cu_win.extend((seqlens.cumsum(0) * unit + cu_win[-1]).tolist())
        base += t * gh * gw
    cu_win_t = torch.unique_consecutive(torch.tensor(cu_win, dtype=torch.int32))
    frames = torch.tensor([h * w for t, h, w in grid_thw for _ in range(t)], dtype=torch.int32)
    cu_frames = F.pad(frames.cumsum(0, dtype=torch.int32), (1, 0), value=0)
    return torch.cat(window_index), cu_win_t, cu_frames


def mrope_position_ids(input_ids: Sequence[int], grids: Sequence[Sequence[int]], image_token_id: int, merge: int,
                       tokens_per_second: int, video_token_id: Optional[int] = None,
                       second_per_grid_ts: Optional[Sequence[float]] = None) -> torch.Tensor:
    """(t, h, w) positions of ONE unpadded prompt whose image / video token runs correspond, in order, to `grids`. [3, L] int64.
    transformers 5.5.0 multiplies the temporal START position by time_interval = tokens_per_second * int(second_per_grid)
    -- constant over the whole grid, and applied to still images too with second_per_grid = 1 (:1018-1019, :1113); the parity
    target is the installed transformers, so this does the same. `second_per_grid_ts`: one entry per vision run, default 1."""
    ids = list(input_ids)
    spg = iter(second_per_grid_ts) if second_per_grid_ts is not None else None

    def kind(tok):          # mm_token_type_ids: text 0, image 1, video 2 -- adjacent runs of different kinds are separate groups
        return 1 if tok == image_token_id else (2 if video_token_id is not None and tok == video_token_id else 0)

    pos: List[torch.Tensor] = []
    cur, i, g = 0, 0, 0
    while i < len(ids):
        is_img = kind(ids[i])
        j = i
        while j < len(ids) and kind(ids[j]) == is_img:
            j += 1
        if not is_img:
            n = j - i
            pos.append(torch.arange(n).view(1, -1).expand(3, -1) + cur)
            cur += n
        else:
            t, h, w = grids[g]
            g += 1
            gt, gh, gw = t, h // merge, w // merge
            if j - i != gt * gh * gw:
                raise ValueError(f"image token run of {j - i} does not match grid {(t, h, w)}")
            pw = torch.arange(cur, cur + gw).repeat(gh * gt)
            ph = torch.arange(cur, cur + gh).repeat_interleave(gw * gt)
            interval = tokens_per_second * (int(next(spg)) if spg is not None else 1)
            pt = torch.full((gt * gh * gw,), cur * interval, dtype=torch.long)
            pos.append(torch.stack([pt, ph, pw], dim=0))
            cur += max(h, w) // merge
        i = j
    return torch.cat(pos, dim=1)


def rope_tables(head_dim_text: int, rope_theta: float, mrope_section: Sequence[int], head_dim_vis: int):
    """(text_inv_freq[64], text_axis[64], vis_inv_freq[hd/2], vis_axis[hd/2]) for vqa_qwen25vl_set_rope."""
    t_inv = 1.0 / (rope_theta ** (torch.arange(0, head_dim_text, 2, dtype=torch.int64).to(torch.float) / head_dim_text))
    t_axis = torch.cat([torch.full((n,), a, dtype=torch.int32) for a, n in enumerate(mrope_section)])
    assert t_axis.numel() == head_dim_text // 2
    q = head_dim_vis // 2                      # Qwen2_5_VisionRotaryEmbedding(dim = head_dim // 2)
    v_inv_q = 1.0 / (10000.0 ** (torch.arange(0, q, 2, dtype=torch.float) / q))    # [hd/4]
    v_inv = torch.cat([v_inv_q, v_inv_q])      # rotary_pos_emb = [freqs(h) | freqs(w)], then emb = cat(rot, rot)
    v_axis = torch.cat([torch.zeros(q // 2, dtype=torch.int32), torch.ones(q // 2, dtype=torch.int32)])
    return t_inv.float().contiguous(), t_axis.contiguous(), v_inv.float().contiguous(), v_axis.contiguous()


def build_batch_indices(input_ids: List[Sequence[int]], grids: Sequence[Sequence[int]], image_of_sample: Sequence[int],
                        image_token_id: int, merge: int, tokens_per_second: int, pad_id: int = 0,
                        video_token_id: Optional[int] = None, second_per_grid_ts: Optional[Sequence[float]] = None):
    """Right-pad a batch of prompts and build the per-token arrays the engine consumes. Each prompt holds ONE vision run (image
    or video tokens) fed by grid `image_of_sample[b]`; second_per_grid_ts is per grid (videos: temporal_patch_size / fps).
    Returns dict(input_ids [B,S], seq_lens [B], feat_index [B,S], position_ids [3, B*S]) as int32 CPU tensors."""
    unit = merge * merge
    feat_off = [0]
    for t, h, w in grids:
        feat_off.append(feat_off[-1] + t * h * w // unit)
    B = len(input_ids)
    S = max(len(x) for x in input_ids)
    ids = torch.full((B, S), pad_id, dtype=torch.int32)
    lens = torch.zeros(B, dtype=torch.int32)
    feat = torch.full((B, S), -1, dtype=torch.int32)
    pos = torch.zeros(3, B, S, dtype=torch.int32)
    for b, seq in enumerate(input_ids):
        seq_t = torch.as_tensor(list(seq), dtype=torch.int32)
        n = seq_t.numel()
        ids[b, :n] = seq_t
        lens[b] = n
        img = image_of_sample[b]
        m = seq_t == image_token_id
        if video_token_id is not None:
            m = m | (seq_t == video_token_id)
        feat[b, :n][m] = torch.arange(feat_off[img], feat_off[img + 1], dtype=torch.int32)
        spg = None if second_per_grid_ts is None else [second_per_grid_ts[img]]
        pos[:, b, :n] = mrope_position_ids(seq_t.tolist(), [grids[img]], image_token_id, merge, tokens_per_second, video_token_id,
                                           spg).to(torch.int32)
    return dict(input_ids=ids, seq_lens=lens, feat_index=feat, position_ids=pos.reshape(3, B * S).contiguous())


def first_generated_positions(idx) -> torch.Tensor:
    """mRoPE position of the first generated token of every prompt of `build_batch_indices(...)`: the position of the prompt's last token
    + 1; generated token t sits at that + t on all three axes. transformers' generate() advances the last prompt position ids by one per
    step (modeling_qwen2_5_vl.py:1576-1612, generation/utils.py), which is below max(prompt positions) + 1 when a video's temporal index
    exceeds the text positions. The chat template ends every prompt with text, where the three axes agree. [B] int32."""
    B, S = idx["input_ids"].shape
    pos = idx["position_ids"].view(3, B, S)
    last = pos[:, torch.arange(B), idx["seq_lens"].long() - 1]                       # [3, B]
    if not bool((last == last[0]).all()):
        raise ValueError("generation needs prompts that end with a text token")
    return (last[0] + 1).to(torch.int32)


def rollout_answer_score(tokens: Sequence[int], logp: torch.Tensor, answer_ids: Sequence[int], special_ids, mode: str = "forward") -> dict:
    """Which steps of a greedy rollout score which answer tokens, and the score: the reference's rule (qwen2vl_model.py), restated.
    tokens: the L generated ids of one sample (a stopping EOS included); logp: fp32 [>= L, >= len(answer_ids)], logp[s, j] = log p(s,
    answer_ids[j]) (engine.rollout_scores); special_ids: the tokenizer's {eos, bos, pad} ids (not the stop list); mode: "forward"
    (Qwen2VLModel.forward, :239-289), "start" or "end" (forward_with_trace's score_position, :381-416).
      * forward: a last token in special_ids sets offset 1 and n = min(n, L - 1) (n <= 0 raises); then n = min(n, L); answer token i is
        scored at step L - n + i - offset.
      * end: the same special-token rule; start = max(0, L - n - offset); n = min(n, L - start); n <= 0 raises.
      * start: start = 0, n = min(n, L).
    p_i = exp(logp) in fp32; score = (prod_i p_i) ** (1 / n) over Python floats. Returns dict(score, start, steps, n, probs). No device work."""
    L, n = len(tokens), len(answer_ids)
    if L < 1 or n < 1:
        raise ValueError("a rollout of at least one token and a non-empty answer are needed")
    offset = 0
    if mode in ("forward", "end") and int(tokens[-1]) in special_ids:
        offset, n = 1, min(n, L - 1)                                       # :247-257, :392-400
        if n <= 0 and mode == "forward":
            raise ValueError("No content tokens to score after removing special tokens")
    if mode == "forward":
        n = min(n, L)                                                      # :259-263
        start = L - n - offset                                             # :267 position -(n - i + offset)
    elif mode == "end":
        start = max(0, L - n - offset)                                     # :403-406
        n = min(n, L - start)                                              # :408-413
    elif mode == "start":
        start = 0                                                          # :382-384
        n = min(n, L - start)
    else:
        raise ValueError(f"mode must be 'forward', 'start' or 'end', got {mode!r}")
    if n <= 0:
        raise ValueError("No tokens available to score at the specified position")      # :415-416
    steps = list(range(start, start + n))
    probs = [float(torch.exp(logp[s, i].float())) for i, s in enumerate(steps)]
    joint = 1.0
    for p in probs:
        joint *= p
    return dict(score=joint ** (1.0 / n), start=start, steps=steps, n=n, probs=probs)


def build_packed_indices(input_ids: List[Sequence[int]], grids: Sequence[Sequence[int]], image_of_sample: Sequence[int],
                         image_token_id: int, merge: int, tokens_per_second: int, video_token_id: Optional[int] = None,
                         second_per_grid_ts: Optional[Sequence[float]] = None, align: int = 1):
    """KV-prefix sharing (SURVEY 8(f)1): prompts that start with the same tokens up to the end of their vision run -- the chat prefix and
    the image's pad tokens, i.e. every text scored against one image (reference score.py:104-106) -- share that prefix as ONE packed
    sequence; each prompt keeps only its remaining tokens as its own sequence. Returns the int32 CPU arrays vqa_qwen25vl_score takes over packed rows
    plus sizes: dict(input_ids [R], feat_index [R], position_ids [3, R], cu_seqlens [n_seq + 1], kv_prefix [n_seq], pair_row [B],
    pair_seq [B], total_rows, n_seq, max_seq_len, max_prompt_len, n_shared). A prompt whose prefix nobody else uses is stored whole
    (kv_prefix -1), so the packed form never has more rows than sum(len(prompt)).
    align: the shared prefix is cut to a multiple of `align` tokens (the rest stays in each prompt's own sequence). The engine passes the
    attention kernel's key tile (128): a prefix of whole key tiles leaves every suffix row's attention bit-identical to the unshared
    prefill, so sharing a prefix never changes a score."""
    unit = merge * merge
    feat_off = [0]
    for t, h, w in grids:
        feat_off.append(feat_off[-1] + t * h * w // unit)
    vis = {image_token_id} | ({video_token_id} if video_token_id is not None else set())
    prompts = [list(map(int, p)) for p in input_ids]
    cut = []                                    # prefix length of each prompt = index after its last vision token
    for p in prompts:
        last = max((i for i, t in enumerate(p) if t in vis), default=-1)
        cut.append((last + 1) // align * align)
    groups = {}
    for b, p in enumerate(prompts):
        if cut[b] > 0 and cut[b] < len(p):
            groups.setdefault((image_of_sample[b], tuple(p[:cut[b]])), []).append(b)
    shared = {k: v for k, v in groups.items() if len(v) > 1}
    seqs, kvp, pos_rows, feat_rows = [], [], [], []       # packed sequences in order: shared prefixes first, then one per prompt
    prefix_seq = {}

    def positions(b):
        img = image_of_sample[b]
        spg = None if second_per_grid_ts is None else [second_per_grid_ts[img]]
        return mrope_position_ids(prompts[b], [grids[img]], image_token_id, merge, tokens_per_second, video_token_id, spg).to(torch.int32)

    def feats(ids, img):
        t = torch.as_tensor(ids, dtype=torch.int32)
        f = torch.full((len(ids),), -1, dtype=torch.int32)
        m = torch.zeros(len(ids), dtype=torch.bool)
        for v in vis:
            m |= t == v
        if bool(m.any()):
            f[m] = torch.arange(feat_off[img], feat_off[img + 1], dtype=torch.int32)
        return f

    pos_cache = {}
    for key, members in shared.items():
        img, pre = key
        b0 = members[0]
        pos_cache[b0] = positions(b0)
        prefix_seq[key] = len(seqs)
        seqs.append(list(pre)); kvp.append(-1)
        pos_rows.append(pos_cache[b0][:, :len(pre)]); feat_rows.append(feats(prompts[b0], img)[:len(pre)])
    pair_seq, pair_last = [], []
    for b, p in enumerate(prompts):
        key = (image_of_sample[b], tuple(p[:cut[b]]))
        pos = pos_cache.get(b)
        if pos is None:
            pos = positions(b)
        if key in shared:
            own, start, pre = p[cut[b]:], cut[b], prefix_seq[key]
        else:
            own, start, pre = p, 0, -1
        pair_seq.append(len(seqs))
        seqs.append(own); kvp.append(pre)
        pos_rows.append(pos[:, start:])
        feat_rows.append(feats(p, image_of_sample[b])[start:])
    lens = [len(x) for x in seqs]
    cu = torch.zeros(len(seqs) + 1, dtype=torch.int32)
    cu[1:] = torch.as_tensor(lens, dtype=torch.int32).cumsum(0)
    pair_row = torch.as_tensor([int(cu[sq + 1]) - 1 for sq in pair_seq], dtype=torch.int32)
    max_prompt = max(lens[sq] + (lens[kvp[sq]] if kvp[sq] >= 0 else 0) for sq in pair_seq)
    return dict(input_ids=torch.as_tensor([t for x in seqs for t in x], dtype=torch.int32), feat_index=torch.cat(feat_rows),
                position_ids=torch.cat(pos_rows, dim=1).contiguous(), cu_seqlens=cu, kv_prefix=torch.as_tensor(kvp, dtype=torch.int32),
                pair_row=pair_row, pair_seq=torch.as_tensor(pair_seq, dtype=torch.int32), total_rows=int(cu[-1]), n_seq=len(seqs),
                max_seq_len=max(lens), max_prompt_len=max_prompt, n_shared=len(shared))

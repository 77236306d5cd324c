"""Qwen2.5-VL: host index logic and oracle pinned to the real transformers implementation (CPU only)."""
import pytest
import torch

from oracle import qwen25vl_oracle as qo
from t2v_metrics_b200 import qwen_host


def hf_model(cfg):
    from transformers import Qwen2_5_VLForConditionalGeneration
    from hf_reference import hf_qwen_config
    return Qwen2_5_VLForConditionalGeneration(hf_qwen_config(cfg)).eval()


TINY = dict(hidden=256, heads=2, kv_heads=1, mrope_section=(16, 24, 24))   # head_dim 128 like the 7B model


@pytest.fixture(scope="module")
def tiny():
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    return cfg, hf_model(cfg)


@pytest.mark.parametrize("grids", [[(1, 8, 6)], [(1, 4, 4), (1, 6, 10)], [(1, 16, 12)], [(2, 4, 6)]])
def test_vision_index_logic_matches_transformers(tiny, grids):
    cfg, m = tiny
    vis = m.model.visual
    g = torch.tensor(grids)
    widx_hf, cu_hf = vis.get_window_index(g)
    cu_hf = torch.unique_consecutive(torch.tensor(cu_hf, dtype=torch.int32))
    widx, cu_win, cu_frames = qwen_host.vision_window_index(grids, cfg.spatial_merge_size, cfg.window_size, cfg.patch_size)
    assert torch.equal(widx, widx_hf) and torch.equal(cu_win, cu_hf)
    cu_full = torch.nn.functional.pad(torch.repeat_interleave(g[:, 1] * g[:, 2], g[:, 0]).cumsum(0, dtype=torch.int32), (1, 0))
    assert torch.equal(cu_frames, cu_full)
    # rotary angles: table built from (pos ids, inv_freq, axis) == transformers' rot_pos_emb
    rot_hf = vis.rot_pos_emb(g)                                                    # [L, head_dim/2]
    pos = qwen_host.vision_rot_pos_ids(grids, cfg.spatial_merge_size)
    _, _, v_inv, v_axis = qwen_host.rope_tables(cfg.head_dim, cfg.rope_theta, cfg.mrope_section, cfg.vit_hidden // cfg.vit_heads)
    mine = pos[:, v_axis.long()].float() * v_inv[None]
    assert torch.equal(mine, rot_hf)


def test_mrope_positions_and_tables_match_transformers(tiny):
    cfg, m = tiny
    inp = qo.make_synthetic_inputs(cfg, 3, (84, 56), 11, ragged=True)
    for b, ids in enumerate(inp["input_ids"]):
        grid = [inp["grid_thw"][b]]
        hf_pos, _ = m.model.get_rope_index(ids[None], (ids == cfg.image_token_id).long()[None], image_grid_thw=torch.tensor(grid),
                                           attention_mask=torch.ones(1, len(ids), dtype=torch.long))
        mine = qwen_host.mrope_position_ids(ids.tolist(), grid, cfg.image_token_id, cfg.spatial_merge_size, cfg.tokens_per_second)
        assert torch.equal(mine, hf_pos[:, 0])
        assert torch.equal(mine, qo.mrope_position_ids(ids, grid, cfg))
    t_inv, t_axis, _, _ = qwen_host.rope_tables(cfg.head_dim, cfg.rope_theta, cfg.mrope_section, cfg.vit_hidden // cfg.vit_heads)
    assert torch.equal(t_inv, m.model.language_model.rotary_emb.inv_freq.float())
    assert t_axis.tolist() == [0] * 16 + [1] * 24 + [2] * 24


@pytest.mark.parametrize("spg", [None, [2.0], [0.5]])
def test_mrope_positions_video_match_transformers(tiny, spg):
    """SURVEY 8(d) config 5 / 8(c) iii: video runs (mm_token_type 2, video_grid_thw, second_per_grid_ts) in the installed
    transformers: temporal index = start * tokens_per_second * int(second_per_grid), constant over the grid."""
    cfg, m = tiny
    inp = qo.make_synthetic_inputs(cfg, 2, (56, 84), 9, ragged=True, frames=3)
    for b, ids in enumerate(inp["input_ids"]):
        grid = [inp["grid_thw"][b]]
        tt = torch.where(ids == cfg.video_token_id, 2, 0)[None]
        hf_pos, _ = m.model.get_rope_index(ids[None], tt, video_grid_thw=torch.tensor(grid),
                                           second_per_grid_ts=None if spg is None else torch.tensor(spg),
                                           attention_mask=torch.ones(1, len(ids), dtype=torch.long))
        mine = qwen_host.mrope_position_ids(ids.tolist(), grid, cfg.image_token_id, cfg.spatial_merge_size, cfg.tokens_per_second,
                                            cfg.video_token_id, spg)
        assert torch.equal(mine, hf_pos[:, 0])
        assert torch.equal(mine, qo.mrope_position_ids(ids, grid, cfg, spg))


def test_qwen_oracle_matches_transformers_video(tiny):
    """The oracle on a video input (grid t = 2 temporal patches, video token run) against Qwen2_5_VLForConditionalGeneration fed
    pixel_values_videos / video_grid_thw."""
    cfg, m = tiny
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    inp = qo.make_synthetic_inputs(cfg, 2, (56, 84), 10, ragged=True, frames=2)
    spg = [2.0, 2.0]
    o = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], return_all=True,
                          second_per_grid_ts=spg)
    t, gh, gw = inp["grid_thw"][0]
    P = t * gh * gw
    for b, ids in enumerate(inp["input_ids"]):
        with torch.no_grad():
            out = m(input_ids=ids[None], pixel_values_videos=inp["pixel_patches"][b * P:(b + 1) * P],
                    video_grid_thw=torch.tensor([list(inp["grid_thw"][b])]), second_per_grid_ts=torch.tensor([spg[b]]),
                    mm_token_type_ids=torch.where(ids == cfg.video_token_id, 2, 0)[None],
                    attention_mask=torch.ones(1, len(ids), dtype=torch.long))
        lg = out.logits[0, -1].float()
        assert float((lg - o["logits"][b]).abs().max()) < 5e-5
        assert abs(float(torch.softmax(lg, -1)[inp["answer_ids"][b]]) - float(o["scores"][b])) < 1e-6


def test_build_batch_indices_round_trip(tiny):
    cfg, _ = tiny
    inp = qo.make_synthetic_inputs(cfg, 4, (56, 56), 9, ragged=True, n_images=2)
    idx = qwen_host.build_batch_indices([x.tolist() for x in inp["input_ids"]], inp["grid_thw"], inp["image_of_sample"],
                                        cfg.image_token_id, cfg.spatial_merge_size, cfg.tokens_per_second)
    B, S = idx["input_ids"].shape
    n_tok = 4 * 4 // 4
    for b in range(B):
        n = int(idx["seq_lens"][b])
        assert idx["input_ids"][b, :n].tolist() == inp["input_ids"][b].tolist()
        f = idx["feat_index"][b]
        assert (f[:n] >= 0).sum() == n_tok and (f[n:] == -1).all()
        img = inp["image_of_sample"][b]
        assert f[f >= 0].tolist() == list(range(img * n_tok, (img + 1) * n_tok))
    assert idx["position_ids"].shape == (3, B * S)


@pytest.mark.parametrize("hw", [(84, 56), (56, 112)])
def test_qwen_oracle_matches_transformers(tiny, hw):
    cfg, m = tiny
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    inp = qo.make_synthetic_inputs(cfg, 2, hw, 10, ragged=True)
    o = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], return_all=True)
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    for b, ids in enumerate(inp["input_ids"]):
        with torch.no_grad():
            out = m(input_ids=ids[None], pixel_values=inp["pixel_patches"][b * P:(b + 1) * P],
                    image_grid_thw=torch.tensor([list(inp["grid_thw"][b])]), mm_token_type_ids=(ids == cfg.image_token_id).long()[None],
                    attention_mask=torch.ones(1, len(ids), dtype=torch.long))
        lg = out.logits[0, -1].float()
        assert float((lg - o["logits"][b]).abs().max()) < 5e-5
        assert abs(float(torch.softmax(lg, -1)[inp["answer_ids"][b]]) - float(o["scores"][b])) < 1e-6


def test_repetition_penalty_semantics():
    """SURVEY F8: the logits processor rescales ids present in the prompt before the softmax."""
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor
    torch.manual_seed(0)
    logits = torch.randn(50)
    prompt = torch.tensor([3, 7, 7, 11])
    ref = torch.softmax(RepetitionPenaltyLogitsProcessor(1.05)(prompt[None], logits[None].clone())[0], -1)[7]
    assert abs(float(qo.answer_probability(logits, 7, 1.0, prompt, 1.05)) - float(ref)) < 1e-7


def test_generation_config_penalty_lookup(tmp_path):
    """SURVEY F8: the reference's scores pass through the processors of the checkpoint's generation_config.json; the plugin reads the
    repetition penalty from the file beside the checkpoint, 1.0 (off) when there is none."""
    import json
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import _generation_config_penalty
    ckpt = tmp_path / "model.safetensors"
    ckpt.write_bytes(b"")
    assert _generation_config_penalty(str(ckpt)) == 1.0
    (tmp_path / "generation_config.json").write_text(json.dumps({"repetition_penalty": 1.05, "temperature": 0.1}))
    assert _generation_config_penalty(str(ckpt)) == 1.05
    assert _generation_config_penalty(str(tmp_path)) == 1.05
    assert _generation_config_penalty("/nonexistent/dir/model.bin") == 1.0


def load_qwen_golden(golden_dir):
    """tests/golden/qwen_tiny.pt (tools/make_golden_qwen.py): outputs of the real Qwen2_5_VLForConditionalGeneration; the weights are
    regenerated from the seed and pinned by their checksum."""
    import hashlib
    import os
    blob = torch.load(os.path.join(golden_dir, "qwen_tiny.pt"), weights_only=False)
    cfg = qo.Qwen25VLConfig(**blob["config"])
    sd = qo.make_synthetic_state_dict(cfg, seed=blob["weights_seed"])
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().view(torch.uint8).numpy().tobytes())
    assert h.hexdigest() == blob["weights_sha256"], "synthetic weights differ from the ones the golden was generated with"
    return blob, cfg, sd


@pytest.mark.parametrize("case", ["images", "video"])
def test_oracle_matches_committed_hf_golden(golden_dir, case):
    """The oracle against the committed outputs of the real transformers model (fp32 logits, answer probability, and the probability
    after RepetitionPenaltyLogitsProcessor(1.3) and temperature 0.5)."""
    blob, cfg, sd = load_qwen_golden(golden_dir)
    c = blob["cases"][case]
    inp, hf = c["inputs"], c["hf"]
    o = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], inp["image_of_sample"],
                          mode="fp32", return_all=True, second_per_grid_ts=c["second_per_grid_ts"])
    assert float((o["logits"] - hf["logits"]).abs().max()) < 5e-5
    assert float((o["scores"] - hf["probs"]).abs().max()) < 1e-6
    pen = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], inp["image_of_sample"],
                            mode="fp32", temperature=0.5, repetition_penalty=1.3, second_per_grid_ts=c["second_per_grid_ts"])
    assert float((torch.log(pen) - torch.log(hf["probs_penalty_1p3_T_0p5"])).abs().max()) < 1e-4


def test_packed_indices_reassemble_every_prompt():
    """KV-prefix sharing (SURVEY 8(f)1): build_packed_indices stores the [chat prefix + vision run] of prompts over one image once.
    Re-assembling prefix rows + own rows must give back exactly the ids, mRoPE positions and feature indices of the padded layout."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    g = torch.Generator().manual_seed(0)
    grids = [(1, 6, 4), (1, 4, 4), (1, 4, 6)]
    ntok = [t * h * w // 4 for t, h, w in grids]
    prompts, img = [], []
    for i in (0, 1):
        for k in range(3):
            prompts.append([5, 6, 7] + [cfg.image_token_id] * ntok[i] + [9] + torch.randint(0, 500, (4 + k,), generator=g).tolist())
            img.append(i)
    prompts.append([1, 2] + [cfg.image_token_id] * ntok[2] + [3, 4, 5])      # nobody shares this one: stored whole
    img.append(2)
    args = (cfg.image_token_id, cfg.spatial_merge_size, cfg.tokens_per_second)
    pk = qwen_host.build_packed_indices(prompts, grids, img, *args, video_token_id=cfg.video_token_id)
    full = qwen_host.build_batch_indices(prompts, grids, img, *args, video_token_id=cfg.video_token_id)
    S = full["input_ids"].shape[1]
    cu = pk["cu_seqlens"].tolist()
    assert pk["n_shared"] == 2 and pk["n_seq"] == 2 + len(prompts) and pk["total_rows"] == cu[-1] < sum(map(len, prompts))
    for b, p in enumerate(prompts):
        sq = int(pk["pair_seq"][b])
        pre = int(pk["kv_prefix"][sq])
        rows = (list(range(cu[pre], cu[pre + 1])) if pre >= 0 else []) + list(range(cu[sq], cu[sq + 1]))
        assert pk["input_ids"][rows].tolist() == p
        assert torch.equal(pk["position_ids"][:, rows], full["position_ids"].view(3, len(prompts), S)[:, b, :len(p)])
        assert torch.equal(pk["feat_index"][rows], full["feat_index"][b, :len(p)])
        assert int(pk["pair_row"][b]) == rows[-1]
    assert int(pk["kv_prefix"][int(pk["pair_seq"][-1])]) == -1
    assert pk["max_prompt_len"] == max(map(len, prompts)) and pk["max_seq_len"] == max(cu[i + 1] - cu[i] for i in range(pk["n_seq"]))


def test_packed_prefix_is_cut_to_whole_key_tiles():
    """With align = 128 (the engine's setting) the shared prefix is the longest common run of whole 128-row key tiles, which may end inside
    the vision run; the suffixes then carry the rest of it, and re-assembly still gives the padded layout exactly."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    grids = [(1, 20, 40), (1, 4, 4)]                 # 200 and 4 vision tokens
    ntok = [t * h * w // 4 for t, h, w in grids]
    prompts = [[5, 6, 7] + [cfg.image_token_id] * ntok[0] + [9, 10 + k, 11] for k in range(3)]
    prompts += [[5, 6] + [cfg.image_token_id] * ntok[1] + [9, 12 + k] for k in range(2)]       # prefix shorter than one tile: not shared
    img = [0, 0, 0, 1, 1]
    args = (cfg.image_token_id, cfg.spatial_merge_size, cfg.tokens_per_second)
    pk = qwen_host.build_packed_indices(prompts, grids, img, *args, video_token_id=cfg.video_token_id, align=128)
    full = qwen_host.build_batch_indices(prompts, grids, img, *args, video_token_id=cfg.video_token_id)
    S = full["input_ids"].shape[1]
    cu = pk["cu_seqlens"].tolist()
    assert pk["n_shared"] == 1 and cu[1] - cu[0] == 128
    for b, p in enumerate(prompts):
        sq = int(pk["pair_seq"][b])
        pre = int(pk["kv_prefix"][sq])
        assert (pre >= 0) == (b < 3)
        rows = (list(range(cu[pre], cu[pre + 1])) if pre >= 0 else []) + list(range(cu[sq], cu[sq + 1]))
        assert pk["input_ids"][rows].tolist() == p
        assert torch.equal(pk["position_ids"][:, rows], full["position_ids"].view(3, len(prompts), S)[:, b, :len(p)])
        assert torch.equal(pk["feat_index"][rows], full["feat_index"][b, :len(p)])

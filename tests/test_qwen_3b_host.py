"""Qwen2.5-VL-3B on the host (no GPU): the architecture read from a checkpoint's config.json, the tied lm_head binding, and the oracle
pinned to the committed golden of the real transformers model with tied embeddings and 8 query heads per K/V head."""
import json

import pytest
import torch

from oracle import qwen25vl_oracle as qo
from oracle import qwen25vl_generate as qg
from qwen_tied import EMBED, TINY_GQA8, load_tied_golden, tied_state_dict, with_lm_head
from t2v_metrics_b200.config import QWEN25VL_MODELS, Qwen25VLConfig

# the layout of the published checkpoints' config.json: text fields at the top level, `rope_scaling`, `vision_config`
_VISION = dict(depth=32, hidden_act="silu", hidden_size=1280, intermediate_size=3420, num_heads=16, in_chans=3, patch_size=14,
               spatial_merge_size=2, spatial_patch_size=14, window_size=112, fullatt_block_indexes=[7, 15, 23, 31], tokens_per_second=2,
               temporal_patch_size=2)
_TEXT = dict(architectures=["Qwen2_5_VLForConditionalGeneration"], model_type="qwen2_5_vl", hidden_act="silu", rms_norm_eps=1e-6,
             rope_theta=1000000.0, rope_scaling=dict(type="mrope", mrope_section=[16, 24, 24]), image_token_id=151655,
             video_token_id=151656, vision_start_token_id=151652, vision_end_token_id=151653, bos_token_id=151643, eos_token_id=151645)
PUBLISHED = {
    "qwen2.5-vl-3b": dict(_TEXT, hidden_size=2048, intermediate_size=11008, num_hidden_layers=36, num_attention_heads=16,
                          num_key_value_heads=2, vocab_size=151936, tie_word_embeddings=True, vision_config=dict(_VISION, out_hidden_size=2048)),
    "qwen2.5-vl-7b": dict(_TEXT, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28, num_attention_heads=28,
                          num_key_value_heads=4, vocab_size=152064, tie_word_embeddings=False, vision_config=dict(_VISION, out_hidden_size=3584)),
}


@pytest.mark.parametrize("entry", ["VQAScore", "get_score_model"])
def test_3b_is_accepted_by_name_and_the_listing_is_unchanged(entry, tmp_path):
    """VQAScore(model="qwen2.5-vl-3b") and get_score_model pass the registry and reach the plugin's load (here it stops at the missing
    weights of a checkpoint directory whose config.json is the 3B's). list_all_models() still lists the bench.py workloads only."""
    import t2v_metrics_b200 as t2v
    assert t2v.list_all_models() == ["clip-flant5-xxl", "clip-flant5-xl", "qwen2.5-vl-7b"]
    assert "qwen2.5-vl-3b" in t2v.VQAScore.list_all_models(None)
    (tmp_path / "config.json").write_text(json.dumps(PUBLISHED["qwen2.5-vl-3b"]))
    make = t2v.VQAScore if entry == "VQAScore" else t2v.get_score_model
    with pytest.raises(FileNotFoundError, match="no weights"):
        make(model="qwen2.5-vl-3b", device="cpu", tokenizer=_NoTokenizer(), checkpoint=str(tmp_path))
    with pytest.raises(NotImplementedError):
        t2v.get_score_model("qwen2.5-vl-32b")


def test_3b_is_registered_with_the_group_size_the_kernels_take():
    cfg = QWEN25VL_MODELS["qwen2.5-vl-3b"]["config"]()
    assert QWEN25VL_MODELS["qwen2.5-vl-3b"]["weights"] == "Qwen/Qwen2.5-VL-3B-Instruct"
    assert (cfg.hidden, cfg.layers, cfg.heads, cfg.kv_heads, cfg.head_dim, cfg.mlp, cfg.vocab) == (2048, 36, 16, 2, 128, 11008, 151936)
    assert cfg.tie_word_embeddings and cfg.heads // cfg.kv_heads == 8 and cfg.out_hidden == 2048
    assert not QWEN25VL_MODELS["qwen2.5-vl-7b"]["config"]().tie_word_embeddings


@pytest.mark.parametrize("name", sorted(PUBLISHED))
def test_from_hf_config_reproduces_the_table(name, tmp_path):
    """Both layouts: the published flat file, and transformers 5.5.0's Qwen2_5_VLConfig(...).to_dict() of it (text fields under
    text_config, rope under rope_parameters), from a dict, a file and a directory."""
    from transformers import Qwen2_5_VLConfig
    want = QWEN25VL_MODELS[name]["config"]()
    flat = PUBLISHED[name]
    nested = Qwen2_5_VLConfig(**json.loads(json.dumps(flat))).to_dict()
    assert "text_config" in nested and "hidden_size" not in nested
    assert Qwen25VLConfig.from_hf_config(flat) == want
    assert Qwen25VLConfig.from_hf_config(nested) == want
    (tmp_path / "config.json").write_text(json.dumps(nested, default=str))
    assert Qwen25VLConfig.from_hf_config(str(tmp_path)) == want
    assert Qwen25VLConfig.from_hf_config(str(tmp_path / "config.json")) == want


class _NoTokenizer:
    pass


def test_mismatched_config_json_raises_before_anything_is_bound(tmp_path):
    """A 7B config.json in the directory given as the 3B's checkpoint: ValueError naming the fields, before the weights are read (there
    are none) and before the engine is created (there is no GPU here). A matching config.json passes and the load reaches the weights."""
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    (tmp_path / "config.json").write_text(json.dumps(PUBLISHED["qwen2.5-vl-7b"]))
    with pytest.raises(ValueError, match=r"hidden = 3584 \(expected 2048\).*tie_word_embeddings = False \(expected True\)"):
        Qwen2VLModel("qwen2.5-vl-3b", device="cpu", tokenizer=_NoTokenizer(), checkpoint=str(tmp_path))
    (tmp_path / "config.json").write_text(json.dumps(PUBLISHED["qwen2.5-vl-3b"]))
    with pytest.raises(FileNotFoundError, match="no weights"):
        Qwen2VLModel("qwen2.5-vl-3b", device="cpu", tokenizer=_NoTokenizer(), checkpoint=str(tmp_path))


def _tiny_engine_cfg(tied):
    from qwen_tied import engine_config
    import dataclasses
    return dataclasses.replace(engine_config(qo.Qwen25VLConfig.tiny(**TINY_GQA8)), tie_word_embeddings=tied)


def test_tied_lm_head_is_the_embedding_tensor():
    from t2v_metrics_b200.engine import convert_qwen_state_dict
    cfg = _tiny_engine_cfg(True)
    sd = tied_state_dict(qo.Qwen25VLConfig.tiny(**TINY_GQA8), seed=3)
    assert "lm_head.weight" not in sd
    out = convert_qwen_state_dict(sd, cfg, "cpu")
    assert out["llm.lm_head"].data_ptr() == out["llm.embed"].data_ptr()
    assert torch.equal(out["llm.embed"], sd[EMBED])
    # a tied checkpoint that also stores lm_head.weight: the embedding wins, as in HF's tie_weights()
    extra = dict(sd, **{"lm_head.weight": torch.zeros_like(sd[EMBED])})
    out = convert_qwen_state_dict(extra, cfg, "cpu")
    assert out["llm.lm_head"].data_ptr() == out["llm.embed"].data_ptr() and torch.equal(out["llm.lm_head"], sd[EMBED])


def test_untied_config_without_lm_head_raises():
    from t2v_metrics_b200.engine import convert_qwen_state_dict
    sd = tied_state_dict(qo.Qwen25VLConfig.tiny(**TINY_GQA8), seed=3)
    with pytest.raises(KeyError, match="no lm_head.weight and its config does not tie"):
        convert_qwen_state_dict(sd, _tiny_engine_cfg(False), "cpu")


@pytest.mark.parametrize("case", ["images", "video"])
def test_oracle_matches_committed_tied_gqa8_golden(golden_dir, case):
    """The oracle with lm_head bound to the embedding against the real transformers model with tie_word_embeddings=True: logits, answer
    probability plain and penalised, the top-5 trace, the greedy tokens under the repetition penalty on their decisive steps, and the
    per-step answer probabilities of the 4-token rollout teacher-forced on HF's tokens."""
    blob, cfg, sd = load_tied_golden(golden_dir)
    sd = with_lm_head(sd)
    c = blob["cases"][case]
    inp, hf, spg = c["inputs"], c["hf"], c["second_per_grid_ts"]
    args = (sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"])
    o = qo.qwen25vl_score(*args, inp["answer_ids"], inp["image_of_sample"], mode="fp32", return_all=True, second_per_grid_ts=spg)
    assert float((o["logits"] - hf["logits"]).abs().max()) < 5e-5
    assert float((o["scores"] - hf["probs"]).abs().max()) < 1e-6
    pen = qo.qwen25vl_score(*args, inp["answer_ids"], inp["image_of_sample"], mode="fp32", temperature=0.5, repetition_penalty=1.3,
                            second_per_grid_ts=spg)
    assert float((torch.log(pen) - torch.log(hf["probs_penalty_1p3_T_0p5"])).abs().max()) < 1e-4
    top = torch.topk(torch.softmax(o["logits"], -1), 5, dim=-1)
    assert torch.equal(top.indices.to(torch.int32), hf["top5_ids"])
    assert torch.allclose(top.values, hf["top5_probs"], rtol=2e-4, atol=1e-7)
    g = qg.qwen25vl_generate(*args, blob["gen_new_tokens"], (), inp["image_of_sample"], repetition_penalty=blob["gen_penalty"],
                             second_per_grid_ts=spg, forced=hf["gen_ids"])
    for b, ids in enumerate(hf["gen_ids"]):
        s = g["scores"][b]
        top2 = s.topk(2, dim=-1).values
        assert torch.allclose(top2[:, 0] - top2[:, 1], hf["gen_margins"][b], atol=1e-4)
        decisive = hf["gen_margins"][b] > 1e-4
        assert s.argmax(-1)[decisive].tolist() == torch.tensor(ids)[decisive].tolist()
    r = qg.qwen25vl_generate(*args, blob["rollout_new_tokens"], (), inp["image_of_sample"], second_per_grid_ts=spg, forced=hf["roll_ids"])
    for b, ans in enumerate(c["rollout_answers"]):
        p = torch.softmax(r["scores"][b], -1)[:, ans]
        assert torch.allclose(p, hf["roll_p"][b], rtol=2e-4, atol=1e-7), (p, hf["roll_p"][b])

"""Qwen2.5-VL greedy generation, CPU side: the generation oracle and the first-generated-position helper pinned to the real transformers
`generate(do_sample=False)`, the committed golden, and the plugin's refusals (no GPU needed)."""
import hashlib
import os

import pytest
import torch

from oracle import qwen25vl_oracle as qo
from oracle import qwen25vl_generate as qg
from t2v_metrics_b200 import qwen_host
from test_qwen_host import hf_model, TINY


@pytest.fixture(scope="module")
def tiny_hf():
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m = hf_model(cfg)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    return cfg, sd, m


def load_generate_golden(golden_dir):
    """tests/golden/qwen_generate_tiny.pt (tools/make_golden_qwen_generate.py) with its weights and inputs regenerated from their seeds."""
    blob = torch.load(os.path.join(golden_dir, "qwen_generate_tiny.pt"), weights_only=False)
    cfg = qo.Qwen25VLConfig(**blob["config"])
    sd = qo.make_synthetic_state_dict(cfg, seed=blob["weights_seed"])
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().view(torch.uint8).numpy().tobytes())
    assert h.hexdigest() == blob["weights_sha256"], "synthetic weights differ from the ones the golden was generated with"
    return blob, cfg, sd


def golden_case_inputs(cfg, case):
    s = case["inputs"]
    inp = qo.make_synthetic_inputs(cfg, s["batch"], tuple(s["hw"]), s["text_len"], seed=s["seed"], ragged=s["ragged"], n_images=s["n_images"],
                                   frames=s["frames"])
    h = hashlib.sha256()
    h.update(inp["pixel_patches"].contiguous().numpy().tobytes())
    for ids in inp["input_ids"]:
        h.update(ids.to(torch.int64).numpy().tobytes())
    assert h.hexdigest() == case["inputs_sha256"], "synthetic inputs differ from the ones the golden was generated with"
    return inp, s["spg"]


def hf_generate_ids(m, cfg, inp, spg, max_new, penalty, eos_ids):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from make_golden_qwen_generate import hf_generate
    return hf_generate(m, cfg, inp, spg, max_new, penalty, eos_ids)


@pytest.mark.parametrize("video,pen", [(False, 1.0), (False, 1.3), (True, 1.0), (True, 1.3)])
def test_oracle_generate_matches_transformers(tiny_hf, video, pen):
    """The oracle's cached greedy decode is token-identical to Qwen2_5_VLForConditionalGeneration.generate(do_sample=False) in fp32, with
    and without the repetition penalty (which covers the generated ids too), for images and a video grid."""
    cfg, sd, m = tiny_hf
    inp = qo.make_synthetic_inputs(cfg, 2, (56, 84) if video else (84, 56), 10, seed=7, ragged=True, frames=2 if video else 1)
    spg = [2.0, 2.0] if video else None
    hf_ids, _ = hf_generate_ids(m, cfg, inp, spg, 10, pen, ())
    o = qg.qwen25vl_generate(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], 10, (), repetition_penalty=pen,
                             second_per_grid_ts=spg)
    assert o["tokens"] == hf_ids


def test_oracle_generate_stops_on_eos_like_transformers(tiny_hf):
    cfg, sd, m = tiny_hf
    inp = qo.make_synthetic_inputs(cfg, 2, (84, 56), 10, seed=8, ragged=True)
    free, _ = hf_generate_ids(m, cfg, inp, None, 10, 1.0, ())
    stop = free[0][3]
    eos = (stop, next(t for t in range(cfg.vocab) if all(t not in x for x in free)))
    hf_ids, _ = hf_generate_ids(m, cfg, inp, None, 10, 1.0, eos)
    o = qg.qwen25vl_generate(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], 10, eos)
    assert o["tokens"] == hf_ids and o["tokens"][0] == free[0][:free[0].index(stop) + 1]


def test_teacher_forced_scores_reproduce_the_greedy_path(tiny_hf):
    """Fed its own greedy tokens, the teacher-forced run gives the same processed scores step by step, and their arg-max is the path."""
    cfg, sd, _ = tiny_hf
    inp = qo.make_synthetic_inputs(cfg, 2, (84, 56), 10, seed=9, ragged=True)
    free = qg.qwen25vl_generate(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], 8, (), repetition_penalty=1.3)
    tf = qg.qwen25vl_generate(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], 8, (), repetition_penalty=1.3,
                              forced=free["tokens"])
    for b in range(2):
        assert torch.equal(tf["scores"][b], free["scores"][b])
        assert tf["scores"][b].argmax(-1).tolist() == free["tokens"][b]


@pytest.mark.parametrize("video", [False, True])
def test_first_generated_positions_are_the_ones_transformers_generate_feeds(tiny_hf, video):
    """The position ids HF generate() passes to the language model at the first decode step. With a video (second_per_grid 2: temporal
    index start * 4) the prompt's largest position is on the temporal axis and exceeds the last text position, so the rope_deltas
    reading max(positions) + 1 would be wrong here; the video case checks that the helper does not use it."""
    cfg, _, m = tiny_hf
    inp = qo.make_synthetic_inputs(cfg, 2, (56, 84), 9, seed=4, ragged=True, frames=2 if video else 1)
    spg = [2.0] * 2 if video else None
    idx = qwen_host.build_batch_indices([x.tolist() for x in inp["input_ids"]], inp["grid_thw"], list(range(2)), cfg.image_token_id,
                                        cfg.spatial_merge_size, cfg.tokens_per_second, video_token_id=cfg.video_token_id, second_per_grid_ts=spg)
    first = qwen_host.first_generated_positions(idx)
    seen = []
    hook = m.model.language_model.register_forward_pre_hook(lambda mod, a, kw: seen.append(kw["position_ids"].clone()), with_kwargs=True)
    try:
        hf_generate_ids(m, cfg, inp, spg, 3, 1.0, ())
    finally:
        hook.remove()
    decode = [p for p in seen if p.shape[-1] == 1]          # prefill, 2 decode steps per prompt
    assert len(decode) == 4
    for b in range(2):
        for t in range(2):
            p = decode[2 * b + t].view(-1, 1)[-3:, 0]         # (t, h, w) rows
            assert p.tolist() == [int(first[b]) + t] * 3
    if video:
        B, S = idx["input_ids"].shape
        assert any(int(idx["position_ids"].view(3, B, S)[:, b].max()) + 1 > int(first[b]) for b in range(2))


@pytest.mark.parametrize("case", ["images_pen1.0", "images_pen1.3", "video_pen1.0", "video_pen1.3", "eos"])
def test_oracle_matches_committed_generate_golden(golden_dir, case):
    blob, cfg, sd = load_generate_golden(golden_dir)
    c = blob["cases"][case]
    inp, spg = golden_case_inputs(cfg, c)
    o = qg.qwen25vl_generate(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], blob["max_new_tokens"], c["eos_ids"],
                             inp["image_of_sample"], repetition_penalty=c["penalty"], second_per_grid_ts=spg)
    # fp32 CPU arithmetic orders its sums differently from the stored run: paths are compared up to the first fp32 near-tie (margin < 1e-3)
    compared = 0
    for b, s in enumerate(o["scores"]):
        m = c["margins"][b]
        n = next((t for t in range(len(m)) if float(m[t]) < 1e-3), len(m))
        assert o["tokens"][b][:n + 1] == c["ids"][b][:n + 1] and (n < len(m) or o["tokens"][b] == c["ids"][b])
        top2 = s[:n + 1].topk(2, dim=-1).values
        assert float(((top2[:, 0] - top2[:, 1]) - m[:n + 1]).abs().max()) < 1e-4
        compared += n
    assert compared >= 8


class _NoLaunchEngine:
    def __getattr__(self, name):
        raise AssertionError(f"engine.{name} used: the call must be refused before any launch")


def _bare_plugin():
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    p = Qwen2VLModel.__new__(Qwen2VLModel)
    p.engine = _NoLaunchEngine()
    p.cfg = qo.Qwen25VLConfig.tiny(**TINY)
    p.repetition_penalty = 1.0
    p.model_name = "qwen2.5-vl-7b"
    return p


@pytest.mark.parametrize("kw", [dict(temperature=0.7), dict(do_sample=True), dict(temperature=0.0, do_sample=True)])
def test_generate_refuses_sampling_before_any_launch(kw):
    with pytest.raises(NotImplementedError, match="greedy"):
        _bare_plugin().generate(images=["a.png"], texts=["describe"], **kw)


def test_generate_refuses_videos_before_any_launch():
    with pytest.raises(NotImplementedError):
        _bare_plugin().generate(images=["clip.mp4"], texts=["describe"])


def test_generate_eos_ids_come_from_the_generation_config(tmp_path):
    import json
    p = _bare_plugin()
    p._checkpoint = str(tmp_path / "model.safetensors")
    p.tokenizer = type("Tok", (), {"eos_token_id": 7})()
    assert p._eos_ids() == [7]
    (tmp_path / "generation_config.json").write_text(json.dumps({"eos_token_id": [151645, 151643]}))
    assert p._eos_ids() == [151645, 151643]

"""CLIP-FlanT5 greedy generation, CPU side: the generation oracle pinned to the real transformers T5ForConditionalGeneration.generate on
spliced embeddings, the committed golden, and the plugin's refusals and EOS source (no GPU needed)."""
import json
import os
import sys

import pytest
import torch

from oracle import clipt5_oracle as orc
from oracle import clipt5_generate as cg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import make_golden_clipt5_generate as mk  # noqa: E402


@pytest.fixture(scope="module")
def tiny_hf():
    cfg = orc.ClipT5Config.tiny()
    sd = orc.make_synthetic_state_dict(cfg, seed=mk.WEIGHTS_SEED)
    return cfg, sd, mk.hf_t5(cfg, sd)


def load_generate_golden(golden_dir):
    """tests/golden/clipt5_generate_tiny.pt (tools/make_golden_clipt5_generate.py) with its weights and inputs regenerated from their seeds
    and checked against the stored checksums."""
    blob = torch.load(os.path.join(golden_dir, "clipt5_generate_tiny.pt"), weights_only=False)
    cfg = orc.ClipT5Config(**blob["config"])
    sd = orc.make_synthetic_state_dict(cfg, seed=blob["weights_seed"])
    assert orc.state_dict_sha256(sd) == blob["weights_sha256"], "synthetic weights differ from the ones the golden was generated with"
    inp = mk.case_inputs(cfg, blob["inputs"])
    assert mk.inputs_checksum(inp) == blob["inputs_sha256"], "synthetic inputs differ from the ones the golden was generated with"
    return blob, cfg, sd, inp


def hf_ids(t5, sd, cfg, inp, max_new, eos_ids):
    embeds, mask, _ = cg.encode_prompts(sd, cfg, inp["pixels"], inp["input_ids"], inp["text_lens"], inp.get("image_index"))
    return mk.hf_generate(t5, embeds, mask, max_new, list(eos_ids))[0]


def oracle_ids(sd, cfg, inp, max_new, eos_ids=(), **kw):
    return cg.clipt5_generate(sd, cfg, inp["pixels"], inp["input_ids"], inp["text_lens"], max_new, eos_ids, inp.get("image_index"), **kw)


@pytest.mark.parametrize("seed,n_images", [(5, None), (7, 2)])
def test_oracle_generate_matches_transformers(tiny_hf, seed, n_images):
    """The oracle's greedy decode is token-identical to T5ForConditionalGeneration.generate(do_sample=False, num_beams=1) in fp32 on the
    spliced prompts: ragged prompt lengths, and (n_images=2) the first image shared by two prompts."""
    cfg, sd, t5 = tiny_hf
    inp = orc.make_synthetic_inputs(cfg, 3, 13, seed=seed, ragged=True, n_images=n_images)
    assert len(set(inp["text_lens"].tolist())) > 1
    assert oracle_ids(sd, cfg, inp, 10)["tokens"] == hf_ids(t5, sd, cfg, inp, 10, ())


def test_oracle_generate_stops_on_eos_like_transformers(tiny_hf):
    cfg, sd, t5 = tiny_hf
    inp = orc.make_synthetic_inputs(cfg, 2, 12, seed=8, ragged=True)
    free = hf_ids(t5, sd, cfg, inp, 10, ())
    stop = free[0][3]
    eos = (stop, next(t for t in range(cfg.vocab) if all(t not in x for x in free)))
    ref = hf_ids(t5, sd, cfg, inp, 10, eos)
    got = oracle_ids(sd, cfg, inp, 10, eos)["tokens"]
    assert got == ref and got[0] == free[0][:free[0].index(stop) + 1]
    assert got[1] == free[1][:len(got[1])]


def test_teacher_forced_scores_reproduce_the_greedy_path(tiny_hf):
    """Fed its own greedy tokens, the teacher-forced run gives the same scores step by step, and their arg-max is the path."""
    cfg, sd, _ = tiny_hf
    inp = orc.make_synthetic_inputs(cfg, 2, 12, seed=9, ragged=True)
    free = oracle_ids(sd, cfg, inp, 6)
    tf = oracle_ids(sd, cfg, inp, 6, forced=free["tokens"])
    for b in range(2):
        assert torch.equal(tf["scores"][b], free["scores"][b])
        assert tf["scores"][b].argmax(-1).tolist() == free["tokens"][b]


@pytest.mark.parametrize("case", ["free", "eos"])
def test_oracle_matches_committed_generate_golden(golden_dir, case):
    blob, cfg, sd, inp = load_generate_golden(golden_dir)
    c = blob["cases"][case]
    o = oracle_ids(sd, cfg, inp, blob["max_new_tokens"], c["eos_ids"])
    # fp32 CPU arithmetic may order its sums differently from the stored run: paths are compared up to the first fp32 near-tie (< 1e-3)
    compared = 0
    for b, s in enumerate(o["scores"]):
        m = c["margins"][b]
        n = next((t for t in range(len(m)) if float(m[t]) < 1e-3), len(m))
        assert o["tokens"][b][:n + 1] == c["ids"][b][:n + 1] and (n < len(m) or o["tokens"][b] == c["ids"][b])
        top2 = s[:n + 1].topk(2, dim=-1).values
        assert float(((top2[:, 0] - top2[:, 1]) - m[:n + 1]).abs().max()) < 1e-4
        compared += n
    assert compared >= 8
    if case == "eos":
        assert any(len(x) < blob["max_new_tokens"] for x in c["ids"]) and any(len(x) == blob["max_new_tokens"] for x in c["ids"])


class _NoLaunchEngine:
    def __getattr__(self, name):
        raise AssertionError(f"engine.{name} used: the call must be refused before any launch")


class _WordTokenizer:
    """Stand-in T5 tokenizer: one id per word (3 + hash mod 400), every chunk ending in </s> (1)."""
    pad_token_id = 0
    eos_token_id = 1

    def __call__(self, chunk):
        import types
        return types.SimpleNamespace(input_ids=[3 + (sum(map(ord, w)) % 400) for w in chunk.split()] + [1])


def _bare_plugin():
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import CLIPT5Model
    p = CLIPT5Model.__new__(CLIPT5Model)
    p.engine = _NoLaunchEngine()
    p.cfg = orc.ClipT5Config.tiny()
    p.model_name = "clip-flant5-xxl"
    p.conversational_style = "t5_chat"
    p.context_len = 2048
    p.tokenizer = _WordTokenizer()
    p._checkpoint = None
    return p


@pytest.mark.parametrize("kw", [dict(temperature=0.7), dict(do_sample=True), dict(temperature=0.0, do_sample=True)])
def test_generate_refuses_sampling_before_any_launch(kw):
    with pytest.raises(NotImplementedError, match="greedy"):
        _bare_plugin().generate(images=["a.png"], texts=["describe"], **kw)


def test_generate_refuses_image_placeholder_in_caption_before_any_launch():
    with pytest.raises(ValueError, match="placeholder"):
        _bare_plugin().generate(images=["a.png", "b.png"], texts=["a dog", "a <image> of a cat"])


def test_generate_eos_ids_come_from_the_generation_config(tmp_path):
    p = _bare_plugin()
    p._checkpoint = str(tmp_path / "model.safetensors")
    p.tokenizer = type("Tok", (), {"eos_token_id": 1})()
    assert p._eos_ids() == [1]
    (tmp_path / "generation_config.json").write_text(json.dumps({"eos_token_id": [1, 32001]}))
    assert p._eos_ids() == [1, 32001]
    (tmp_path / "generation_config.json").write_text(json.dumps({"eos_token_id": 5}))
    assert p._eos_ids() == [5]

"""Qwen2.5-VL sampled generation, CPU side: how the plugin resolves (temperature, top_k, top_p) against transformers' own resolution,
per-prompt seeds, the fp64 warper restatement against HF's warper objects, Philox4x32-10 against Random123's known answers, the sampled
decode restatement against HF generate(do_sample=True) where HF is deterministic, and the sampling struct's ctypes layout."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

import sample_ref as sr
from oracle import qwen25vl_oracle as qo
from test_qwen_host import TINY, hf_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ parameter resolution
class _RecordingEngine:
    """Stands in for QwenVLEngine: sample_prompts / generate_prompts are methods of the class, and record what they receive."""
    calls = []

    def generate_workspace_bytes(self, b, s, p, n):
        return 1

    def generate_prompts(self, pix, grids, prompts, n, eos, **kw):
        self.calls.append(("greedy", None, kw["repetition_penalty"]))
        return [[1] for _ in prompts]

    def sample_prompts(self, pix, grids, prompts, n, eos, seeds, temperature, top_k, top_p, **kw):
        self.calls.append(("sample", (temperature, top_k, top_p), kw["repetition_penalty"], list(seeds)))
        return [[1] for _ in prompts]


class _Tok:
    eos_token_id = 7

    def encode(self, s, add_special_tokens=False):
        return [ord(c) % 50 for c in s]

    def decode(self, ids, skip_special_tokens=False, clean_up_tokenization_spaces=True):
        return " ".join(map(str, ids))


def _plugin(tmp_path, gen_config=None, penalty=1.05):
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    p = Qwen2VLModel.__new__(Qwen2VLModel)
    p.engine = _RecordingEngine()
    _RecordingEngine.calls = []
    p.cfg = qo.Qwen25VLConfig.tiny(**TINY)
    p.repetition_penalty = penalty
    p.model_name = "qwen2.5-vl-7b"
    p.tokenizer = _Tok()
    p._checkpoint = str(tmp_path / "model.safetensors")
    if gen_config is not None:
        (tmp_path / "generation_config.json").write_text(json.dumps(gen_config))
    p._vision = lambda images, fps=None: (list(range(len(images))), torch.zeros(4, 1176), [(1, 2, 2)] * len(images), [p.cfg.image_token_id] * len(images), None)
    return p


# (do_sample, temperature) -> sampled? as the reference decides (qwen2vl_model.py:512-551)
TRUTH = [(None, 0.0, False), (None, 0.7, True), (True, 0.0, False), (True, 0.7, True), (False, 0.7, False), (False, 0.0, False)]


@pytest.mark.parametrize("do_sample,temperature,sampled", TRUTH)
@pytest.mark.parametrize("gen_config,top_k", [(None, 50), ({"top_k": 20, "top_p": 0.5, "temperature": 0.1}, 20), ({"top_k": 0}, 0),
                                              ({"repetition_penalty": 1.05}, 50)])
def test_sampling_parameters_follow_the_reference(tmp_path, do_sample, temperature, sampled, gen_config, top_k):
    p = _plugin(tmp_path, gen_config)
    p.generate(["a.png", "b.png"], ["x", "y"], max_new_tokens=4, temperature=temperature, do_sample=do_sample, top_p=0.8)
    call = _RecordingEngine.calls[-1]
    if not sampled:
        assert call[0] == "greedy" and call[2] == 1.05
    else:
        # temperature and top_p are the call's, top_k the file's (else 50), the penalty the plugin's
        assert call[0] == "sample" and call[1] == (temperature, top_k, 0.8) and call[2] == 1.05 and len(call[3]) == 2


@pytest.mark.parametrize("key,value", [("min_p", 0.05), ("typical_p", 0.9), ("epsilon_cutoff", 3e-4), ("eta_cutoff", 3e-4), ("top_h", 0.5)])
def test_other_warpers_are_refused_before_any_launch(tmp_path, key, value):
    p = _plugin(tmp_path, {key: value})
    p._vision = None          # an image read would fail with TypeError
    with pytest.raises(NotImplementedError, match=key):
        p.generate(["a.png"], ["x"], temperature=0.7)
    assert _RecordingEngine.calls == []
    p = _plugin(tmp_path)
    p.generate(["a.png"], ["x"], temperature=0.0)
    assert _RecordingEngine.calls[-1][0] == "greedy"


def test_engine_without_sampling_is_refused_on_its_class(tmp_path):
    p = _plugin(tmp_path)

    class GreedyOnly:
        def __init__(self):
            self.sample_prompts = lambda *a, **k: None      # an instance attribute does not make a class capable

    p.engine = GreedyOnly()
    with pytest.raises(NotImplementedError, match="greedy"):
        p.generate(["a.png"], ["x"], temperature=0.7)


def test_hf_builds_the_same_processors(tmp_path):
    """transformers' own _prepare_generation_config and _get_logits_processor on a tiny Qwen2_5_VLForConditionalGeneration with a
    checkpoint generation_config.json yield exactly [RepetitionPenalty, Temperature, TopK, TopP] with the plugin's values."""
    from transformers import GenerationConfig
    from transformers.generation import logits_process as lp
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import sampling_params
    for file, want_k in (({"top_k": 20, "repetition_penalty": 1.05}, 20), ({"repetition_penalty": 1.05}, 50)):
        (tmp_path / "generation_config.json").write_text(json.dumps(file))
        cfg = qo.Qwen25VLConfig.tiny(**TINY)
        m = hf_model(cfg)
        m.generation_config = GenerationConfig.from_pretrained(str(tmp_path))
        gc, _ = m._prepare_generation_config(None, do_sample=True, temperature=0.7, top_p=0.9)
        procs = m._get_logits_processor(generation_config=gc, input_ids_seq_length=4, encoder_input_ids=torch.zeros(1, 4, dtype=torch.long),
                                        prefix_allowed_tokens_fn=None, logits_processor=None, device="cpu")
        assert [type(x) for x in procs] == [lp.RepetitionPenaltyLogitsProcessor, lp.TemperatureLogitsWarper, lp.TopKLogitsWarper,
                                            lp.TopPLogitsWarper]
        T, k, p = sampling_params(str(tmp_path / "model.safetensors"), None, 0.7, 0.9)
        assert (procs[1].temperature, procs[2].top_k, procs[3].top_p) == (T, k, p) and k == want_k
        assert procs[0].penalty == 1.05


def test_seeds_are_reproducible(tmp_path):
    p = _plugin(tmp_path)
    run = lambda **kw: (p.generate(["a.png"] * 3, ["x", "y", "z"], temperature=0.7, **kw), _RecordingEngine.calls[-1][3])[1]
    g = lambda: torch.Generator().manual_seed(4)
    a, b = run(generator=g()), run(generator=g())
    torch.manual_seed(4)
    c = run()
    torch.manual_seed(4)
    d = run()
    assert a == b and c == d and len(set(a)) == 3 and all(0 <= s < 2 ** 63 for s in a + c)
    assert run(generator=torch.Generator().manual_seed(5)) != a


# ------------------------------------------------------------------------------------------------ warpers and Philox
@pytest.mark.parametrize("V", [152064, 151936, 1000])
def test_fp64_warpers_equal_hf_warper_objects(V):
    """The restatement's kept set equals HF's TopK / TopP warpers run on the same fp32 scores, except ids of the tie group at a top-p cut
    (HF's unstable sort orders a tie group arbitrarily) and ids whose cumulative mass is within 1e-5 of 1 - top_p (HF's fp32 cumsum)."""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    gen = torch.Generator().manual_seed(V)
    rows = [(torch.randn(V, generator=gen) * 3).bfloat16(), (torch.randint(-16, 9, (V,), generator=gen).float() / 8).bfloat16()]
    for row in rows:
        for T in (0.7, 1.0):
            x = sr.processed_scores(row[None], None, 1.0, T)[0]
            for k, p in ((0, 0.9), (50, 0.9), (1, 1.0), (50, 1.0), (0, 0.5), (V + 5, 1e-6), (0, 1e-8)):
                s = torch.from_numpy(x.copy())[None]
                if k:
                    s = TopKLogitsWarper(top_k=min(k, V))(None, s)
                if p < 1.0:
                    s = TopPLogitsWarper(top_p=p)(None, s)
                hf = np.isfinite(s[0].numpy())
                kept, cum, thr = sr.warp_row(x, k, p)
                diff = np.nonzero(hf != kept)[0]
                if len(diff):
                    # the tie group at the cut: the lowest score either side keeps (HF's sort may order that group either way)
                    in_tie = (x[diff] == x[kept].min()) | (x[diff] == x[hf].min())
                    assert np.all(in_tie | (np.abs(cum[diff] - thr) < 1e-5)), (V, T, k, p, diff[:5])


def test_philox_matches_random123_known_answers():
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert tuple(int(v) for v in sr.philox4x32_10(np.array(ctr, dtype=np.uint32), key)) == want


def test_gumbel_uniforms_are_open_and_exact():
    g = sr.gumbel(2 ** 64 - 1, 7, 4099)
    assert g.shape == (4099,) and np.isfinite(g).all()
    assert not np.array_equal(g, sr.gumbel(2 ** 64 - 1, 8, 4099))


# ------------------------------------------------------------------------------------------------ sampled decode vs HF
@pytest.mark.parametrize("top_k,top_p", [(1, 0.9), (0, 1e-6)])
def test_sampled_decode_matches_hf_where_hf_is_deterministic(top_k, top_p):
    """top_k = 1, or top_p = 1e-6 without top_k, leaves one token per step: HF generate(do_sample=True) is then deterministic, and the
    restatement's sampled decode must give its tokens, in fp32 on the tiny model, with and without the repetition penalty."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    m = hf_model(cfg)
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    inp = qo.make_synthetic_inputs(cfg, 2, (84, 56), 10, seed=7, ragged=True)
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    for pen in (1.0, 1.3):
        want = []
        for b, ids in enumerate(inp["input_ids"]):
            out = m.generate(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long),
                             pixel_values=inp["pixel_patches"][b * P:(b + 1) * P], image_grid_thw=torch.tensor([list(inp["grid_thw"][b])]),
                             mm_token_type_ids=(ids == cfg.image_token_id).long()[None], max_new_tokens=8, do_sample=True, temperature=0.7,
                             top_k=top_k, top_p=top_p, repetition_penalty=pen, eos_token_id=None, pad_token_id=0)
            want.append(out[0, len(ids):].tolist())
        got = sr.qwen25vl_sample(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], 8, [3, 4], 0.7, top_k, top_p,
                                 repetition_penalty=pen)
        assert got["tokens"] == want


# ------------------------------------------------------------------------------------------------ ABI
def test_sampling_struct_layout_matches_header():
    from t2v_metrics_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqa_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\} vqa_qwen25vl_sampling;", text).group(1)
    cls = _lib.VqaQwen25VLSampling
    assert [f[0] for f in cls._fields_] == re.findall(r"(\w+);", body)
    assert ctypes.sizeof(cls) == 24 and cls.temperature.offset == 8 and cls.top_k.offset == 12 and cls.top_p.offset == 16
    # top_p is a double in the header and the binding: a float field would round the caller's top_p before 1 - top_p is formed
    assert re.search(r"\bdouble\s+top_p;", body) and dict(cls._fields_)["top_p"] is ctypes.c_double
    s = cls(top_p=0.9)
    assert s.top_p == 0.9

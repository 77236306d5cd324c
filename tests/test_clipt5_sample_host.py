"""CLIP-FlanT5 sampled generation, CPU side: the sampled decode restatement against HF T5 generate(do_sample=True) where HF is
deterministic, the processors HF builds for a FlanT5 generation config, and the plugin's parameter resolution, refusals, seeds, grouping
of identical pairs and chunking, with a stand-in engine (no GPU needed)."""
import copy
import json

import pytest
import torch

import sample_ref as sr
from sample_ref_clipt5 import clipt5_sample
from oracle import clipt5_oracle as orc
from oracle import clipt5_generate as cg
from test_clipt5_generate_host import tiny_hf  # noqa: F401  (fixture)

FLANT5_GENERATION_CONFIG = {"decoder_start_token_id": 0, "eos_token_id": 1, "pad_token_id": 0}


# ------------------------------------------------------------------------------------------------ restatement vs HF
@pytest.mark.parametrize("top_k,top_p", [(1, 0.9), (0, 1e-6)])
def test_sampled_decode_matches_hf_where_hf_is_deterministic(tiny_hf, top_k, top_p):  # noqa: F811
    """top_k = 1, or top_p = 1e-6 without top_k, leaves one token per step: HF T5 generate(inputs_embeds, do_sample=True) is then
    deterministic, and clipt5_sample must give its tokens in fp32 on the tiny model (ragged prompts, one image shared)."""
    cfg, sd, t5 = tiny_hf
    inp = orc.make_synthetic_inputs(cfg, 3, 13, seed=5, ragged=True, n_images=2)
    embeds, mask, _ = cg.encode_prompts(sd, cfg, inp["pixels"], inp["input_ids"], inp["text_lens"], inp["image_index"])
    gc = copy.deepcopy(t5.generation_config)
    gc.eos_token_id, gc.max_new_tokens, gc.max_length, gc.min_length = None, 8, None, 0
    gc.do_sample, gc.num_beams, gc.temperature, gc.top_k, gc.top_p = True, 1, 0.7, top_k, top_p
    with torch.no_grad():
        want = t5.generate(inputs_embeds=embeds, attention_mask=mask.long(), generation_config=gc)[:, 1:].tolist()
    got = clipt5_sample(sd, cfg, inp["pixels"], inp["input_ids"], inp["text_lens"], 8, [3, 4, 5], 0.7, top_k, top_p,
                        image_index=inp["image_index"])
    assert got["tokens"] == want


def test_hf_builds_temperature_top_k_top_p_for_a_flant5_config(tiny_hf, tmp_path):  # noqa: F811
    """transformers' own _prepare_generation_config and _get_logits_processor on T5ForConditionalGeneration with FlanT5's
    generation_config.json yield exactly [Temperature, TopK, TopP] with the values sampling_params resolves."""
    from transformers import GenerationConfig
    from transformers.generation import logits_process as lp
    from t2v_metrics_b200.models.vqascore_models.sampling import sampling_params
    _, _, t5 = tiny_hf
    for extra, want_k in (({}, 50), ({"top_k": 20}, 20)):
        (tmp_path / "generation_config.json").write_text(json.dumps({**FLANT5_GENERATION_CONFIG, **extra}))
        m = copy.copy(t5)
        m.generation_config = GenerationConfig.from_pretrained(str(tmp_path))
        gc, _ = m._prepare_generation_config(None, do_sample=True, temperature=0.7, top_p=0.9)
        procs = m._get_logits_processor(generation_config=gc, input_ids_seq_length=1, encoder_input_ids=torch.zeros(1, 4, dtype=torch.long),
                                        prefix_allowed_tokens_fn=None, logits_processor=None, device="cpu")
        assert [type(x) for x in procs] == [lp.TemperatureLogitsWarper, lp.TopKLogitsWarper, lp.TopPLogitsWarper]
        T, k, p = sampling_params(str(tmp_path / "model.safetensors"), None, 0.7, 0.9)
        assert (procs[0].temperature, procs[1].top_k, procs[2].top_p) == (T, k, p) and k == want_k


# ------------------------------------------------------------------------------------------------ plugin with a stand-in engine
class _RecordingEngine:
    """Stands in for ClipT5Engine: generate_tensors / sample_tensors are methods of the class and record what they receive. A sample's
    ids are [3 + seed % 997] so the strings show which seed each one was drawn with."""
    calls = []
    device = torch.device("cpu")

    def generate_tensors(self, pixels, input_ids, lens, n, eos, image_index=None):
        self.calls.append(("greedy", input_ids.shape[0]))
        return [[3] for _ in range(input_ids.shape[0])]

    def sample_tensors(self, pixels, input_ids, lens, n, eos, seeds, temperature, top_k, top_p, image_index=None, prompt_of_sample=None):
        n_prompts = input_ids.shape[0]
        assert sorted(set(prompt_of_sample)) == list(range(n_prompts)) and len(prompt_of_sample) == len(seeds)
        rows = [input_ids[i, :int(lens[i])].tolist() for i in range(n_prompts)]
        self.calls.append(("sample", (temperature, top_k, top_p), list(seeds), n_prompts, [rows[q] for q in prompt_of_sample]))
        return [[3 + s % 997] for s in seeds]


class _WordTokenizer:
    pad_token_id = 0
    eos_token_id = 1

    def __call__(self, chunk):
        import types
        return types.SimpleNamespace(input_ids=[3 + (sum(map(ord, w)) % 400) for w in chunk.split()] + [1])

    def decode(self, ids, skip_special_tokens=False):
        return " ".join(str(i) for i in ids)


def _plugin(tmp_path, gen_config=None):
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import CLIPT5Model
    p = CLIPT5Model.__new__(CLIPT5Model)
    p.engine = _RecordingEngine()
    _RecordingEngine.calls = []
    p.cfg = orc.ClipT5Config.tiny()
    p.model_name = "clip-flant5-xxl"
    p.conversational_style = "t5_chat"
    p.context_len = 2048
    p.tokenizer = _WordTokenizer()
    p._checkpoint = str(tmp_path / "model.safetensors")
    p.load_images = lambda paths, num_frames=8: torch.zeros(len(paths), 3, 4, 4)
    if gen_config is not None:
        (tmp_path / "generation_config.json").write_text(json.dumps(gen_config))
    return p


# (do_sample, temperature) -> sampled? as the reference decides (qwen2vl_model.py:512-551)
TRUTH = [(None, 0.0, False), (None, 0.7, True), (True, 0.0, False), (True, 0.7, True), (False, 0.7, False), (False, 0.0, False)]


@pytest.mark.parametrize("do_sample,temperature,sampled", TRUTH)
@pytest.mark.parametrize("gen_config,top_k", [(None, 50), ({**FLANT5_GENERATION_CONFIG, "top_k": 20, "temperature": 0.1}, 20),
                                              ({"top_k": 0}, 0)])
def test_sampling_parameters_follow_the_reference(tmp_path, do_sample, temperature, sampled, gen_config, top_k):
    p = _plugin(tmp_path, gen_config)
    p.generate(["a.png", "b.png"], ["x", "y"], max_new_tokens=4, temperature=temperature, do_sample=do_sample, top_p=0.8)
    call = _RecordingEngine.calls[-1]
    if not sampled:
        assert call[0] == "greedy"
    else:
        # temperature and top_p are the call's, top_k the file's (else 50)
        assert call[0] == "sample" and call[1] == (temperature, top_k, 0.8) and len(call[2]) == 2


@pytest.mark.parametrize("key,value", [("min_p", 0.05), ("typical_p", 0.9), ("epsilon_cutoff", 3e-4), ("eta_cutoff", 3e-4), ("top_h", 0.5),
                                       ("repetition_penalty", 1.2)])
def test_unsupported_processors_are_refused_before_any_launch(tmp_path, key, value):
    p = _plugin(tmp_path, {key: value})
    p.load_images = None          # an image read would fail with TypeError
    with pytest.raises(NotImplementedError, match=key):
        p.generate(["a.png"], ["x"], temperature=0.7)
    assert _RecordingEngine.calls == []
    if key == "repetition_penalty":      # the greedy path is as before: FlanT5's greedy decode applies no processor either way
        p = _plugin(tmp_path)
        p.generate(["a.png"], ["x"], temperature=0.0)
        assert _RecordingEngine.calls[-1][0] == "greedy"


def test_engine_without_sampling_is_refused_on_its_class(tmp_path):
    p = _plugin(tmp_path)

    class GreedyOnly:
        def __init__(self):
            self.sample_tensors = lambda *a, **k: None      # an instance attribute does not make a class capable

    p.engine = GreedyOnly()
    with pytest.raises(NotImplementedError, match="greedy"):
        p.generate(["a.png"], ["x"], temperature=0.7)


def test_seeds_are_reproducible(tmp_path):
    p = _plugin(tmp_path)

    def run(**kw):
        out = p.generate(["a.png"] * 3, ["x", "y", "z"], temperature=0.7, **kw)
        return out, _RecordingEngine.calls[-1][2]
    g = lambda: torch.Generator().manual_seed(4)
    a, b = run(generator=g()), run(generator=g())
    torch.manual_seed(4)
    c = run()
    torch.manual_seed(4)
    d = run()
    assert a == b and c == d and len(set(a[1])) == 3 and all(0 <= s < 2 ** 63 for s in a[1] + c[1])
    assert run(generator=torch.Generator().manual_seed(5)) != a


@pytest.mark.parametrize("cap", [4, 64])
def test_identical_pairs_share_an_encoding_and_keep_their_seeds_and_order(tmp_path, cap):
    """Groups of identical (image, text) pairs of sizes 3, 2, 1, 4 and 5, interleaved in the caller's order: each engine call encodes its
    distinct pairs once (n_prompts = distinct pairs in the call), a group that fits a call is never split, and every string is the one
    drawn with the seed the caller's order gives that pair, as without grouping."""
    p = _plugin(tmp_path)
    p.GENERATE_MAX_PAIRS = cap
    sizes = {"g0": 3, "g1": 2, "g2": 1, "g3": 4, "g4": 5}
    pending = dict(sizes)
    order = []
    while any(pending.values()):         # round-robin: the members of a group are not adjacent
        for g in sizes:
            if pending[g]:
                order.append(g)
                pending[g] -= 1
    images = [f"{g}.png" if g != "g2" else "g0.png" for g in order]      # g2 shares g0's image with another text
    texts = [f"caption {g}" for g in order]
    out = p.generate(images, texts, max_new_tokens=4, temperature=0.7, generator=torch.Generator().manual_seed(11))
    seeds = torch.randint(0, 2 ** 63 - 1, (len(order),), dtype=torch.int64, generator=torch.Generator().manual_seed(11)).tolist()
    assert out == [str(3 + s % 997) for s in seeds]
    calls = [c for c in _RecordingEngine.calls if c[0] == "sample"]
    assert all(len(c[2]) <= cap for c in calls)
    assert sum(c[3] for c in calls) == (len(sizes) if cap == 64 else len(sizes) + 1)      # only the 5-group exceeds a 4-pair call
    where = {}
    for ci, c in enumerate(calls):
        assert len({tuple(r) for r in c[4]}) == c[3]          # one encoded prompt per distinct pair of the call
        for s in c[2]:
            where.setdefault(order[seeds.index(s)], set()).add(ci)
    assert all(len(where[g]) == 1 for g in sizes if sizes[g] <= cap)
    # each sample continued its own pair's prompt
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import format_question
    prompts = p._prompt_ids([format_question(t) for t in texts])
    for c in calls:
        for s, row in zip(c[2], c[4]):
            assert row == prompts[seeds.index(s)]

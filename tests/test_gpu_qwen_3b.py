"""Qwen2.5-VL with a tied lm_head and 8 query heads per K/V head (the 3B's layout) on a real H100: the engine against the committed golden
of the real transformers model (tests/golden/qwen_tied_gqa8_tiny.pt) on the paths the plugin's forward, forward_with_trace, generate and
forward(max_new_tokens=4) run, for still images and a frame stack, with KV-prefix sharing on and off; and the plugin itself on
`qwen2.5-vl-3b` with a tied state dict. Tolerances are those of the untied golden tests (test_gpu_qwen.py, test_gpu_qwen_generate.py,
test_gpu_qwen_rollout_score.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import qwen25vl_oracle as qo
from qwen_tied import engine_config, load_tied_golden, with_lm_head
from test_gpu_qwen_generate import decisive_prefix, prompts_of, teacher_forced
from test_gpu_qwen_rollout_score import logp_gap

CASES = ["images", "video"]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


_GOLD = {}


def golden(golden_dir, dev):
    """(blob, oracle cfg, tied sd, the oracle's view of it, engine) once per module."""
    if not _GOLD:
        from t2v_metrics_b200.engine import QwenVLEngine
        blob, cfg, sd = load_tied_golden(golden_dir)
        eng = QwenVLEngine(engine_config(cfg), dev)
        eng.load_state_dict(sd)
        _GOLD.update(blob=blob, cfg=cfg, sd=sd, osd=with_lm_head(sd), eng=eng)
    g = _GOLD
    return g["blob"], g["cfg"], g["sd"], g["osd"], g["eng"]


def test_tied_binding_is_one_device_tensor(golden_dir, dev):
    _, _, _, _, eng = golden(golden_dir, dev)
    assert eng._weights["llm.lm_head"].data_ptr() == eng._weights["llm.embed"].data_ptr()
    assert eng._weights["llm.embed"].is_cuda


@pytest.mark.parametrize("share", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_score_and_trace_match_tied_golden(golden_dir, dev, case, share):
    """forward: the answer probability plain and after the repetition penalty 1.3 at T = 0.5; forward_with_trace: the top-5 of the last
    position, against softmax of HF's fp32 logits."""
    blob, cfg, _, osd, eng = golden(golden_dir, dev)
    c = blob["cases"][case]
    inp, hf, spg = c["inputs"], c["hf"], c["second_per_grid_ts"]
    o16 = qo.qwen25vl_score(osd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], inp["image_of_sample"],
                            mode="bf16", second_per_grid_ts=spg)
    gap = float((torch.log(o16) - torch.log(hf["probs"])).abs().max())
    prompts = prompts_of(inp)
    kw = dict(second_per_grid_ts=spg, share_prefix=share)
    p = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"], inp["image_of_sample"], **kw).cpu()
    ids, probs = eng.topk_last(5)
    ids, probs = ids.cpu(), probs.cpu()
    pp = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"], inp["image_of_sample"], temperature=0.5,
                           repetition_penalty=1.3, **kw).cpu()
    e = float((torch.log(p) - torch.log(hf["probs"])).abs().max())
    ep = float((torch.log(pp) - torch.log(hf["probs_penalty_1p3_T_0p5"])).abs().max())
    print(f"\n[tied golden {case} share={share}] engine {p.tolist()} HF {hf['probs'].tolist()} |dlogp| {e:.3e}; penalised {ep:.3e}; "
          f"oracle bf16-vs-HF {gap:.3e}")
    assert e <= 2.0 * gap + 2e-2
    assert ep <= 2.0 * gap / 0.5 + 4e-2
    full = torch.softmax(hf["logits"], -1)
    for b in range(len(prompts)):
        assert float((torch.log(probs[b]) - torch.log(full[b, ids[b].long()])).abs().max()) < 6e-2
        top = hf["top5_probs"][b]
        if float(top[0] - top[1]) > 2e-2 * float(top[0]):
            assert int(ids[b, 0]) == int(hf["top5_ids"][b, 0])


@pytest.mark.parametrize("case", CASES)
def test_generate_matches_tied_golden(golden_dir, dev, case):
    """generate: 8 greedy tokens under the repetition penalty, HF's ids up to the first step whose HF margin is below 2x the oracle's
    bf16-vs-fp32 score gap at that step."""
    blob, cfg, _, osd, eng = golden(golden_dir, dev)
    c = blob["cases"][case]
    inp, hf, spg = c["inputs"], c["hf"], c["second_per_grid_ts"]
    toks = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), blob["gen_new_tokens"], (),
                                image_of_sample=inp["image_of_sample"], repetition_penalty=blob["gen_penalty"], second_per_grid_ts=spg)
    s32, s16 = teacher_forced(osd, cfg, inp, hf["gen_ids"], blob["gen_penalty"], spg)
    compared = 0
    for b, hf_ids in enumerate(hf["gen_ids"]):
        thr = 2.0 * (s16[b] - s32[b]).abs().amax(-1) + 1e-3
        n = decisive_prefix(hf["gen_margins"][b] - thr, 0.0)
        print(f"\n[tied generate {case}] b={b} engine {toks[b]}\n    HF {hf_ids} decisive steps {n}")
        assert toks[b][:n] == hf_ids[:n]
        compared += n
    assert compared >= 4


@pytest.mark.parametrize("case", CASES)
def test_rollout_matches_tied_golden(golden_dir, dev, case):
    """forward(max_new_tokens=4): on HF's decisive steps the rollout's tokens are HF's and every answer log-probability is within 2x the
    oracle's bf16-vs-fp32 gap (+ 1e-3) of log softmax(HF scores)."""
    blob, cfg, _, osd, eng = golden(golden_dir, dev)
    c = blob["cases"][case]
    inp, hf, spg = c["inputs"], c["hf"], c["second_per_grid_ts"]
    answers = c["rollout_answers"]
    r = eng.rollout_scores(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), answers, blob["rollout_new_tokens"], (),
                           image_of_sample=inp["image_of_sample"], second_per_grid_ts=spg)
    s32, s16 = teacher_forced(osd, cfg, inp, hf["roll_ids"], 1.0, spg)
    compared = 0
    for b, hf_ids in enumerate(hf["roll_ids"]):
        top2 = s32[b].topk(2, dim=-1).values
        thr = 2.0 * (s16[b] - s32[b]).abs().amax(-1) + 1e-3
        n = decisive_prefix(top2[:, 0] - top2[:, 1] - thr, 0.0)
        assert r["tokens"][b][:n] == hf_ids[:n]
        # step 0 is the prompt's own position, common to both paths whatever the margins
        m = max(n, 1)
        gap = logp_gap(s16[b], s32[b], 1.0)[:m, None]
        err = (r["logp"][b, :m, :len(answers[b])] - torch.log(hf["roll_p"][b][:m].double()).float()).abs()
        print(f"\n[tied rollout {case}] b={b} decisive steps {n} max err {float(err.max()):.3e}")
        assert bool((err <= 2.0 * gap + 1e-3).all()), (err, gap)
        compared += m
    assert compared >= len(hf["roll_ids"])


class _Tokenizer:
    """Stand-in tokenizer: characters -> code points (mod 500); ids 600+ (vision) and 630+ ("special") are dropped by skip_special_tokens."""
    eos_token_id = 639
    pad_token_id = 638
    bos_token_id = None

    def encode(self, s, add_special_tokens=False):
        return [ord(ch) % 500 for ch in s]

    def decode(self, ids, skip_special_tokens=False, clean_up_tokenization_spaces=True):
        return " ".join(str(int(i)) for i in ids if not (skip_special_tokens and int(i) >= 630))


def test_plugin_runs_qwen25_vl_3b_with_a_tied_state_dict(golden_dir, dev, tmp_path):
    """The `qwen2.5-vl-3b` plugin with the tied golden's weights (no lm_head.weight anywhere): its lm_head binding is the embedding's
    device tensor, and forward, forward_with_trace, generate and forward(max_new_tokens=4) run and agree with each other."""
    import numpy as np
    from PIL import Image
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    blob, cfg, sd, _, _ = golden(golden_dir, dev)
    rng = np.random.default_rng(0)
    paths = []
    for i, (h, w) in enumerate(((60, 90), (84, 56))):
        p = tmp_path / f"{i}.png"
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(p)
        paths.append(str(p))
    model = Qwen2VLModel("qwen2.5-vl-3b", device=str(dev), tokenizer=_Tokenizer(), state_dict=dict(sd), config=engine_config(cfg),
                         checkpoint=str(tmp_path / "none.bin"), min_pixels=56 * 56, max_pixels=112 * 112)
    w = model.engine._weights
    assert w["llm.lm_head"].data_ptr() == w["llm.embed"].data_ptr()
    images, texts = [paths[0], paths[1], paths[0]], ["a red car", "two dogs", "a blue sky"]
    s = model.forward(images, texts)
    s_tr, trace = model.forward_with_trace(images, texts)
    assert s.shape == (3,) and bool(((s > 0) & (s <= 1)).all()) and torch.equal(s.cpu(), s_tr.cpu()) and len(trace) == 3
    out = model.generate(images=images, texts=texts, max_new_tokens=6)
    assert len(out) == 3 and all(isinstance(x, str) and x for x in out)
    s4 = model.forward(images, texts, max_new_tokens=4)
    assert s4.shape == (3,) and bool(((s4 > 0) & (s4 <= 1)).all())

"""Qwen2.5-VL scoring over a greedy rollout, CPU side: the reference's rule for which steps score which answer tokens
(qwen_host.rollout_answer_score), and the teacher-forced generation oracle's per-step probabilities and top-5 pinned to the real
transformers generate(output_scores=True) through the committed golden (no GPU needed)."""
import hashlib
import math
import os

import pytest
import torch

from oracle import qwen25vl_oracle as qo
from oracle import qwen25vl_generate as qg
from t2v_metrics_b200 import qwen_host
from test_qwen_generate_host import golden_case_inputs

EOS, PAD, BOS, STOP = 90, 91, 92, 93        # STOP: on the stop list of generation, not in the tokenizer's special set
SPECIAL = {EOS, PAD, BOS}


def _logp(L, n):
    """logp[s, j] = log(0.01 * (s + 1) + 0.001 * j): every (step, answer index) pair has its own probability."""
    s = torch.arange(L, dtype=torch.float32)[:, None]
    j = torch.arange(n, dtype=torch.float32)[None, :]
    return torch.log(0.01 * (s + 1) + 0.001 * j)


# (tokens, answer ids, mode, expected (step, answer index) pairs) -- reference line numbers in t2v_metrics/models/vqascore_models/qwen2vl_model.py
CASES = [
    # EOS last, answer fits: offset 1, token i at L - n + i - 1 (:247-257, :267)
    ([1, 2, 3, 4, EOS], [7, 8], "forward", [(2, 0), (3, 1)]),
    ([1, 2, 3, 4, EOS], [7, 8], "end", [(2, 0), (3, 1)]),                          # :392-403
    # EOS last with n > L - 1: n = L - 1, the answer's first L - 1 tokens (:254)
    ([1, 2, EOS], [7, 8, 9, 10], "forward", [(0, 0), (1, 1)]),
    ([1, 2, EOS], [7, 8, 9, 10], "end", [(0, 0), (1, 1)]),                         # :399, :403-413
    # length stop with L < n: n = L, answer truncated to its first L tokens (:259-263; :405-413)
    ([1, 2], [7, 8, 9], "forward", [(0, 0), (1, 1)]),
    ([1, 2], [7, 8, 9], "end", [(0, 0), (1, 1)]),
    # pad or bos last: the same special-token rule as EOS (:240-255)
    ([1, 2, 3, PAD], [7], "forward", [(2, 0)]),
    ([1, 2, 3, BOS], [7, 8], "end", [(1, 0), (2, 1)]),
    # a stop-list id outside the tokenizer's special set is scored like content (:247 tests the tokenizer's ids, not the stop list)
    ([1, 2, 3, STOP], [7, 8], "forward", [(2, 0), (3, 1)]),
    ([1, 2, 3, STOP], [7, 8], "end", [(2, 0), (3, 1)]),
    # "start" against "end": start scores from step 0 and ignores a trailing special token (:382-384)
    ([1, 2, 3, 4, 5, EOS], [7, 8], "start", [(0, 0), (1, 1)]),
    ([1, 2, 3, 4, 5, EOS], [7, 8], "end", [(3, 0), (4, 1)]),
    ([1, 2, EOS], [7, 8, 9, 10], "start", [(0, 0), (1, 1), (2, 2)]),             # n = min(n, L) (:408-413)
    ([1, 2, 3, 4, 5], [7, 8], "end", [(3, 0), (4, 1)]),                           # no special token: start = L - n (:403)
]


@pytest.mark.parametrize("tokens,answer,mode,pairs", CASES)
def test_rollout_selection_rule(tokens, answer, mode, pairs):
    lp = _logp(len(tokens), len(answer))
    r = qwen_host.rollout_answer_score(tokens, lp, answer, SPECIAL, mode)
    assert list(zip(r["steps"], range(r["n"]))) == pairs
    assert r["start"] == pairs[0][0] and r["n"] == len(pairs)
    probs = [float(torch.exp(lp[s, i])) for s, i in pairs]
    assert r["probs"] == probs
    assert r["score"] == math.prod(probs) ** (1.0 / len(pairs))            # geometric mean over Python floats (:265-289)


def test_eos_as_the_only_token_raises_each_modes_message():
    lp = _logp(1, 2)
    with pytest.raises(ValueError, match="^No content tokens to score after removing special tokens$"):      # :256-257
        qwen_host.rollout_answer_score([EOS], lp, [7, 8], SPECIAL, "forward")
    with pytest.raises(ValueError, match="^No tokens available to score at the specified position$"):      # :415-416
        qwen_host.rollout_answer_score([EOS], lp, [7, 8], SPECIAL, "end")
    r = qwen_host.rollout_answer_score([EOS], lp, [7, 8], SPECIAL, "start")
    assert r["steps"] == [0] and r["n"] == 1


def test_probabilities_are_fp32_and_the_product_is_python_float():
    lp = torch.tensor([[-0.1, -2.0], [-3.0, -0.7]], dtype=torch.float32)
    r = qwen_host.rollout_answer_score([4, 5], lp, [7, 8], SPECIAL, "forward")
    p = [float(torch.exp(torch.tensor(-0.1))), float(torch.exp(torch.tensor(-0.7)))]
    assert r["probs"] == p and r["score"] == (p[0] * p[1]) ** 0.5


def load_rollout_golden(golden_dir):
    """tests/golden/qwen_rollout_tiny.pt (tools/make_golden_qwen_rollout.py) with its weights regenerated from their seed."""
    blob = torch.load(os.path.join(golden_dir, "qwen_rollout_tiny.pt"), weights_only=False)
    cfg = qo.Qwen25VLConfig(**blob["config"])
    sd = qo.make_synthetic_state_dict(cfg, seed=blob["weights_seed"])
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().view(torch.uint8).numpy().tobytes())
    assert h.hexdigest() == blob["weights_sha256"], "synthetic weights differ from the ones the golden was generated with"
    return blob, cfg, sd


@pytest.mark.parametrize("case", ["pen1.0", "pen1.3_T0.7", "eos"])
def test_oracle_step_probabilities_match_committed_hf_golden(golden_dir, case):
    """Teacher-forced on HF's ids, the oracle's processed fp32 scores give HF's per-step p(s, answer id) = softmax(scores[s] / T)[id] and
    its top-5 (ids wherever the 5th and 6th probabilities are apart, probabilities everywhere), with the penalty over prompt and generated
    ids, T != 1 and an EOS stop; fp32 CPU sums in another order bound the difference."""
    blob, cfg, sd = load_rollout_golden(golden_dir)
    c = blob["cases"][case]
    inp, spg = golden_case_inputs(cfg, c)
    o = qg.qwen25vl_generate(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], blob["max_new_tokens"], (),
                             inp["image_of_sample"], repetition_penalty=c["penalty"], second_per_grid_ts=spg, forced=c["ids"])
    T = c["temperature"]
    if case == "eos":
        assert any(len(x) < blob["max_new_tokens"] and x[-1] in c["eos_ids"] for x in c["ids"])
    for b, ids in enumerate(c["ids"]):
        s = o["scores"][b]
        assert s.shape[0] == len(ids)
        probs = torch.softmax(s / T, dim=-1)
        p = probs[:, c["answer_ids"][b]]
        assert torch.allclose(p, c["p"][b], rtol=2e-4, atol=1e-7), (p, c["p"][b])
        top = torch.topk(probs, 6, dim=-1)
        assert torch.allclose(top.values[:, :5], c["top5_probs"][b], rtol=2e-4, atol=1e-7)
        apart = (top.values[:, 4] - top.values[:, 5]) > 1e-3 * top.values[:, 4]
        assert bool((top.indices[apart, :5].to(torch.int32) == c["top5_ids"][b][apart]).all())
        assert int(apart.sum()) >= len(ids) // 2

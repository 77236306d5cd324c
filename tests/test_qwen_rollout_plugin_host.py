"""Qwen2VLModel.forward(max_new_tokens > 1), CPU side: its refusals, and its wiring onto a scored rollout -- answer ids, EOS ids, chunking
and image subsets, the host rule -- with a stand-in engine (no GPU needed)."""
import types

import pytest
import torch

from oracle import qwen25vl_oracle as qo
from t2v_metrics_b200 import qwen_host
from test_qwen_host import TINY


class _NoImages:
    """A plugin stand-in whose image loading must never run."""

    def load_images(self, paths):
        raise AssertionError("images read: the call must be refused first")


@pytest.mark.parametrize("engine", [None, types.SimpleNamespace(score_prompts=lambda *a, **k: None)])
def test_rollout_scoring_without_a_rollout_engine_is_refused_before_any_work(engine):
    """max_new_tokens > 1 runs on the engine's scored decode loop: a plugin with no engine, or with an engine object that has no
    rollout_scores, refuses loudly before reading images; max_new_tokens < 1 is a ValueError."""
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    p = Qwen2VLModel.__new__(Qwen2VLModel)
    p.engine = engine
    p.load_images = _NoImages().load_images
    with pytest.raises(NotImplementedError, match="max_new_tokens=1"):
        p.forward(["a.png"], ["a dog"], max_new_tokens=4)
    with pytest.raises(NotImplementedError, match="max_new_tokens=1"):
        p.forward_with_trace(["a.png"], ["a dog"], max_new_tokens=4, score_position="start")
    with pytest.raises(ValueError, match="max_new_tokens"):
        Qwen2VLModel._rollout(p, ["a.png"], ["a dog"], "{}", "Yes", 0, 1.0, 1.0, "forward", 0)


class _Tok:
    eos_token_id, pad_token_id, bos_token_id = 639, 638, None

    def encode(self, s, add_special_tokens=False):
        return [ord(ch) % 500 for ch in s]

    def decode(self, ids, skip_special_tokens=False):
        return " ".join(str(int(i)) for i in ids if not (skip_special_tokens and int(i) >= 630))


class _RolloutEngine:
    """Records every rollout_scores call; the rollout of a prompt is `tokens_of(prompt)`, logp[s, j] = -(s + 1) * (j + 2) / 10."""

    def __init__(self, tokens_of, bytes_per_pair=0):
        self.calls, self.tokens_of, self.bytes_per_pair = [], tokens_of, bytes_per_pair

    def generate_workspace_bytes(self, batch, seq_len, n_patches, max_new_tokens):
        return batch * self.bytes_per_pair

    def rollout_scores(self, pixel_patches, grid_thw, prompts, answer_ids, max_new_tokens, eos_ids, temperature=1.0, repetition_penalty=1.0,
                       top_k=0, image_of_sample=None):
        self.calls.append(dict(pixels=pixel_patches.clone(), grids=list(grid_thw), prompts=prompts, answers=answer_ids, k=max_new_tokens,
                               eos=list(eos_ids), T=temperature, pen=repetition_penalty, top_k=top_k, img=list(image_of_sample)))
        B, n_max = len(prompts), max(len(a) for a in answer_ids)
        toks = [self.tokens_of(p)[:max_new_tokens] for p in prompts]
        s = torch.arange(max_new_tokens, dtype=torch.float32)[:, None] + 1
        j = torch.arange(n_max, dtype=torch.float32)[None, :] + 2
        logp = (-(s * j) / 10).expand(B, -1, -1).clone()
        out = dict(tokens=toks, lengths=torch.tensor([len(t) for t in toks]), logp=logp, topk_ids=None, topk_probs=None)
        if top_k:
            out["topk_ids"] = torch.arange(top_k, dtype=torch.int32).expand(B, max_new_tokens, -1).clone()
            out["topk_probs"] = torch.full((B, max_new_tokens, top_k), 0.125)
        return out


def _plugin(engine, grids):
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    p = Qwen2VLModel.__new__(Qwen2VLModel)
    p.engine, p.tokenizer, p.cfg, p.repetition_penalty = engine, _Tok(), qo.Qwen25VLConfig.tiny(**TINY), 1.1
    p.model_name, p._checkpoint = "qwen2.5-vl-7b", "/nonexistent/model.safetensors"
    # image g: grids[g] patch rows, every value g (so the patches a chunk receives name their images)
    p.load_images = lambda paths: (torch.cat([torch.full((t * h * w, 4), float(int(x[3:-4])))
                                              for x, (t, h, w) in zip(paths, (grids[int(x[3:-4])] for x in paths))]),
                                   [grids[int(x[3:-4])] for x in paths])
    return p


@pytest.mark.parametrize("max_pairs,budget,chunks", [(32, 1 << 40, [[0, 1, 2]]), (2, 1 << 40, [[0, 1], [2]]), (32, 1500, [[0], [1], [2]])])
def test_forward_with_max_new_tokens_runs_chunked_scored_rollouts(max_pairs, budget, chunks):
    grids = [(1, 4, 4), (1, 4, 6), (1, 6, 4)]
    eng = _RolloutEngine(lambda p: [len(p) % 7 + 1, 2, 3, 639], bytes_per_pair=1000)
    p = _plugin(eng, grids)
    p.ROLLOUT_MAX_PAIRS, p.ROLLOUT_WORKSPACE_BUDGET = max_pairs, budget
    images, texts = ["img2.png", "img0.png", "img2.png"], ["a cat", "dogs", "a hat"]
    out = p.forward(images, texts, question_template="Q {}", answer_template="Yes {}", max_new_tokens=6, temperature=0.5)
    assert out.dtype == torch.float32 and out.shape == (3,)
    assert [len(c["prompts"]) for c in eng.calls] == [len(c) for c in chunks]
    want = []
    for c, pairs in zip(eng.calls, chunks):
        assert c["k"] == 6 and c["eos"] == [639] and c["T"] == 0.5 and c["pen"] == 1.1 and c["top_k"] == 0
        assert len(c["grids"]) == len({images[i] for i in pairs})                      # each chunk gets the images it uses, once
        for b, i in enumerate(pairs):
            assert c["answers"][b] == _Tok().encode("Yes " + texts[i])                  # the whole answer, every token
            g = c["img"][b]
            assert float(c["pixels"][sum(t * h * w for t, h, w in c["grids"][:g]), 0]) == float(images[i][3:-4])   # its own image's rows
            lp = torch.tensor([[-(s + 1) * (j + 2) / 10 for j in range(len(c["answers"][b]))] for s in range(6)])
            want.append(qwen_host.rollout_answer_score(eng.tokens_of(c["prompts"][b])[:6], lp, c["answers"][b], {639, 638}, "forward")["score"])
    assert out.tolist() == torch.tensor(want, dtype=torch.float32).tolist()


def test_trace_with_max_new_tokens_has_the_reference_schema():
    grids = [(1, 4, 4)]
    eng = _RolloutEngine(lambda p: [5, 6, 7, 8, 639])
    p = _plugin(eng, grids)
    probs, traces = p.forward_with_trace(["img0.png"], ["a cat"], answer_template="Yes", max_new_tokens=8, score_position="end")
    (tr,) = traces
    assert eng.calls[0]["top_k"] == 5
    assert set(tr) == {"generated_text", "generated_length", "score_position", "score_start_idx", "scored_indices", "scored_tokens_text",
                       "probability", "token_details"}
    # L = 5 with EOS last, n = 3 ("Yes"): start = 5 - 3 - 1 = 1, steps 1..3, the EOS step not scored
    assert tr["generated_length"] == 5 and tr["score_start_idx"] == 1 and tr["scored_indices"] == [1, 2, 3]
    assert tr["generated_text"] == "5 6 7 8" and tr["scored_tokens_text"] == "6 7 8" and tr["score_position"] == "end"
    det = tr["token_details"]
    assert [d["position"] for d in det] == [1, 2, 3] and [d["expected_token_id"] for d in det] == _Tok().encode("Yes")
    assert [d["top_alternatives"][0] for d in det] == [dict(token_id=0, token_text="0", probability=0.125)] * 3
    assert float(probs[0]) == float(torch.tensor(tr["probability"], dtype=torch.float32))

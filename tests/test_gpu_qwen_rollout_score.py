"""Qwen2.5-VL scoring over a greedy rollout on a real H100: the per-step answer log-probability kernel against torch, the engine's scored
rollout against the teacher-forced CPU oracle, the committed HF golden and today's single-prefill scoring path, its launches and graphs,
the plugin's forward / forward_with_trace with max_new_tokens > 1, and HF bf16 generate(output_scores=True) at 7B width."""
import dataclasses
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import qwen25vl_oracle as qo
from test_gpu_qwen import TINY, make_engine
from test_gpu_qwen_generate import prompts_of, teacher_forced, decisive_prefix
from test_qwen_generate_host import golden_case_inputs
from test_qwen_rollout_score_host import load_rollout_golden
from t2v_metrics_b200 import qwen_host


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


def processed_torch(logits_bf16, bitmap_rows, penalty, temperature):
    """fp32 scores of the scoring path: bf16 -> fp32 -> penalty on the ids of each row's bitmap -> * (1/T in fp32)."""
    x = logits_bf16.float().clone()
    for b, ids in enumerate(bitmap_rows):
        if ids is not None and len(ids):
            v = x[b, ids]
            x[b, ids] = torch.where(v < 0, v * penalty, v / penalty)
    return x * torch.tensor(1.0 / temperature, dtype=torch.float32)


@pytest.mark.parametrize("V", [152064, 1001])
@pytest.mark.parametrize("pen", [1.0, 1.3])
@pytest.mark.parametrize("T", [0.5, 1.0, 2.0])
def test_answer_logprob_kernel_matches_torch(dev, V, pen, T):
    """log_softmax over the whole vocabulary at the answer ids, and the top-5 with tied logits ordered lower id first (a stable descending
    sort: what topk_softmax_kernel does, and torch.topk's values). A finished row and the entries past a row's answer count stay
    untouched."""
    from t2v_metrics_b200.engine import ops
    B, max_new, n_max, K = 4, 3, 5, 5
    g = torch.Generator().manual_seed(V + int(T * 10) + int(pen * 10))
    logits = (torch.randn(B, V, generator=g) * 4).to(torch.bfloat16)
    tied = [7, 100, 500]
    logits[1, tied] = logits[1].float().max().to(torch.bfloat16) + 1          # three ids share the row's top score
    words = (V + 31) // 32
    pen_ids = [torch.randperm(V, generator=g)[:200] for _ in range(B)]
    pen_ids[1] = pen_ids[1][~torch.isin(pen_ids[1], torch.tensor(tied))]
    answers = torch.randint(0, V, (B, n_max), generator=g)
    answers[0, 1] = int(pen_ids[0][0])                                          # a penalised answer id
    answers[1, 0] = tied[1]
    counts = torch.tensor([5, 2, 3, 0], dtype=torch.int32)
    lengths = torch.tensor([0, 2, 1, 1], dtype=torch.int32)
    done = torch.tensor([0, 0, 1, 0], dtype=torch.int32)
    bitmap = None
    if pen != 1.0:
        bm = torch.zeros(B, words * 32, dtype=torch.int64)
        for b in range(B):
            bm[b, pen_ids[b]] = 1
        bits = (bm.view(B, words, 32) << torch.arange(32)).sum(-1)                # bit n & 31 of word n >> 5
        bitmap = torch.where(bits >= 2 ** 31, bits - 2 ** 32, bits).to(torch.int32).to(dev)
    i32 = lambda t: t.to(torch.int32).to(dev)
    logp, ids, probs = ops.answer_logprob(logits.to(dev), i32(answers), i32(counts), i32(lengths), i32(done), max_new, temperature=T,
                                          penalty_bitmap=bitmap, repetition_penalty=pen, top_k=K)
    torch.cuda.synchronize()
    logp, ids, probs = logp.cpu(), ids.cpu(), probs.cpu()
    x = processed_torch(logits, pen_ids if pen != 1.0 else [None] * B, pen, T)
    ref = torch.log_softmax(x, dim=-1)
    for b in range(B):
        t = int(lengths[b])
        untouched = [s for s in range(max_new) if s != t or done[b]]
        assert bool(logp[b, untouched].isnan().all()) and bool((ids[b, untouched] == -1).all())
        if done[b]:
            continue
        c = int(counts[b])
        assert bool(logp[b, t, c:].isnan().all())
        want = ref[b, answers[b, :c]]
        # relative error of the sum of exps: fp32 rounding along the kernel's addition chain (ceil(V / 256) terms per thread, then a
        # 5-level warp tree and 8 warps; torch's own chain is shorter) and the __expf approximation
        rel = (math.ceil(V / 256) + 64) * 2.0 ** -24 + 2.0 ** -18
        tol = rel + 2.0 ** -22 * float(want.abs().max() if c else 0)
        assert float((logp[b, t, :c] - want).abs().max() if c else 0) <= tol, (b, logp[b, t, :c], want)
        order = torch.sort(x[b], descending=True, stable=True).indices[:K]
        assert ids[b, t].tolist() == order.tolist(), (b, ids[b, t], order)
        tv = torch.topk(torch.softmax(x[b], -1), K)
        assert torch.allclose(probs[b, t], tv.values, rtol=2 * rel, atol=0), (probs[b, t], tv.values)
        if b == 1:
            assert ids[b, t, :3].tolist() == tied and set(tv.indices[:3].tolist()) == set(tied)


def run_rollout(eng, inp, case, blob, answers, spg=None, top_k=5, **kw):
    return eng.rollout_scores(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), answers, blob["max_new_tokens"], case["eos_ids"],
                              temperature=case["temperature"], repetition_penalty=case["penalty"], top_k=top_k,
                              image_of_sample=inp["image_of_sample"], second_per_grid_ts=spg, **kw)


@pytest.mark.parametrize("case", ["pen1.0", "pen1.3_T0.7", "eos"])
def test_rollout_tokens_equal_generate_tokens(golden_dir, dev, case):
    """The scoring hook reads the step's logits and writes only its own outputs: the tokens are generate_prompts' tokens, bit for bit."""
    blob, cfg, sd = load_rollout_golden(golden_dir)
    c = blob["cases"][case]
    inp, spg = golden_case_inputs(cfg, c)
    eng = make_engine(cfg, sd, dev)
    toks = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), blob["max_new_tokens"], c["eos_ids"],
                                image_of_sample=inp["image_of_sample"], repetition_penalty=c["penalty"], second_per_grid_ts=spg)
    r = run_rollout(eng, inp, c, blob, c["answer_ids"], spg)
    assert r["tokens"] == toks
    assert r["lengths"].tolist() == [len(t) for t in toks]


def oracle_logp(s, answers, T):
    return torch.log_softmax(s / T, dim=-1)[:, answers]


def logp_gap(s16, s32, T):
    """Per step, a bound on the oracle's bf16-vs-fp32 log-probability gap: a log-probability is a score / T minus the log-sum-exp, which
    moves by at most the largest score / T change, so twice the step's largest processed-score gap / T (the generate tests bound tokens
    by the same per-step largest gap)."""
    return 2.0 * (s16 - s32).abs().amax(-1) / T


@pytest.mark.parametrize("video,pen,T", [(False, 1.3, 0.7), (False, 1.0, 1.0), (True, 1.3, 2.0)])
def test_rollout_logprobs_match_the_oracle_on_its_own_path(dev, video, pen, T):
    """Teacher-forced on the engine's own tokens, every step's answer log-probabilities are within 2x the oracle's bf16-vs-fp32 log-prob
    gap at that step of the fp32 oracle's (the bound the generate tests put on tokens)."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=21)
    inp = qo.make_synthetic_inputs(cfg, 3, (56, 84) if video else (84, 56), 12, seed=22, ragged=True, frames=2 if video else 1)
    spg = [2.0] * 3 if video else None
    answers = [[5, 17, 300], [42], [9, 9]]
    eng = make_engine(cfg, sd, dev)
    r = eng.rollout_scores(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), answers, 10, (), temperature=T, repetition_penalty=pen,
                           second_per_grid_ts=spg)
    s32, s16 = teacher_forced(sd, cfg, inp, r["tokens"], pen, spg)
    for b in range(3):
        L = len(r["tokens"][b])
        o32 = oracle_logp(s32[b], answers[b], T)
        got = r["logp"][b, :L, :len(answers[b])]
        gap = logp_gap(s16[b], s32[b], T)[:, None]
        err = (got - o32).abs()
        print(f"\n[rollout self-consistency video={video} pen={pen} T={T}] b={b} max err {float(err.max()):.3e} max gap {float(gap.max()):.3e}")
        assert bool((err <= 2.0 * gap + 1e-3).all()), (err, gap)
        assert bool(r["logp"][b, L:].isnan().all())


@pytest.mark.parametrize("case", ["pen1.0", "pen1.3_T0.7", "eos"])
def test_rollout_matches_committed_hf_golden(golden_dir, dev, case):
    """Against HF generate(output_scores=True) in fp32: on the steps before the first near-tie of HF's path (the decisive-prefix rule of
    the generate tests), the tokens are HF's and each answer log-probability is within 2x the oracle's bf16-vs-fp32 gap (+ 1e-3) of
    log softmax(HF scores / T); the top-1 of the step is HF's token."""
    blob, cfg, sd = load_rollout_golden(golden_dir)
    c = blob["cases"][case]
    inp, spg = golden_case_inputs(cfg, c)
    eng = make_engine(cfg, sd, dev)
    r = run_rollout(eng, inp, c, blob, c["answer_ids"], spg)
    s32, s16 = teacher_forced(sd, cfg, inp, c["ids"], c["penalty"], spg)
    compared = 0
    for b, hf_ids in enumerate(c["ids"]):
        thr = 2.0 * (s16[b] - s32[b]).abs().amax(-1) + 1e-3
        n = decisive_prefix(c["margins"][b] - thr, 0.0)
        assert r["tokens"][b][:n] == hf_ids[:n]
        ans = c["answer_ids"][b]
        gap = logp_gap(s16[b], s32[b], c["temperature"])[:n, None]
        hf = torch.log(c["p"][b][:n].double()).float()
        err = (r["logp"][b, :n, :len(ans)] - hf).abs()
        print(f"\n[rollout golden {case}] b={b} decisive steps {n} max err {float(err.max()) if n else 0:.3e}")
        assert bool((err <= 2.0 * gap + 1e-3).all()), (err, gap)
        assert r["topk_ids"][b, :n, 0].tolist() == hf_ids[:n]
        compared += n
    assert compared >= 8


@pytest.mark.parametrize("pen,T", [(1.0, 1.0), (1.3, 0.7)])
def test_rollout_step0_equals_the_single_prefill_scoring_path(dev, pen, T):
    """Step 0 of a rollout and score_tensors (the padded prefill of score_prompts(share_prefix=False)) run the same prefill and the same
    lm_head tile loop, so the bf16 logits, the processed scores and their maximum are the same numbers. Only the sum of exps differs: the
    scoring path sums 128-column tiles in its GEMM epilogue and combines them, the kernel sums per thread with __expf. The bound is that
    arithmetic: fp32 rounding along both addition chains plus the exp approximations."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=23)
    inp = qo.make_synthetic_inputs(cfg, 4, (84, 56), 12, seed=24, ragged=True, n_images=2)
    eng = make_engine(cfg, sd, dev)
    prompts = prompts_of(inp)
    answers = [int(a) for a in inp["answer_ids"]]
    r = eng.rollout_scores(inp["pixel_patches"], inp["grid_thw"], prompts, [[a] for a in answers], 3, (), temperature=T,
                           repetition_penalty=pen, image_of_sample=inp["image_of_sample"])
    idx = qwen_host.build_batch_indices(prompts, inp["grid_thw"], inp["image_of_sample"], cfg.image_token_id, cfg.spatial_merge_size,
                                        cfg.tokens_per_second, video_token_id=cfg.video_token_id)
    d = {k: v.to(dev) for k, v in idx.items()}
    _, ref = eng.score_tensors(inp["pixel_patches"].to(dev), inp["grid_thw"], d["input_ids"], d["seq_lens"], d["feat_index"], d["position_ids"],
                               torch.tensor(answers, dtype=torch.int32, device=dev), T, return_logprobs=True, repetition_penalty=pen)
    ref = ref.cpu()
    got = r["logp"][:, 0, 0]
    tol = (math.ceil(cfg.vocab / 256) + 128 + 64) * 2.0 ** -24 + 2.0 ** -18 + 2.0 ** -22 * float(ref.abs().max())
    print(f"\n[rollout step 0 pen={pen} T={T}] max |diff| {float((got - ref).abs().max()):.3e} bound {tol:.3e}")
    assert float((got - ref).abs().max()) <= tol, (got, ref)


@pytest.mark.parametrize("pen,top_k", [(1.0, 0), (1.3, 5)])
def test_rollout_launch_counts_graphs_and_scoring_after(dev, pen, top_k):
    """The scored prefill and step enqueue what last_launch_count() reports (the nodes of a captured graph), one launch more than the plain
    generate prefill and step, whose counts are unchanged by a rollout; graph replay equals direct steps; scoring after a rollout is
    bit-identical."""
    from test_gpu_clipt5 import captured_node_count
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=25)
    inp = qo.make_synthetic_inputs(cfg, 3, (84, 56), 12, seed=26, ragged=True, n_images=2)
    fresh = make_engine(cfg, sd, dev)
    ref = fresh.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), inp["answer_ids"], inp["image_of_sample"],
                              repetition_penalty=pen).cpu()
    eng = make_engine(cfg, sd, dev)
    args = (inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), 10, (5,))
    kw = dict(image_of_sample=inp["image_of_sample"], repetition_penalty=pen)
    answers = [[1, 2, 3], [4], [5, 6]]
    plain = eng.generate_begin(*args, **kw)
    plain_prefill = captured_node_count(plain["prefill"])
    plain_step = captured_node_count(lambda: eng.generate_step(plain))
    assert plain_step == eng.last_launch_count()
    st = eng.generate_begin(*args, **kw, score=dict(answer_ids=answers, temperature=0.8, top_k=top_k))
    assert captured_node_count(st["prefill"]) == eng.last_launch_count() == plain_prefill + 1
    st["prefill"]()
    assert captured_node_count(lambda: eng.generate_step(st)) == eng.last_launch_count() == plain_step + 1
    print(f"\n[rollout launches pen={pen}] prefill {plain_prefill} + 1, step {plain_step} + 1")
    rk = dict(temperature=0.8, repetition_penalty=pen, top_k=top_k, image_of_sample=inp["image_of_sample"])
    graphed = eng.rollout_scores(*args[:3], answers, *args[3:], **rk, use_graph=True)
    graphed2 = eng.rollout_scores(*args[:3], answers, *args[3:], **rk, use_graph=True)
    direct = eng.rollout_scores(*args[:3], answers, *args[3:], **rk, use_graph=False)
    for other in (graphed2, direct):
        assert other["tokens"] == graphed["tokens"]
        assert torch.equal(other["logp"].nan_to_num(7.0), graphed["logp"].nan_to_num(7.0))
        if top_k:
            assert torch.equal(other["topk_ids"], graphed["topk_ids"]) and torch.equal(other["topk_probs"].nan_to_num(7.0),
                                                                                       graphed["topk_probs"].nan_to_num(7.0))
    assert captured_node_count(lambda: eng.generate_step(plain)) == plain_step
    got = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), inp["answer_ids"], inp["image_of_sample"],
                            repetition_penalty=pen).cpu()
    assert torch.equal(got, ref)


class _ChatTokenizer:
    """Stand-in tokenizer: characters -> code points (mod 500); ids >= 630 are special (eos 639, pad 638) and dropped by
    skip_special_tokens."""
    pad_token_id = 638
    bos_token_id = None

    def __init__(self, eos=639):
        self.eos_token_id = eos

    def encode(self, s, add_special_tokens=False):
        return [ord(ch) % 500 for ch in s]

    def decode(self, ids, skip_special_tokens=False):
        special = {self.eos_token_id, self.pad_token_id}
        return " ".join(str(int(i)) for i in ids if not (skip_special_tokens and (int(i) >= 630 or int(i) in special)))


@pytest.fixture(scope="module")
def plugin(dev, tmp_path_factory):
    import numpy as np
    from PIL import Image
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    ocfg = qo.Qwen25VLConfig.tiny(**TINY)
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    cfg = Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(ocfg).items() if k in fields})
    sd = qo.make_synthetic_state_dict(ocfg, seed=27)
    d = tmp_path_factory.mktemp("rollout_images")
    rng = np.random.default_rng(1)
    paths = []
    for i, (h, w) in enumerate(((60, 90), (84, 56))):
        p = d / f"{i}.png"
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(p)
        paths.append(str(p))
    model = Qwen2VLModel("qwen2.5-vl-7b", device=str(dev), tokenizer=_ChatTokenizer(), state_dict=dict(sd), config=cfg,
                         checkpoint=str(d / "none.bin"), min_pixels=56 * 56, max_pixels=112 * 112, repetition_penalty=1.2)
    return model, paths


def _engine_side(model, paths, images, texts, qt, at, k, T, mode, top_k=0):
    from t2v_metrics_b200.models.vqascore_models.qwen_utils import build_prompt_ids
    tok = model.tokenizer
    patches, grids = model.load_images(paths)
    which = [paths.index(p) for p in images]
    prompts = [build_prompt_ids(tok, qt.format(t), grids[i][1] * grids[i][2] // 4, model.cfg.image_token_id) for t, i in zip(texts, which)]
    answers = [tok.encode(at.format(t)) for t in texts]
    r = model.engine.rollout_scores(patches, grids, prompts, answers, k, [tok.eos_token_id], temperature=T,
                                    repetition_penalty=model.repetition_penalty, top_k=top_k, image_of_sample=which)
    special = {tok.eos_token_id, tok.pad_token_id}
    return r, [qwen_host.rollout_answer_score(r["tokens"][b], r["logp"][b], answers[b], special, mode) for b in range(len(texts))], answers


def test_plugin_forward_and_trace_follow_the_host_rule_on_the_engine_rollout(plugin):
    model, paths = plugin
    images, texts = [paths[0], paths[1], paths[0]], ["a red car", "two dogs", "a blue sky"]
    qt, at = 'Does this figure show "{}"?', "Yes, it does"
    out = model.forward(images, texts, question_template=qt, answer_template=at, max_new_tokens=6, temperature=0.9)
    assert out.dtype == torch.float32 and out.shape == (3,) and out.device.type == "cpu"
    _, want, answers = _engine_side(model, paths, images, texts, qt, at, 6, 0.9, "forward")
    assert all(len(a) > 1 for a in answers)                       # multi-token answers: the geometric mean of their probabilities
    for b, w in enumerate(want):
        assert float(out[b]) == float(torch.tensor(w["score"], dtype=torch.float32))
        assert math.isclose(w["score"], math.prod(w["probs"]) ** (1 / w["n"]), rel_tol=1e-12)
    keys = {"generated_text", "generated_length", "score_position", "score_start_idx", "scored_indices", "scored_tokens_text", "probability",
            "token_details"}
    for pos in ("start", "end"):
        probs, traces = model.forward_with_trace(images, texts, question_template=qt, answer_template=at, max_new_tokens=6, temperature=0.9,
                                                 score_position=pos)
        r, want, answers = _engine_side(model, paths, images, texts, qt, at, 6, 0.9, pos, top_k=5)
        assert probs.tolist() == torch.tensor([w["score"] for w in want], dtype=torch.float32).tolist()
        for b, (tr, w) in enumerate(zip(traces, want)):
            assert set(tr) == keys
            toks = r["tokens"][b]
            assert tr["generated_length"] == len(toks) and tr["score_start_idx"] == w["start"] and tr["scored_indices"] == w["steps"]
            assert tr["generated_text"] == model.tokenizer.decode(toks, skip_special_tokens=True)
            assert tr["probability"] == w["score"] and len(tr["token_details"]) == w["n"]
            for i, det in enumerate(tr["token_details"]):
                assert set(det) == {"position", "expected_token_id", "expected_token_text", "probability", "top_alternatives"}
                assert det["position"] == w["steps"][i] and det["expected_token_id"] == answers[b][i] and det["probability"] == w["probs"][i]
                assert [a["token_id"] for a in det["top_alternatives"]] == r["topk_ids"][b, w["steps"][i]].tolist()
                assert len(det["top_alternatives"]) == 5


def test_plugin_rollout_value_errors_and_max_new_tokens_1_unchanged(plugin):
    """A tokenizer whose eos id is the first greedy token of every prompt ends each rollout after one token: forward and "end" raise the
    reference's messages, "start" scores step 0. max_new_tokens=1 keeps the single-prefill path: bit-identical before and after rollouts."""
    model, paths = plugin
    images, texts = [paths[0], paths[1]], ["a red car", "two dogs"]
    before = model.forward(images, texts)
    tok = model.tokenizer
    r, _, _ = _engine_side(model, paths, images[:1], texts[:1], 'Does this figure show "{}"? Please answer Yes or No.', "Yes", 4, 1.0,
                           "start")
    first = r["tokens"][0][0]
    try:
        model.tokenizer = _ChatTokenizer(eos=first)
        with pytest.raises(ValueError, match="No content tokens to score after removing special tokens"):
            model.forward(images[:1], texts[:1], max_new_tokens=4)
        with pytest.raises(ValueError, match="No tokens available to score at the specified position"):
            model.forward_with_trace(images[:1], texts[:1], max_new_tokens=4, score_position="end")
        probs, traces = model.forward_with_trace(images[:1], texts[:1], max_new_tokens=4, score_position="start")
        assert traces[0]["generated_length"] == 1 and traces[0]["scored_indices"] == [0]
    finally:
        model.tokenizer = tok
    after = model.forward(images, texts)
    assert torch.equal(before, after)


def test_qwen25vl_7b_rollout_logprobs_match_reference_bf16_on_this_gpu(dev):
    """Qwen2.5-VL-7B width, B = 2, 448x448 images + 32 text ids, 16 new tokens: answer log-probabilities of the engine's scored rollout
    against log softmax of HF bf16 sdpa generate(output_scores=True) per sample on the same GPU and weights, at every step conditioned on a
    path the two share. Random weights give probabilities near 1 / vocab, so log-probabilities are compared. Both sides take bf16 logits of
    magnitude ~10, whose rounding step is 1/16; the generate test bounds the engine's chosen token within 0.25 of HF's best processed score
    for the same reason. A log-probability is its logit minus the log-sum-exp, which moves by at most the largest logit change: with 0.25
    for each, the bound is 0.5."""
    import gc
    import hf_reference as hf
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.engine import QwenVLEngine
    cfg = qo.Qwen25VLConfig.qwen25_vl_7b()
    B, N = 2, 16
    sd = qo.make_synthetic_state_dict(cfg, seed=0, gen_device=dev)
    inp = qo.make_synthetic_inputs(cfg, B, (448, 448), 32, seed=1, ragged=True)
    answers = [[9454, 11, 432, 1558], [2753]]
    model = hf.build_hf_qwen(cfg, sd, dtype=torch.bfloat16, device=dev, attn="sdpa")
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    ref_ids, ref_logp = [], []
    with torch.no_grad():
        for b, ids in enumerate(inp["input_ids"]):
            ids = ids.to(dev)
            out = model.generate(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long, device=dev),
                                 pixel_values=inp["pixel_patches"][b * P:(b + 1) * P].to(dev, torch.bfloat16),
                                 image_grid_thw=torch.tensor([list(inp["grid_thw"][b])], device=dev),
                                 mm_token_type_ids=(ids == cfg.image_token_id).long()[None], max_new_tokens=N, min_new_tokens=N,
                                 do_sample=False, eos_token_id=None, pad_token_id=0, output_scores=True, return_dict_in_generate=True)
            ref_ids.append(out.sequences[0, len(ids):].tolist())
            ref_logp.append(torch.stack([torch.log_softmax(s[0].float(), -1)[answers[b]] for s in out.scores]).cpu())
    del model
    gc.collect()
    torch.cuda.empty_cache()
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    eng = QwenVLEngine(Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(cfg).items() if k in fields}), dev)
    eng.load_state_dict(sd)
    r = eng.rollout_scores(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), answers, N, ())
    compared = 0
    for b in range(B):
        toks = r["tokens"][b]
        shared = next((t for t in range(N) if toks[t] != ref_ids[b][t]), N)
        steps = min(shared + 1, N)          # the steps conditioned on a common prefix, the first differing one included
        err = (r["logp"][b, :steps, :len(answers[b])] - ref_logp[b][:steps]).abs()
        print(f"\n[qwen-7b rollout] b={b} shared prefix {shared} max |logp diff| {float(err.max()):.3e}")
        assert float(err.max()) <= 0.5, (b, err)
        compared += steps
    del sd, eng
    gc.collect()
    torch.cuda.empty_cache()
    assert compared >= 4

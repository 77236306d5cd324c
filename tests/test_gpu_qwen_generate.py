"""Qwen2.5-VL greedy generation on a real H100: the engine's prefill + decode loop against the CPU generation oracle (teacher-forced on
the engine's own tokens), the committed HF golden, and HF bf16 generate at full width."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import qwen25vl_oracle as qo
from oracle import qwen25vl_generate as qg
from test_gpu_qwen import TINY, make_engine
from test_qwen_generate_host import load_generate_golden, golden_case_inputs


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


def prompts_of(inp):
    return [x.tolist() for x in inp["input_ids"]]


def teacher_forced(sd, cfg, inp, tokens, pen, spg=None):
    """Processed scores of every step on the given token paths, fp32 and bf16 oracle, and their per-step gap."""
    args = (sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], max(len(t) for t in tokens), ())
    kw = dict(image_of_sample=inp["image_of_sample"], repetition_penalty=pen, second_per_grid_ts=spg, forced=tokens)
    s32 = qg.qwen25vl_generate(*args, mode="fp32", **kw)["scores"]
    s16 = qg.qwen25vl_generate(*args, mode="bf16", **kw)["scores"]
    return s32, s16


def decisive_prefix(margins, thr):
    """Number of leading steps whose top-1 / top-2 margin is at least thr (beyond them a near-tie may send two paths apart)."""
    n = 0
    for m in margins:
        if float(m) < thr:
            break
        n += 1
    return n


@pytest.mark.parametrize("video,pen", [(False, 1.0), (False, 1.3), (True, 1.3)])
def test_engine_tokens_are_the_oracles_argmax_on_its_own_path(dev, video, pen):
    """Self-consistency: teacher-forced on the engine's own tokens, every one of them is within 2x the oracle's bf16-vs-fp32 score gap of
    the fp32 arg-max at its step. Every step is checked, so a near-tie that sends the engine and the oracle apart cannot skip steps."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=11)
    inp = qo.make_synthetic_inputs(cfg, 3, (56, 84) if video else (84, 56), 12, seed=12, ragged=True, frames=2 if video else 1)
    spg = [2.0] * 3 if video else None
    eng = make_engine(cfg, sd, dev)
    toks = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), 12, (), repetition_penalty=pen, second_per_grid_ts=spg)
    assert [len(t) for t in toks] == [12] * 3
    s32, s16 = teacher_forced(sd, cfg, inp, toks, pen, spg)
    for b in range(3):
        gap = (s16[b] - s32[b]).abs().amax(-1)
        chosen = s32[b].gather(-1, torch.tensor(toks[b])[:, None])[:, 0]
        short = s32[b].amax(-1) - chosen
        print(f"\n[generate self-consistency video={video} pen={pen}] b={b} tokens {toks[b]} max shortfall {float(short.max()):.3e} "
              f"max bf16 gap {float(gap.max()):.3e}")
        assert bool((short <= 2.0 * gap + 1e-3).all()), (short, gap)


@pytest.mark.parametrize("case", ["images_pen1.0", "images_pen1.3", "video_pen1.0", "video_pen1.3", "eos"])
def test_engine_matches_committed_hf_generate_golden(golden_dir, dev, case):
    """Against HF generate(do_sample=False) in fp32: ids equal up to the first step whose HF top-1 / top-2 margin is below 2x the oracle's
    bf16-vs-fp32 score gap at that step on the HF path; at least 8 steps per case are compared."""
    blob, cfg, sd = load_generate_golden(golden_dir)
    c = blob["cases"][case]
    inp, spg = golden_case_inputs(cfg, c)
    eng = make_engine(cfg, sd, dev)
    toks = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), blob["max_new_tokens"], c["eos_ids"],
                                image_of_sample=inp["image_of_sample"], repetition_penalty=c["penalty"], second_per_grid_ts=spg)
    s32, s16 = teacher_forced(sd, cfg, inp, c["ids"], c["penalty"], spg)
    compared = 0
    for b, hf_ids in enumerate(c["ids"]):
        thr = 2.0 * (s16[b] - s32[b]).abs().amax(-1) + 1e-3
        n = decisive_prefix(c["margins"][b] - thr, 0.0)
        print(f"\n[generate golden {case}] b={b} engine {toks[b]}\n    HF {hf_ids} decisive steps {n} (threshold <= {float(thr.max()):.3e})")
        assert toks[b][:n] == hf_ids[:n]
        if n == len(hf_ids):
            assert toks[b] == hf_ids          # the same length too: EOS and max_new_tokens stops
        compared += n
    assert compared >= 8


def test_repetition_penalty_covers_generated_ids(golden_dir, dev):
    """Penalty 1.3 on prompts whose unpenalised greedy path repeats tokens it generated itself. On the engine's path, teacher-forced raw
    oracle scores penalised over prompt + generated ids must put every engine token within tolerance of the arg-max, and at some step a
    penalty over the prompt ids alone would have preferred another token decisively: only generated ids entering the bitmap explain the
    engine's path."""
    blob, cfg, sd = load_generate_golden(golden_dir)
    c0 = blob["cases"]["images_pen1.0"]
    inp, _ = golden_case_inputs(cfg, c0)
    assert any(len(set(x)) < len(x) for x in c0["ids"])          # the unpenalised path repeats generated tokens
    eng = make_engine(cfg, sd, dev)
    toks = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), blob["max_new_tokens"], (),
                                image_of_sample=inp["image_of_sample"], repetition_penalty=1.3)
    r32, r16 = teacher_forced(sd, cfg, inp, toks, 1.0)            # raw fp32 scores on the engine's path
    decisive_prompt_only = 0
    for b, path in enumerate(toks):
        prompt = inp["input_ids"][b].long()
        for t, tok in enumerate(path):
            tol = 2.6 * float((r16[b][t] - r32[b][t]).abs().max()) + 1e-3
            full = qg.process_logits(r32[b][t], torch.cat([prompt, torch.tensor(path[:t], dtype=torch.long)]), 1.3)
            only = qg.process_logits(r32[b][t], prompt, 1.3)
            assert float(full.max() - full[tok]) <= tol, (b, t)
            decisive_prompt_only += float(only.max() - only[tok]) > tol
    print(f"\n[generate penalty] engine {toks}; steps where a prompt-only penalty would pick another token: {decisive_prompt_only}")
    assert decisive_prompt_only >= 1


def test_eos_ragged_prompts_and_batch_invariance(golden_dir, dev):
    """Sequences stop independently on an EOS id, nothing is emitted after it (-1), lengths are right, and each prompt generated on its own
    gives the batch's tokens on its decisive steps."""
    blob, cfg, sd = load_generate_golden(golden_dir)
    c = blob["cases"]["eos"]
    inp, _ = golden_case_inputs(cfg, c)
    eng = make_engine(cfg, sd, dev)
    prompts, N = prompts_of(inp), blob["max_new_tokens"]
    st = eng.generate_begin(inp["pixel_patches"], inp["grid_thw"], prompts, N, c["eos_ids"], image_of_sample=inp["image_of_sample"])
    for _ in range(N - 1):
        eng.generate_step(st)
    tokens, lengths = st["tokens"].cpu(), st["lengths"].cpu()
    assert int(st["all_done"].cpu()[0]) == 1
    batch = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, N, c["eos_ids"], image_of_sample=inp["image_of_sample"])
    eos = set(c["eos_ids"])
    for b in range(len(prompts)):
        n = int(lengths[b])
        assert tokens[b, :n].tolist() == batch[b]
        assert bool((tokens[b, n:] == -1).all())
        assert n == N or batch[b][-1] in eos
        assert not any(t in eos for t in batch[b][:-1])
    assert any(len(x) < N for x in batch) and any(len(x) == N for x in batch)     # one stops early, another runs to the limit
    s32, s16 = teacher_forced(sd, cfg, inp, batch, 1.0)
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    for b in range(len(prompts)):
        img = inp["image_of_sample"][b]
        one = eng.generate_prompts(inp["pixel_patches"][img * P:(img + 1) * P], [inp["grid_thw"][img]], [prompts[b]], N, c["eos_ids"])[0]
        top2 = s32[b].topk(2, dim=-1).values
        n = decisive_prefix(top2[:, 0] - top2[:, 1] - 2.0 * (s16[b] - s32[b]).abs().amax(-1) - 1e-3, 0.0)
        assert one[:n] == batch[b][:n]


@pytest.mark.parametrize("pen", [1.0, 1.3])
def test_generate_launch_counts_equal_captured_graph_nodes(dev, pen):
    """last_launch_count() of the generate prefill and of one decode step is what each enqueues (the nodes of a CUDA graph capturing it),
    and the graph-replayed decode loop gives the tokens of direct step calls."""
    from test_gpu_clipt5 import captured_node_count
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=13)
    inp = qo.make_synthetic_inputs(cfg, 3, (84, 56), 12, seed=14, ragged=True, n_images=2)
    eng = make_engine(cfg, sd, dev)
    args = (inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), 10, (5,))
    kw = dict(image_of_sample=inp["image_of_sample"], repetition_penalty=pen)
    st = eng.generate_begin(*args, **kw)
    assert captured_node_count(st["prefill"]) == eng.last_launch_count()
    n_prefill = eng.last_launch_count()
    st["prefill"]()
    assert captured_node_count(lambda: eng.generate_step(st)) == eng.last_launch_count()
    print(f"\n[generate launches pen={pen}] prefill {n_prefill}, step {eng.last_launch_count()}")
    graphed = eng.generate_prompts(*args, **kw, use_graph=True)
    graphed2 = eng.generate_prompts(*args, **kw, use_graph=True)          # replays the graph captured by the previous call
    direct = eng.generate_prompts(*args, **kw, use_graph=False)
    assert graphed == direct == graphed2


def test_scoring_after_generation_is_unchanged(dev):
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=15)
    inp = qo.make_synthetic_inputs(cfg, 3, (84, 56), 12, seed=16, ragged=True, n_images=2)
    fresh = make_engine(cfg, sd, dev)
    ref = fresh.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), inp["answer_ids"], inp["image_of_sample"],
                              repetition_penalty=1.3).cpu()
    eng = make_engine(cfg, sd, dev)
    eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), 8, (), image_of_sample=inp["image_of_sample"],
                         repetition_penalty=1.3)
    got = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), inp["answer_ids"], inp["image_of_sample"],
                            repetition_penalty=1.3).cpu()
    assert torch.equal(got, ref)


class _DigitTokenizer:
    """Stand-in tokenizer: characters -> code points (mod 500); ids 600+ (vision) and 630+ ("special") are dropped by decode."""
    eos_token_id = 639

    def encode(self, s, add_special_tokens=False):
        return [ord(ch) % 500 for ch in s]

    def decode(self, ids, skip_special_tokens=False, clean_up_tokenization_spaces=True):
        assert skip_special_tokens and clean_up_tokenization_spaces is False
        return " " + " ".join(str(i) for i in ids if not (skip_special_tokens and i >= 630)) + " "


def test_plugin_generate_returns_the_decoded_engine_ids(dev, tmp_path):
    import numpy as np
    from PIL import Image
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    ocfg = qo.Qwen25VLConfig.tiny(**TINY)
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    cfg = Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(ocfg).items() if k in fields})
    sd = qo.make_synthetic_state_dict(ocfg, seed=17)
    rng = np.random.default_rng(0)
    paths = []
    for i, (h, w) in enumerate(((60, 90), (84, 56))):
        p = tmp_path / f"{i}.png"
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(p)
        paths.append(str(p))
    tok = _DigitTokenizer()
    model = Qwen2VLModel("qwen2.5-vl-7b", device=str(dev), tokenizer=tok, state_dict=dict(sd), config=cfg, checkpoint=str(tmp_path / "none.bin"),
                         min_pixels=56 * 56, max_pixels=112 * 112)
    images, texts = [paths[0], paths[1], paths[0]], ["a red car", "two dogs", "a blue sky"]
    out = model.generate(images=images, texts=texts, max_new_tokens=6)
    assert isinstance(out, list) and len(out) == 3 and all(isinstance(s, str) for s in out)
    patches, grids = model.load_images(paths)
    from t2v_metrics_b200.models.vqascore_models.qwen_utils import build_prompt_ids
    prompts = [build_prompt_ids(tok, t, grids[i][1] * grids[i][2] // 4, cfg.image_token_id) for t, i in zip(texts, (0, 1, 0))]
    ids = model.engine.generate_prompts(patches, grids, prompts, 6, [639], image_of_sample=[0, 1, 0], repetition_penalty=1.0)
    assert out == [tok.decode(x, skip_special_tokens=True, clean_up_tokenization_spaces=False).strip() for x in ids]
    assert all(len(s) > 0 for s in out)


def test_qwen25vl_7b_generate_matches_reference_bf16_on_this_gpu(dev):
    """Qwen2.5-VL-7B width, B = 2, 448x448 images + 32 text ids, 16 new tokens: the engine's decode loop against HF bf16 sdpa
    generate(do_sample=False) per sample on the same GPU and weights. Random weights give flat logits (top-1 / top-2 margins of 0 to 0.3,
    where bf16 logits of magnitude ~10 are rounded to 1/16), so near-ties are frequent: at every step where the engine's path still equals
    HF's, the engine's token must score within 0.25 of HF's best processed score at that step."""
    import gc
    import hf_reference as hf
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.engine import QwenVLEngine
    cfg = qo.Qwen25VLConfig.qwen25_vl_7b()
    B, N = 2, 16
    sd = qo.make_synthetic_state_dict(cfg, seed=0, gen_device=dev)
    inp = qo.make_synthetic_inputs(cfg, B, (448, 448), 32, seed=1, ragged=True)
    model = hf.build_hf_qwen(cfg, sd, dtype=torch.bfloat16, device=dev, attn="sdpa")
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    ref_ids, ref_scores = [], []      # HF ids and processed scores [N, vocab] per sample
    with torch.no_grad():
        for b, ids in enumerate(inp["input_ids"]):
            ids = ids.to(dev)
            out = model.generate(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long, device=dev),
                                 pixel_values=inp["pixel_patches"][b * P:(b + 1) * P].to(dev, torch.bfloat16),
                                 image_grid_thw=torch.tensor([list(inp["grid_thw"][b])], device=dev),
                                 mm_token_type_ids=(ids == cfg.image_token_id).long()[None], max_new_tokens=N, min_new_tokens=N,
                                 do_sample=False, eos_token_id=None, pad_token_id=0, output_scores=True, return_dict_in_generate=True)
            ref_ids.append(out.sequences[0, len(ids):].tolist())
            ref_scores.append(torch.stack([s[0].float() for s in out.scores]).cpu())
    del model
    gc.collect()
    torch.cuda.empty_cache()
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    eng = QwenVLEngine(Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(cfg).items() if k in fields}), dev)
    eng.load_state_dict(sd)
    toks = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], prompts_of(inp), N, ())
    compared = 0
    for b in range(B):
        scores = ref_scores[b]
        top2 = scores.topk(2, dim=-1).values
        shared = next((t for t in range(N) if toks[b][t] != ref_ids[b][t]), N)
        print(f"\n[qwen-7b generate] b={b} engine {toks[b]}\n    HF bf16 {ref_ids[b]}\n    HF margins "
              f"{[round(float(x), 3) for x in top2[:, 0] - top2[:, 1]]} shared prefix {shared}")
        for t in range(min(shared + 1, N)):          # the steps conditioned on a common prefix, the first differing one included
            assert float(scores[t].max() - scores[t, toks[b][t]]) <= 0.25, (b, t)
        compared += min(shared + 1, N)
    del sd, eng
    gc.collect()
    torch.cuda.empty_cache()
    assert compared >= 4

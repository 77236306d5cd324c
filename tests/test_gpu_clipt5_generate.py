"""CLIP-FlanT5 greedy generation on a real H100: the engine's encoder pass + cached decode loop against the CPU generation oracle
(teacher-forced on the engine's own tokens), the committed HF golden, and HF bf16 generate at clip-flant5-xxl width."""
import dataclasses
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import clipt5_oracle as orc
from oracle import clipt5_generate as cg
from test_gpu_clipt5 import captured_node_count, load_case, make_engine
from test_clipt5_generate_host import load_generate_golden


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


def device_inputs(inp, dev):
    i32 = lambda t: None if t is None else t.to(dev, torch.int32).contiguous()
    return inp["pixels"].to(dev).contiguous(), i32(inp["input_ids"]), i32(inp["text_lens"]), i32(inp.get("image_index"))


def generate(eng, inp, dev, max_new, eos=(), **kw):
    px, ids, lens, idx = device_inputs(inp, dev)
    return eng.generate_tensors(px, ids, lens, max_new, eos, image_index=idx, **kw)


def teacher_forced(sd, cfg, inp, tokens):
    """Scores of every step on the given token paths, fp32 and bf16 oracle."""
    args = (sd, cfg, inp["pixels"], inp["input_ids"], inp["text_lens"], max(len(t) for t in tokens), (), inp.get("image_index"))
    return cg.clipt5_generate(*args, mode="fp32", forced=tokens)["scores"], cg.clipt5_generate(*args, mode="bf16", forced=tokens)["scores"]


def decisive_prefix(margins):
    """Number of leading steps whose margin is positive (beyond them a near-tie may send two paths apart)."""
    n = 0
    for m in margins:
        if float(m) < 0:
            break
        n += 1
    return n


@pytest.mark.parametrize("kw", [{}, dict(round_attention_scores=True), dict(fuse_norms=True)])
def test_engine_tokens_are_the_oracles_argmax_on_its_own_path(dev, kw):
    """Self-consistency: teacher-forced on the engine's own tokens, every one of them is within 2x the oracle's bf16-vs-fp32 score gap
    (+ 1e-3) of the fp32 arg-max at its step. Every step is checked, so a near-tie cannot skip steps."""
    cfg = orc.ClipT5Config.tiny()
    sd = orc.make_synthetic_state_dict(cfg, seed=21)
    inp = orc.make_synthetic_inputs(cfg, 3, 14, seed=22, ragged=True, n_images=2)
    eng = make_engine(cfg, sd, dev, **kw)
    toks = generate(eng, inp, dev, 12)
    assert [len(t) for t in toks] == [12] * 3
    s32, s16 = teacher_forced(sd, cfg, inp, toks)
    for b in range(3):
        gap = (s16[b] - s32[b]).abs().amax(-1)
        chosen = s32[b].gather(-1, torch.tensor(toks[b])[:, None])[:, 0]
        short = s32[b].amax(-1) - chosen
        print(f"\n[clipt5 generate self-consistency {kw}] b={b} tokens {toks[b]} max shortfall {float(short.max()):.3e} "
              f"max bf16 gap {float(gap.max()):.3e}")
        assert bool((short <= 2.0 * gap + 1e-3).all()), (short, gap)


@pytest.mark.parametrize("case", ["free", "eos"])
def test_engine_matches_committed_hf_generate_golden(golden_dir, dev, case):
    """Against HF generate(do_sample=False) in fp32: ids equal up to the first step whose HF top-1 / top-2 margin is below 2x the oracle's
    bf16-vs-fp32 score gap (+ 1e-3) at that step on the HF path; at least 8 steps compared; where the whole path is decisive, the full ids
    (and so the lengths) are equal."""
    blob, cfg, sd, inp = load_generate_golden(golden_dir)
    c = blob["cases"][case]
    eng = make_engine(cfg, sd, dev)
    toks = generate(eng, inp, dev, blob["max_new_tokens"], c["eos_ids"])
    s32, s16 = teacher_forced(sd, cfg, inp, c["ids"])
    compared = 0
    for b, hf_ids in enumerate(c["ids"]):
        thr = 2.0 * (s16[b] - s32[b]).abs().amax(-1) + 1e-3
        n = decisive_prefix(c["margins"][b] - thr)
        print(f"\n[clipt5 generate golden {case}] b={b} engine {toks[b]}\n    HF {hf_ids} decisive steps {n} (threshold <= {float(thr.max()):.3e})")
        assert toks[b][:n] == hf_ids[:n]
        if n == len(hf_ids):
            assert toks[b] == hf_ids
        compared += n
    assert compared >= 8


def test_eos_ragged_prompts_and_batch_invariance(golden_dir, dev):
    """Sequences stop independently on an EOS id, nothing is emitted after it (-1), and each prompt generated on its own gives the
    batch's tokens on its decisive steps."""
    blob, cfg, sd, inp = load_generate_golden(golden_dir)
    c = blob["cases"]["eos"]
    N = blob["max_new_tokens"]
    eng = make_engine(cfg, sd, dev)
    px, ids, lens, idx = device_inputs(inp, dev)
    st = eng.generate_begin(px, ids, lens, N, c["eos_ids"], image_index=idx)
    for _ in range(N - 1):
        eng.generate_step(st)
    tokens, lengths = st["tokens"].cpu(), st["lengths"].cpu()
    assert int(st["all_done"].cpu()[0]) == 1
    batch = generate(eng, inp, dev, N, c["eos_ids"])
    eos = set(c["eos_ids"])
    for b in range(len(batch)):
        n = int(lengths[b])
        assert tokens[b, :n].tolist() == batch[b]
        assert bool((tokens[b, n:] == -1).all())
        assert n == N or batch[b][-1] in eos
        assert not any(t in eos for t in batch[b][:-1])
    assert any(len(x) < N for x in batch) and any(len(x) == N for x in batch)
    s32, s16 = teacher_forced(sd, cfg, inp, batch)
    for b in range(len(batch)):
        img = int(inp["image_index"][b])
        one_inp = dict(pixels=inp["pixels"][img:img + 1], input_ids=inp["input_ids"][b:b + 1, :int(inp["text_lens"][b])],
                       text_lens=inp["text_lens"][b:b + 1])
        one = generate(eng, one_inp, dev, N, c["eos_ids"])[0]
        top2 = s32[b].topk(2, dim=-1).values
        n = decisive_prefix(top2[:, 0] - top2[:, 1] - 2.0 * (s16[b] - s32[b]).abs().amax(-1) - 1e-3)
        print(f"\n[clipt5 generate alone] b={b} batch {batch[b]} alone {one} decisive {n}")
        assert one[:n] == batch[b][:n]


@pytest.mark.parametrize("d_ff", [512, 2048])
def test_generate_launch_counts_equal_captured_graph_nodes(dev, d_ff):
    """last_launch_count() of the prefill and of one decode step is what each enqueues (the nodes of a CUDA graph capturing it), and the
    graph-replayed decode loop gives the tokens of direct step calls. d_ff = 2048 puts the decoder's wo GEMM on split-K."""
    cfg = orc.ClipT5Config.tiny(d_ff=d_ff)
    sd = orc.make_synthetic_state_dict(cfg, seed=23)
    inp = orc.make_synthetic_inputs(cfg, 3, 12, seed=24, ragged=True, n_images=2)
    eng = make_engine(cfg, sd, dev)
    px, ids, lens, idx = device_inputs(inp, dev)
    st = eng.generate_begin(px, ids, lens, 10, (5,), image_index=idx)
    assert captured_node_count(st["prefill"]) == eng.last_launch_count()
    n_prefill = eng.last_launch_count()
    st["prefill"]()
    assert captured_node_count(lambda: eng.generate_step(st)) == eng.last_launch_count()
    print(f"\n[clipt5 generate launches d_ff={d_ff}] prefill {n_prefill}, step {eng.last_launch_count()}")
    graphed = generate(eng, inp, dev, 10, (5,), use_graph=True)
    graphed2 = generate(eng, inp, dev, 10, (5,), use_graph=True)          # replays the graph captured by the previous call
    direct = generate(eng, inp, dev, 10, (5,), use_graph=False)
    assert graphed == direct == graphed2


def test_scoring_after_generation_is_unchanged(golden_dir, dev):
    """Generation uses a workspace of its own: scores after a generation are bit-identical to a fresh engine's, on the direct and the
    graph-replayed scoring paths."""
    blob, cfg, sd = load_case("tiny", golden_dir)
    inp = blob["inputs"]
    i32 = lambda t: t.to(dev, torch.int32)
    args = [inp["pixels"].to(dev), i32(inp["input_ids"]), i32(inp["text_lens"]), i32(inp["labels"])]
    fresh = make_engine(cfg, sd, dev)
    ref = fresh.score_tensors(*args).cpu()
    ref_g = fresh.score_tensors_graphed(*args).cpu()
    eng = make_engine(cfg, sd, dev)
    eng.score_tensors_graphed(*args)                        # a scoring graph captured before the generation
    gen_inp = dict(pixels=inp["pixels"], input_ids=inp["input_ids"], text_lens=inp["text_lens"])
    generate(eng, gen_inp, dev, 8)
    assert torch.equal(eng.score_tensors(*args).cpu(), ref)
    assert torch.equal(eng.score_tensors_graphed(*args).cpu(), ref_g)
    assert torch.equal(ref, ref_g)


class _WordTokenizer:
    """Stand-in T5 tokenizer: one id per word (3 + hash mod 400), every chunk ending in </s> (1); decode drops ids below 3 ("special")."""
    pad_token_id = 0
    eos_token_id = 1

    def __call__(self, chunk):
        import types
        return types.SimpleNamespace(input_ids=[3 + (sum(map(ord, w)) % 400) for w in chunk.split()] + [1])

    def decode(self, ids, skip_special_tokens=False):
        assert skip_special_tokens
        return " " + " ".join(str(i) for i in ids if i >= 3) + " "


def test_plugin_generate_returns_the_decoded_engine_ids(dev, tmp_path):
    import numpy as np
    from PIL import Image
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import CLIPT5Model, format_question
    cfg = orc.ClipT5Config.tiny()
    sd = orc.make_synthetic_state_dict(cfg, seed=25)
    rng = np.random.default_rng(0)
    paths = []
    for i, (h, w) in enumerate(((60, 90), (64, 64))):
        p = tmp_path / f"{i}.png"
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(p)
        paths.append(str(p))
    tok = _WordTokenizer()
    model = CLIPT5Model("clip-flant5-xl", device=str(dev), tokenizer=tok, state_dict=dict(sd), config=ClipT5Config(**dataclasses.asdict(cfg)),
                        checkpoint=str(tmp_path / "none.bin"))
    images, texts = [paths[0], paths[1], paths[0]], ["a red car", "two dogs on a sofa", "a blue sky"]
    out = model.generate(images=images, texts=texts, max_new_tokens=6)
    assert isinstance(out, list) and len(out) == 3 and all(isinstance(s, str) for s in out)
    prompts = model._prompt_ids([format_question(t) for t in texts])
    L = max(map(len, prompts))
    ids = torch.zeros(3, L, dtype=torch.int32)
    for i, r in enumerate(prompts):
        ids[i, :len(r)] = torch.tensor(r, dtype=torch.int32)
    pixels = model.load_images(paths)
    want = model.engine.generate_tensors(pixels, ids.to(dev), torch.tensor([len(r) for r in prompts], dtype=torch.int32, device=dev), 6, [1],
                                         image_index=torch.tensor([0, 1, 0], dtype=torch.int32, device=dev))
    assert out == [tok.decode(x, skip_special_tokens=True).strip() for x in want]
    assert all(len(s) > 0 for s in out)


def test_clipt5_xxl_generate_matches_reference_bf16_on_this_gpu(dev):
    """clip-flant5-xxl width, B = 2 ragged prompts, 16 new tokens: the engine's decode loop against HF bf16 T5ForConditionalGeneration.generate
    (do_sample=False, under autocast, as the reference runs) on the same GPU and weights, HF first and released before the engine is built.
    Random weights give flat logits, so near-ties are frequent: at every step where the engine's path still equals HF's, the engine's token
    must score within 0.25 of HF's best score at that step."""
    import copy
    import hf_reference as hf
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.engine import ClipT5Engine
    cfg = orc.ClipT5Config.xxl()
    B, N = 2, 16
    sd = orc.make_synthetic_state_dict(cfg, seed=0, device=dev, gen_device=dev)
    inp = orc.make_synthetic_inputs(cfg, B, 32, seed=1, ragged=True)
    vision, proj, t5 = hf.build_hf_modules(cfg, sd, dtype=torch.bfloat16, device=dev)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        feats = vision(inp["pixels"].to(dev, torch.bfloat16), output_hidden_states=True).hidden_states[-2][:, 1:]
        img = proj(feats.to(torch.bfloat16))
        S = inp["input_ids"].shape[1] - 1 + img.shape[1]
        embeds = torch.zeros(B, S, cfg.d_model, dtype=img.dtype, device=dev)
        mask = torch.zeros(B, S, dtype=torch.long, device=dev)
        for b in range(B):
            ids = inp["input_ids"][b, :int(inp["text_lens"][b])].to(dev)
            s = int((ids == orc.IMAGE_TOKEN_INDEX).nonzero()[0])
            seq = torch.cat([t5.shared(ids[:s]).to(img.dtype), img[b], t5.shared(ids[s + 1:]).to(img.dtype)])
            embeds[b, :len(seq)] = seq
            mask[b, :len(seq)] = 1
        gcfg = copy.deepcopy(t5.generation_config)
        gcfg.eos_token_id, gcfg.max_new_tokens, gcfg.max_length, gcfg.min_length = None, N, None, 0
        gcfg.do_sample, gcfg.num_beams, gcfg.output_scores, gcfg.return_dict_in_generate = False, 1, True, True
        out = t5.generate(inputs_embeds=embeds, attention_mask=mask, generation_config=gcfg)
    ref_ids = out.sequences[:, 1:].tolist()
    ref_scores = torch.stack([s.float() for s in out.scores], dim=1).cpu()        # [B, N, vocab]
    del vision, proj, t5, out, embeds, feats, img
    gc.collect()
    torch.cuda.empty_cache()
    eng = ClipT5Engine(ClipT5Config(**dataclasses.asdict(cfg)), dev)
    eng.load_state_dict(sd)
    del sd
    gc.collect()
    toks = generate(eng, inp, dev, N)
    compared = 0
    for b in range(B):
        scores = ref_scores[b]
        top2 = scores.topk(2, dim=-1).values
        shared = next((t for t in range(N) if toks[b][t] != ref_ids[b][t]), N)
        print(f"\n[clip-flant5-xxl generate] b={b} engine {toks[b]}\n    HF bf16 {ref_ids[b]}\n    HF margins "
              f"{[round(float(x), 3) for x in top2[:, 0] - top2[:, 1]]} shared prefix {shared}")
        for t in range(min(shared + 1, N)):          # the steps conditioned on a common prefix, the first differing one included
            assert float(scores[t].max() - scores[t, toks[b][t]]) <= 0.25, (b, t)
        compared += min(shared + 1, N)
    del eng
    gc.collect()
    torch.cuda.empty_cache()
    assert compared >= 4

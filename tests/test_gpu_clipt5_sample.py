"""CLIP-FlanT5 sampled generation on a real H100: sample_select_kernel as the T5 step calls it (V = 32128, no penalty, no positions), the
encoder expansion of the shared prefill, the tiny model end to end against tests/sample_ref_clipt5.clipt5_sample, sharing against no sharing,
the plugin, and the first draws at clip-flant5-xxl width against the fp64 warpers on HF's bf16 scores."""
import ctypes
import dataclasses
import gc

import numpy as np
import pytest
import torch

import sample_ref as sr
from sample_ref_clipt5 import clipt5_sample
from oracle import clipt5_oracle as orc
from test_gpu_clipt5 import captured_node_count, load_case, make_engine
from test_gpu_clipt5_generate import device_inputs, generate
from test_gpu_qwen_sample import BAND, run_select, sample_rows

pytestmark = pytest.mark.gpu

T5_VOCAB = 32128


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops(dev):
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


# ------------------------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("T", [0.7, 1.0])
def test_t5_vocab_kept_sets_and_draws_match_the_fp64_warpers(ops, T):
    """vqa_op_sample_select with no penalty bitmap and no positions (the T5 step's arguments) at V = 32128 on heavy-tailed, flat and
    Gaussian rows: top-k membership exact, top-p kept sets equal except ids within BAND of 1 - top_p, draws the host's Gumbel-max except
    at fp32 near-ties (or where the kept sets differed)."""
    gen = torch.Generator().manual_seed(int(T * 100))
    logits = sample_rows(T5_VOCAB, gen)[:3]
    seeds = [int(s) for s in torch.randint(0, 2 ** 62, (3,), generator=gen)]
    x = sr.processed_scores(logits, None, 1.0, T)
    band_ids = near = 0
    for k in (0, 1, 50):
        for p in (1e-6, 0.5, 0.9, 1.0):
            toks, kept = run_select(ops, logits, seeds, T, k, p)
            for b in range(3):
                want, cum, thr = sr.warp_row(x[b], k, p)
                if k:
                    assert not (kept[b] & ~(x[b] >= np.sort(x[b])[::-1][k - 1])).any(), (k, p, b)
                diff = np.nonzero(kept[b] != want)[0]
                assert np.all(np.abs(cum[diff] - thr) < BAND), (k, p, b, diff[:10])
                band_ids += len(diff)
                tok, gap = sr.draw(x[b], want, seeds[b], 0)
                if int(toks[b]) != tok:
                    assert len(diff) > 0 or gap < 4e-7 * (abs(float(x[b][tok]) - float(x[b].max())) + 20.0), (k, p, b, int(toks[b]), tok)
                    near += 1
                assert kept[b][int(toks[b])]
    print(f"\n[t5 sample select T={T}] {band_ids} kept-set ids inside the band, {near} draws at fp32 near-ties")


@pytest.mark.parametrize("n_prompts", [1, 3, 6])
def test_expansion_copies_each_slot_from_its_prompt(ops, dev, n_prompts):
    """vqa_op_clipt5_expand_prompts on ragged prompt lengths: slots below n_prompts are untouched, every later slot's xn rows, xt block
    (padding columns included) and length are bit-identical to its prompt's, out-of-range indices are clamped, and nothing past the
    B slots is written."""
    B, S, D = 6, 13, 64
    Sp = (S + 7) // 8 * 8
    gen = torch.Generator().manual_seed(n_prompts)
    xn_all = torch.randn(B + 1, S, D, generator=gen).bfloat16().to(dev)          # slot B is a guard
    xt_all = torch.randn(B + 1, D, Sp, generator=gen).bfloat16().to(dev)
    lens_all = torch.randint(1, S + 1, (B + 1,), generator=gen, dtype=torch.int32).to(dev)
    index = list(range(n_prompts)) + [int(i) for i in torch.randint(0, n_prompts, (B - n_prompts,), generator=gen)]
    if n_prompts < B:
        index[-1] = 1000                 # clamped to n_prompts - 1
    if n_prompts < B - 1:
        index[-2] = -7                   # clamped to 0
    before = [t.clone() for t in (xn_all, xt_all, lens_all)]
    pidx = torch.tensor(index, dtype=torch.int32, device=dev) if n_prompts < B else None
    ops.clipt5_expand_prompts(xn_all[:B], xt_all[:B], lens_all[:B], n_prompts, pidx)
    torch.cuda.synchronize()
    for b in range(B + 1):
        src = b if (b < n_prompts or b == B) else min(max(index[b], 0), n_prompts - 1)
        for t, t0 in zip((xn_all, xt_all, lens_all), before):
            assert torch.equal(t[b], t0[src]), (b, src)
    assert len(set(lens_all[:n_prompts].tolist())) > 1 or n_prompts == 1


# ------------------------------------------------------------------------------------------------ tiny model end to end
@pytest.fixture(scope="module")
def tiny(dev):
    cfg = orc.ClipT5Config.tiny()
    sd = orc.make_synthetic_state_dict(cfg, seed=31)
    inp = orc.make_synthetic_inputs(cfg, 3, 14, seed=32, ragged=True, n_images=2)
    return cfg, sd, inp, make_engine(cfg, sd, dev)


def sample(eng, inp, dev, seeds, T, k, p, max_new=12, prompt_of_sample=None, **kw):
    px, ids, lens, idx = device_inputs(inp, dev)
    return eng.sample_tensors(px, ids, lens, max_new, (), seeds, T, k, p, image_index=idx, prompt_of_sample=prompt_of_sample, **kw)


def test_top1_is_greedy_and_graph_replay_equals_eager(tiny, dev):
    cfg, sd, inp, eng = tiny
    greedy = generate(eng, inp, dev, 12)
    assert sample(eng, inp, dev, [1, 2, 3], 0.7, 1, 0.9) == greedy
    a = sample(eng, inp, dev, [11, 12, 13], 1.0, 0, 0.95)
    b = sample(eng, inp, dev, [11, 12, 13], 1.0, 0, 0.95)
    eager = sample(eng, inp, dev, [11, 12, 13], 1.0, 0, 0.95, use_graph=False)
    other = sample(eng, inp, dev, [91, 92, 93], 1.0, 0, 0.95)
    assert a == b == eager
    assert other != a


def test_sampled_tokens_match_the_oracle_up_to_a_near_tie(tiny, dev):
    """With the same seeds, the engine's tokens equal the bf16 oracle's up to the first step where the draw's margin, or the nearest
    kept-set boundary, is inside the bf16 error bound (0.05 in score, 2e-3 in mass), and everywhere when the two paths never part; at
    least 8 steps are compared."""
    cfg, sd, inp, eng = tiny
    seeds = [5, 6, 7]
    got = sample(eng, inp, dev, seeds, 0.8, 20, 0.9)
    ref = clipt5_sample(sd, cfg, inp["pixels"], inp["input_ids"], inp["text_lens"], 12, seeds, 0.8, 20, 0.9,
                        image_index=inp["image_index"], mode="bf16")
    compared = 0
    for b in range(3):
        n = next((t for t, (m, d) in enumerate(zip(ref["margins"][b], ref["boundary"][b])) if m < 0.05 or d < 2e-3), len(ref["tokens"][b]))
        print(f"\n[t5 sample vs oracle] b={b} engine {got[b]} oracle {ref['tokens'][b]} decisive {n}")
        assert got[b][:n + 1] == ref["tokens"][b][:n + 1] or got[b][:n] == ref["tokens"][b][:n]
        compared += len(got[b]) if got[b] == ref["tokens"][b] else n
    assert compared >= 8


def test_a_seed_gives_the_same_tokens_in_any_slot(tiny, dev):
    cfg, sd, inp, eng = tiny
    a = sample(eng, inp, dev, [5, 6, 7, 9], 1.0, 0, 0.95, prompt_of_sample=[0, 1, 2, 0])     # seed 5 in slot 0, seed 9 in slot 3
    b = sample(eng, inp, dev, [9, 6, 7, 5], 1.0, 0, 0.95, prompt_of_sample=[0, 1, 2, 0])     # and the other way round
    assert a[0] == b[3] and a[3] == b[0] and a[1:3] == b[1:3]
    assert a[0] != a[3]


def test_sampled_launches_and_profiled_work(tiny, dev):
    """The sampled step launches what the greedy step launches, as many as its captured graph's nodes; the shared prefill launches the
    unshared one's kernels plus the expansion, its encoder GEMM FLOPs (prefill minus step) are those of its n_prompts prompts, and the
    expansion's bytes are in the profile."""
    cfg, sd, inp, eng = tiny
    px, ids, lens, idx = device_inputs(inp, dev)
    smp = dict(temperature=0.7, top_k=50, top_p=0.9)

    def prefill_and_step(n, B, sampled=True):
        pi = torch.tensor(list(range(n)) + [0] * (B - n), dtype=torch.int32, device=dev) if B > n else None
        kw = dict(sample=dict(seeds=list(range(B)), **smp), prompt_index=pi) if sampled else {}
        eng.set_profile(True)
        st = eng.generate_begin(px, ids[:n], lens[:n], 8, (), image_index=idx[:n], **kw)
        torch.cuda.synchronize()
        pre = (eng.last_launch_count(), eng.read_profile())
        eng.generate_step(st)
        torch.cuda.synchronize()
        step = (eng.last_launch_count(), eng.read_profile())
        eng.set_profile(False)
        return st, pre, step
    _, g_pre, g_step = prefill_and_step(3, 3, sampled=False)
    st, u_pre, u_step = prefill_and_step(3, 3)
    assert u_step[0] == g_step[0] and u_pre[0] == g_pre[0]
    assert captured_node_count(lambda: eng.generate_step(st)) == eng.last_launch_count() == g_step[0]
    _, s_pre, s_step = prefill_and_step(2, 3)
    _, two_pre, two_step = prefill_and_step(2, 2)
    assert s_pre[0] == u_pre[0] + 1 and s_step[0] == u_step[0]
    enc = lambda pre, step: pre[1]["gemm"][1] - step[1]["gemm"][1]
    assert enc(s_pre, s_step) == pytest.approx(enc(two_pre, two_step), rel=1e-12)
    assert enc(s_pre, s_step) < enc(u_pre, u_step)
    S = ids.shape[1] - 1 + cfg.num_patches
    Sp = (S + 7) // 8 * 8
    expand_bytes = 2.0 * (S * cfg.d_model + cfg.d_model * Sp) * 2 + 8
    assert s_pre[1]["other"][3] - u_pre[1]["other"][3] == pytest.approx(expand_bytes, rel=1e-12)
    print(f"\n[t5 sample launches] prefill greedy {g_pre[0]} sampled {u_pre[0]} shared {s_pre[0]}; step {g_step[0]}; "
          f"encoder GEMM GFLOP shared(2 of 3) {enc(s_pre, s_step) / 1e9:.4f} unshared(3) {enc(u_pre, u_step) / 1e9:.4f}")


def encoder_output(eng, B, NI, L, S):
    """The encoder output slots [B, S, d_model] of the generation workspace after a prefill (its plan is the scoring plan at T = 1)."""
    off = (ctypes.c_size_t * 6)()
    eng._run("vqa_clipt5_debug_layout", B, NI, L, 1, off, 6)
    n = B * S * eng.cfg.d_model * 2
    return eng._gen_workspace[off[0]:off[0] + n].view(torch.bfloat16).view(B, S, eng.cfg.d_model).clone()


def test_sharing_against_separate_prompts(tiny, dev):
    """Pairs 0 and 1 twice each, with sharing (2 encoded prompts, expanded to 4 slots) and as 4 separate prompts, same seeds. The shared
    prefill's expanded slots equal their source slots bit for bit; where the encoder output does not depend on the number of encoded
    prompts, the tokens are equal too."""
    cfg, sd, inp, eng = tiny
    px, ids, lens, idx = device_inputs(inp, dev)
    L, NI = ids.shape[1], px.shape[0]
    S = L - 1 + cfg.num_patches
    seeds = [21, 22, 23, 24]
    shared = eng.sample_tensors(px, ids[:2], lens[:2], 12, (), seeds, 0.9, 0, 0.95, image_index=idx[:2], prompt_of_sample=[0, 1, 0, 1])
    eng.generate_begin(px, ids[:2], lens[:2], 12, (), image_index=idx[:2], prompt_index=torch.tensor([0, 1, 0, 1], dtype=torch.int32,
                       device=dev), sample=dict(seeds=[21, 22, 23, 24], temperature=0.9, top_k=0, top_p=0.95))
    torch.cuda.synchronize()
    enc_shared = encoder_output(eng, 4, NI, L, S)
    assert torch.equal(enc_shared[2], enc_shared[0]) and torch.equal(enc_shared[3], enc_shared[1])
    rep = [0, 1, 0, 1]
    sep = eng.sample_tensors(px, ids[rep].contiguous(), lens[rep].contiguous(), 12, (), seeds, 0.9, 0, 0.95, image_index=idx[rep].contiguous())
    eng.generate_begin(px, ids[rep].contiguous(), lens[rep].contiguous(), 12, (), image_index=idx[rep].contiguous(),
                       sample=dict(seeds=seeds, temperature=0.9, top_k=0, top_p=0.95))
    torch.cuda.synchronize()
    enc_sep = encoder_output(eng, 4, NI, L, S)
    same = torch.equal(enc_sep, enc_shared)
    print(f"\n[t5 sharing] encoder output equal: {same} (max |diff| {float((enc_sep.float() - enc_shared.float()).abs().max()):.3e}); "
          f"shared {shared} separate {sep}")
    assert same
    assert shared == sep


def test_scoring_after_sampled_generation_is_unchanged(golden_dir, dev):
    blob, cfg, sd = load_case("tiny", golden_dir)
    inp = blob["inputs"]
    i32 = lambda t: t.to(dev, torch.int32)
    args = [inp["pixels"].to(dev), i32(inp["input_ids"]), i32(inp["text_lens"]), i32(inp["labels"])]
    fresh = make_engine(cfg, sd, dev)
    ref = fresh.score_tensors(*args).cpu()
    ref_g = fresh.score_tensors_graphed(*args).cpu()
    eng = make_engine(cfg, sd, dev)
    eng.score_tensors_graphed(*args)
    B = inp["input_ids"].shape[0]
    eng.sample_tensors(args[0], args[1], args[2], 8, (), list(range(2 * B)), 0.7, 50, 0.9, prompt_of_sample=list(range(B)) * 2)
    assert torch.equal(eng.score_tensors(*args).cpu(), ref)
    assert torch.equal(eng.score_tensors_graphed(*args).cpu(), ref_g)


# ------------------------------------------------------------------------------------------------ plugin
def test_plugin_samples_repeated_pairs_from_one_encoding(dev, tmp_path):
    import json
    from PIL import Image
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import CLIPT5Model, format_question
    from test_gpu_clipt5_generate import _WordTokenizer
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
    images, texts = [paths[0], paths[1], paths[0], paths[0]], ["a red car", "two dogs", "a red car", "a blue sky"]
    torch.manual_seed(3)
    out = model.generate(images=images, texts=texts, max_new_tokens=6, temperature=0.7)
    torch.manual_seed(3)
    again = model.generate(images=images, texts=texts, max_new_tokens=6, temperature=0.7)
    assert out == again and len(out) == 4
    seeds = torch.randint(0, 2 ** 63 - 1, (4,), dtype=torch.int64, generator=torch.Generator().manual_seed(3)).tolist()
    prompts = model._prompt_ids([format_question(t) for t in ("a red car", "two dogs", "a blue sky")])
    L = max(map(len, prompts))
    ids = torch.zeros(3, L, dtype=torch.int32)
    for i, r in enumerate(prompts):
        ids[i, :len(r)] = torch.tensor(r, dtype=torch.int32)
    want = model.engine.sample_tensors(model.load_images(paths), ids.to(dev), torch.tensor([len(r) for r in prompts], dtype=torch.int32,
                                       device=dev), 6, [1], seeds, 0.7, 50, 0.9, image_index=torch.tensor([0, 1, 0], dtype=torch.int32,
                                       device=dev), prompt_of_sample=[0, 1, 0, 2])
    assert out == [tok.decode(x, skip_special_tokens=True).strip() for x in want]
    for key, value in (("min_p", 0.05), ("repetition_penalty", 1.2)):
        (tmp_path / "generation_config.json").write_text(json.dumps({key: value}))
        before = model.engine.last_launch_count()
        with pytest.raises(NotImplementedError, match=key):
            model.generate(images=images, texts=texts, max_new_tokens=6, temperature=0.7)
        assert model.engine.last_launch_count() == before


# ------------------------------------------------------------------------------------------------ clip-flant5-xxl width
def test_clipt5_xxl_first_draws_lie_in_hf_kept_set(dev):
    """clip-flant5-xxl width, one prompt of 32 text ids, 128 first tokens drawn at T 0.7 / top_k 50 / top_p 0.9 (one encoder pass, expanded
    to 128 slots). HF bf16 T5ForConditionalGeneration's step-0 scores (under autocast, as the reference runs; HF first and released before
    the engine is built) through the fp64 warpers give the kept set; every drawn id is in it unless its score is within 0.25 of the set's
    cut (the engine's own bf16 logits differ from HF's by rounding)."""
    import copy
    import hf_reference as hf
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.engine import ClipT5Engine
    cfg = orc.ClipT5Config.xxl()
    N = 128
    sd = orc.make_synthetic_state_dict(cfg, seed=0, device=dev, gen_device=dev)
    inp = orc.make_synthetic_inputs(cfg, 1, 32, seed=1)
    vision, proj, t5 = hf.build_hf_modules(cfg, sd, dtype=torch.bfloat16, device=dev)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        feats = vision(inp["pixels"].to(dev, torch.bfloat16), output_hidden_states=True).hidden_states[-2][:, 1:]
        img = proj(feats.to(torch.bfloat16))
        ids = inp["input_ids"][0, :int(inp["text_lens"][0])].to(dev)
        s = int((ids == orc.IMAGE_TOKEN_INDEX).nonzero()[0])
        embeds = torch.cat([t5.shared(ids[:s]).to(img.dtype), img[0], t5.shared(ids[s + 1:]).to(img.dtype)])[None]
        mask = torch.ones(1, embeds.shape[1], dtype=torch.long, device=dev)
        gcfg = copy.deepcopy(t5.generation_config)
        gcfg.eos_token_id, gcfg.max_new_tokens, gcfg.max_length, gcfg.min_length = None, 1, None, 0
        gcfg.do_sample, gcfg.num_beams, gcfg.output_scores, gcfg.return_dict_in_generate = False, 1, True, True
        out = t5.generate(inputs_embeds=embeds, attention_mask=mask, generation_config=gcfg)
    logits = out.scores[0][0].cpu()
    del vision, proj, t5, out, embeds, feats, img
    gc.collect()
    torch.cuda.empty_cache()
    eng = ClipT5Engine(ClipT5Config(**dataclasses.asdict(cfg)), dev)
    eng.load_state_dict(sd)
    del sd
    gc.collect()
    px, ids_d, lens_d, _ = device_inputs(inp, dev)
    toks = eng.sample_tensors(px, ids_d, lens_d, 1, (), list(range(N)), 0.7, 50, 0.9, prompt_of_sample=[0] * N)
    x = sr.processed_scores(logits.bfloat16()[None], None, 1.0, 0.7)[0]
    kept, _, _ = sr.warp_row(x, 50, 0.9)
    cut = float(x[kept].min())
    drawn = [t[0] for t in toks]
    outside = [t for t in drawn if not kept[t]]
    print(f"\n[clip-flant5-xxl sampled step 0] {int(kept.sum())} kept, {len(set(drawn))} distinct of {N} draws, {len(outside)} outside")
    assert len(toks) == N and all(len(t) == 1 for t in toks)
    for t in outside:
        assert cut - float(x[t]) <= 0.25, (t, float(x[t]), cut)
    assert len(set(drawn)) > 1
    del eng
    gc.collect()
    torch.cuda.empty_cache()

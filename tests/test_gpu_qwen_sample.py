"""Sampled token selection (sample_select_kernel) on a real H100 through vqa_op_sample_select, and sampled generation end to end on the
tiny model: kept sets against the fp64 restatement of HF's warpers (tests/sample_ref.py), draws against the host's Gumbel-max on the same
Philox stream, a chi-square test of the drawn distribution, the bookkeeping it shares with greedy selection, and the engine and plugin."""
import math

import numpy as np
import pytest
import torch

import sample_ref as sr
from oracle import qwen25vl_oracle as qo
from test_gpu_decode_kernels import SelectState, assert_same_state

pytestmark = pytest.mark.gpu

BAND = 1e-5        # a kept-set difference is allowed only for an id whose fp64 cumulative mass is this close to 1 - top_p


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


def run_select(ops, logits, seeds, T, k, p, bitmap=None, penalty=1.0, lengths=None, max_new=64):
    """One vqa_op_sample_select launch on fresh state -> (tokens drawn [B], kept bool [B, V])."""
    B, V = logits.shape
    st = SelectState(B, V, max_new, bitmap, lengths=lengths).to_device()
    kept = torch.zeros(B, (V + 31) // 32, dtype=torch.int32, device="cuda")
    ops.sample_select(logits.cuda(), torch.as_tensor(seeds, dtype=torch.int64).cuda(), T, k, p, st.tokens, st.lengths, st.done, st.n_done,
                      st.all_done, st.next_ids, pen_bitmap=st.bitmap, repetition_penalty=penalty, kept=kept)
    torch.cuda.synchronize()
    words = kept.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    ids = np.arange(V)
    return st.next_ids.cpu().numpy(), ((words[:, ids // 32] >> (ids % 32)) & 1).astype(bool)


def sample_rows(V, gen):
    """bf16 rows: 0 heavy-tailed (a few large logits over Gaussian noise), 1 flat (a 1/8 grid: huge tie groups), 2 Gaussian * 3 (the CPU
    measurement's row: most values equal a neighbour), 3 the heavy tail under a repetition penalty (bitmap given separately)."""
    r0 = torch.randn(V, generator=gen) * 1.5
    r0[torch.randint(0, V, (40,), generator=gen)] += torch.rand(40, generator=gen) * 12
    r1 = torch.randint(-16, 9, (V,), generator=gen).float() / 8
    r2 = torch.randn(V, generator=gen) * 3
    return torch.stack([r0, r1, r2, r0.clone()]).bfloat16()


def penalty_bitmap(B, V, gen, rows=(3,)):
    words = -(-V // 32)
    bits = torch.zeros(B, words * 32, dtype=torch.bool)
    for b in rows:
        bits[b] = torch.rand(words * 32, generator=gen) < 0.3
    packed = (bits.view(B, words, 32).long() << torch.arange(32)).sum(-1)
    return torch.where(packed >= 1 << 31, packed - (1 << 32), packed).to(torch.int32)


@pytest.mark.parametrize("T", [1e-38, 1e-3, 0.7, 1.0, 100.0])
@pytest.mark.parametrize("V", [152064, 1000])
def test_kept_set_and_draw_match_the_fp64_warpers(ops, V, T):
    """Every (top_k, top_p) of the grid on heavy-tailed, flat and Gaussian rows and under a penalty: top-k membership exact, top-p kept
    sets equal except for ids whose fp64 cumulative mass is within BAND of 1 - top_p, and the drawn token the host's Gumbel-max over the
    host's kept set except where the two best perturbed scores are within fp32 error (or the kept sets differed). top_p = 1e-8 makes
    fp32(1 - top_p) = 1: every cumulative probability is at or below it and only the last id of the ascending order stays. T = 1e-38
    overflows nearly every score to +-inf, which the kernel saturates to +-FLT_MAX (as the restatement does)."""
    gen = torch.Generator().manual_seed(V + int(T * 1000))
    logits = sample_rows(V, gen)
    B = logits.shape[0]
    bitmap = penalty_bitmap(B, V, gen)
    seeds = [int(s) for s in torch.randint(0, 2 ** 62, (B,), generator=gen)]
    x = sr.processed_scores(logits, bitmap, 1.3, T)
    band_ids = near_draws = checked = 0
    for k in (0, 1, 50, V + 5):
        for p in (1e-8, 1e-6, 0.5, 0.9, 1.0):
            toks, kept = run_select(ops, logits, seeds, T, k, p, bitmap, 1.3)
            for b in range(B):
                want, cum, thr = sr.warp_row(x[b], k, p)
                if 0 < k < V:       # top-k is an exact comparison on identical fp32 scores
                    assert not (kept[b] & ~(x[b] >= np.sort(x[b])[::-1][k - 1])).any(), (k, p, b)
                diff = np.nonzero(kept[b] != want)[0]
                assert np.all(np.abs(cum[diff] - thr) < BAND), (k, p, b, diff[:10], cum[diff][:10], thr)
                band_ids += len(diff)
                tok, gap = sr.draw(x[b], want, seeds[b], 0)
                if int(toks[b]) != tok:
                    vbest = abs(float(x[b][tok]) - float(x[b].max())) + 20.0
                    assert len(diff) > 0 or gap < 4e-7 * vbest, (k, p, b, int(toks[b]), tok, gap)
                    near_draws += 1
                assert 0 <= int(toks[b]) < V and kept[b][int(toks[b])], (k, p, b)
                if p == 1e-8:
                    assert kept[b].sum() == 1, (k, b)
                checked += 1
    print(f"\n[sample select V={V} T={T}] {checked} rows: {band_ids} kept-set ids inside the {BAND:g} band, {near_draws} draws at fp32 near-ties")


def test_drawn_distribution_chi_square(ops):
    """2^16 draws (one seed each) of one row under T 0.7, top_k 50, top_p 0.9, against the exact warped probabilities. The seeds are
    fixed, so the statistic is too."""
    from scipy.stats import chisquare
    gen = torch.Generator().manual_seed(5)
    V, N = 1000, 1 << 16
    row = (torch.randn(V, generator=gen) * 2).bfloat16()
    x = sr.processed_scores(row[None], None, 1.0, 0.7)[0]
    kept, _, _ = sr.warp_row(x, 50, 0.9)
    prob = np.where(kept, np.exp(x.astype(np.float64) - x.max()), 0.0)
    prob /= prob.sum()
    toks, _ = run_select(ops, row[None].expand(N, V).contiguous(), list(range(1, N + 1)), 0.7, 50, 0.9)
    assert kept[toks].all()
    ids = np.nonzero(kept)[0]
    obs = np.bincount(toks, minlength=V)[ids]
    exp = prob[ids] * N
    stat, pv = chisquare(obs, exp)
    print(f"\n[sample chi-square] {len(ids)} kept ids, chi2 {stat:.1f}, p {pv:.3f}")
    assert pv > 1e-3


def test_bookkeeping_state_machine_matches_greedy_rules(ops):
    """The 40-step state machine of the greedy selection tests, with each token the host's draw: tokens, lengths, penalty bits, next ids,
    positions, done / n_done / all_done all equal after every step."""
    B, V, max_new = 7, 1001, 40
    eos_ids = [2, 999]
    finish = {6: 0, 0: 5, 1: 12, 2: 12, 5: 20, 4: 39}
    gen = torch.Generator().manual_seed(4)
    words = -(-V // 32)
    bits = torch.rand(B, words * 32, generator=gen) < 0.2
    packed = (bits.view(B, words, 32).long() << torch.arange(32)).sum(-1)
    bitmap = torch.where(packed >= 1 << 31, packed - (1 << 32), packed).to(torch.int32)
    first_pos = torch.randint(5, 900, (B,), generator=gen, dtype=torch.int32)
    seeds = torch.randint(0, 2 ** 62, (B,), generator=gen)
    T, k, p, pen = 0.7, 50, 0.9, 1.25
    ref = SelectState(B, V, max_new, bitmap, first_pos)
    dev = ref.to_device()
    eos_dev = torch.tensor(eos_ids, dtype=torch.int32, device="cuda")
    seeds_dev = seeds.cuda()
    for t in range(max_new):
        logits = torch.randn(B, V, generator=gen) * 2
        logits[:, eos_ids] = -20.0
        for b, step in finish.items():
            if step == t:
                logits[b, eos_ids[b % 2]] = 50.0
        logits = logits.bfloat16()
        x = sr.processed_scores(logits, ref.bitmap, pen, T)
        best = torch.tensor([sr.draw(x[b], sr.warp_row(x[b], k, p)[0], int(seeds[b]), int(ref.lengths[b]))[0] for b in range(B)])
        # SelectState.step_ref picks the arg-max of its scores: give it a one-hot row at the drawn token
        onehot = torch.full((B, V), -1.0).scatter_(1, best[:, None], 1.0).bfloat16()
        ref.step_ref(onehot, eos_ids, 1.0)
        ops.sample_select(logits.cuda(), seeds_dev, T, k, p, dev.tokens, dev.lengths, dev.done, dev.n_done, dev.all_done, dev.next_ids,
                          eos_ids=eos_dev, pen_bitmap=dev.bitmap, repetition_penalty=pen, first_pos=dev.first_pos, pos3=dev.pos3)
        torch.cuda.synchronize()
        assert_same_state(dev, ref, t)
    assert int(ref.all_done[0]) == 1


def test_same_seed_same_tokens_and_top1_is_greedy(ops):
    """A seed gives the same draw in any batch slot; top_k = 1 on rows with a unique maximum is the greedy token."""
    gen = torch.Generator().manual_seed(9)
    V = 152064
    row = (torch.randn(V, generator=gen) * 3).bfloat16()
    row[77] = 30.0
    toks, _ = run_select(ops, row[None].expand(4, V).contiguous(), [123, 456, 123, 456], 0.7, 0, 0.9)
    assert toks[0] == toks[2] and toks[1] == toks[3]
    logits = torch.randn(6, V, generator=gen).bfloat16()
    logits[torch.arange(6), torch.randint(0, V, (6,), generator=gen)] = 8.0
    toks, _ = run_select(ops, logits, list(range(6)), 1.0, 1, 1.0)
    assert toks.tolist() == logits.float().argmax(-1).tolist()


@pytest.mark.parametrize("T,k,p", [(0.0, 0, 1.0), (-1.0, 0, 1.0), (math.inf, 0, 1.0), (math.nan, 0, 1.0), (1.0, -1, 1.0), (1.0, 0, 0.0),
                                   (1.0, 0, 1.5), (1.0, 0, math.nan)])
def test_invalid_sampling_arguments_are_refused(ops, T, k, p):
    logits = torch.zeros(2, 100, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="status -1"):
        run_select(ops, logits, [1, 2], T, k, p)


# ------------------------------------------------------------------------------------------------ end to end on the tiny model
@pytest.fixture(scope="module")
def tiny(ops):
    from test_gpu_qwen import TINY, make_engine
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=21)
    inp = qo.make_synthetic_inputs(cfg, 3, (84, 56), 12, seed=22, ragged=True, n_images=2)
    return cfg, sd, inp, make_engine(cfg, sd, torch.device("cuda:0"))


def _args(inp, n=12):
    return (inp["pixel_patches"], inp["grid_thw"], [x.tolist() for x in inp["input_ids"]], n, ())


def test_sampled_top1_is_greedy_and_reproducible(tiny):
    cfg, sd, inp, eng = tiny
    kw = dict(image_of_sample=inp["image_of_sample"], repetition_penalty=1.3)
    greedy = eng.generate_prompts(*_args(inp), **kw)
    assert eng.sample_prompts(*_args(inp), [1, 2, 3], 0.7, 1, 1.0, **kw) == greedy
    a = eng.sample_prompts(*_args(inp), [11, 12, 13], 1.0, 0, 0.95, **kw)
    b = eng.sample_prompts(*_args(inp), [11, 12, 13], 1.0, 0, 0.95, **kw)
    eager = eng.sample_prompts(*_args(inp), [11, 12, 13], 1.0, 0, 0.95, **kw, use_graph=False)
    other = eng.sample_prompts(*_args(inp), [91, 92, 93], 1.0, 0, 0.95, **kw)
    assert a == b == eager
    assert other != a


def test_sampled_tokens_match_the_oracle_up_to_a_near_tie(tiny):
    """With the same seeds, the engine's tokens equal the bf16 oracle's up to the first step where the draw's margin, or the nearest
    kept-set boundary, is inside the bf16 error bound (0.05 in score, 2e-3 in mass), and everywhere when the two paths never part; at
    least 8 steps are compared."""
    cfg, sd, inp, eng = tiny
    seeds = [5, 6, 7]
    got = eng.sample_prompts(*_args(inp), seeds, 0.8, 20, 0.9, image_of_sample=inp["image_of_sample"], repetition_penalty=1.3)
    ref = sr.qwen25vl_sample(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], 12, seeds, 0.8, 20, 0.9,
                             image_of_sample=inp["image_of_sample"], mode="bf16", repetition_penalty=1.3)
    compared = 0
    for b in range(3):
        n = next((t for t, (m, d) in enumerate(zip(ref["margins"][b], ref["boundary"][b])) if m < 0.05 or d < 2e-3), len(ref["tokens"][b]))
        print(f"\n[sample vs oracle] b={b} engine {got[b]} oracle {ref['tokens'][b]} decisive {n}")
        assert got[b][:n + 1] == ref["tokens"][b][:n + 1] or got[b][:n] == ref["tokens"][b][:n]
        compared += len(got[b]) if got[b] == ref["tokens"][b] else n      # paths that never part are compared in full
    assert compared >= 8


def test_sampled_step_launches_what_the_greedy_step_launches(tiny):
    from test_gpu_clipt5 import captured_node_count
    cfg, sd, inp, eng = tiny
    kw = dict(image_of_sample=inp["image_of_sample"])
    st = eng.generate_begin(*_args(inp, 10), **kw)
    st["prefill"]()
    eng.generate_step(st)
    greedy = eng.last_launch_count()
    st = eng.generate_begin(*_args(inp, 10), **kw, sample=dict(seeds=[1, 2, 3], temperature=0.7, top_k=50, top_p=0.9))
    assert captured_node_count(lambda: eng.generate_step(st)) == eng.last_launch_count() == greedy


def test_plugin_samples_stills_and_frame_stacks(tiny, tmp_path):
    import dataclasses
    from PIL import Image
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    from test_gpu_qwen import TINY
    from test_gpu_qwen_generate import _DigitTokenizer
    ocfg = qo.Qwen25VLConfig.tiny(**TINY)
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    cfg = Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(ocfg).items() if k in fields})
    sd = qo.make_synthetic_state_dict(ocfg, seed=17)
    rng = np.random.default_rng(0)
    still = tmp_path / "a.png"
    Image.fromarray(rng.integers(0, 256, (60, 90, 3), dtype=np.uint8)).save(still)
    stack = tmp_path / "v.npy"
    np.save(stack, rng.integers(0, 256, (4, 56, 84, 3), dtype=np.uint8))

    frames = rng.integers(0, 256, (16, 56, 84, 3), dtype=np.uint8)

    class Reader:
        def open(self, path):
            return 16, 8.0, lambda idx: frames[list(idx)]

    model = Qwen2VLModel("qwen2.5-vl-7b", device="cuda:0", tokenizer=_DigitTokenizer(), state_dict=dict(sd), config=cfg,
                         checkpoint=str(tmp_path / "none.bin"), min_pixels=56 * 56, max_pixels=112 * 112, video_reader=Reader())
    images, texts = [str(still), str(stack), str(tmp_path / "c.mp4")], ["a red car", "two dogs", "a blue sky"]
    torch.manual_seed(3)
    a = model.generate(images, texts, max_new_tokens=6, temperature=0.7)
    torch.manual_seed(3)
    b = model.generate(images, texts, max_new_tokens=6, temperature=0.7)
    g = torch.Generator().manual_seed(3)
    c = model.generate(images, texts, max_new_tokens=6, temperature=0.7, generator=g)
    assert a == b == c and len(a) == 3 and all(isinstance(s, str) for s in a)


def test_sampled_top1_matches_committed_hf_golden(golden_dir, ops):
    """top_k = 1 on the committed golden's weights and inputs against HF's tokens there. HF's generate(do_sample=True, top_k=1) keeps
    only the ids at the maximum, so at every step whose top-1 / top-2 margin is positive it emits the arg-max, which is the golden's id
    (tests/test_qwen_sample_host.py pins the restatement to HF's sampled generate at top_k = 1). Ids are compared as the greedy golden test
    compares them: up to the first step whose HF margin is below 2x the oracle's bf16-vs-fp32 score gap; at least 8 steps per case."""
    from test_gpu_qwen import make_engine
    from test_gpu_qwen_generate import decisive_prefix, teacher_forced
    from test_qwen_generate_host import golden_case_inputs, load_generate_golden
    blob, cfg, sd = load_generate_golden(golden_dir)
    eng = make_engine(cfg, sd, torch.device("cuda:0"))
    for case in ("images_pen1.3", "video_pen1.0", "eos"):
        c = blob["cases"][case]
        inp, spg = golden_case_inputs(cfg, c)
        toks = eng.sample_prompts(inp["pixel_patches"], inp["grid_thw"], [x.tolist() for x in inp["input_ids"]], blob["max_new_tokens"],
                                  c["eos_ids"], list(range(len(inp["input_ids"]))), 0.7, 1, 0.9, image_of_sample=inp["image_of_sample"],
                                  repetition_penalty=c["penalty"], second_per_grid_ts=spg)
        s32, s16 = teacher_forced(sd, cfg, inp, c["ids"], c["penalty"], spg)
        compared = 0
        for b, hf_ids in enumerate(c["ids"]):
            n = decisive_prefix(c["margins"][b] - (2.0 * (s16[b] - s32[b]).abs().amax(-1) + 1e-3), 0.0)
            print(f"\n[sampled top_k 1 vs HF golden {case}] b={b} engine {toks[b]}\n    HF {hf_ids} decisive steps {n}")
            assert toks[b][:n] == hf_ids[:n]
            if n == len(hf_ids):
                assert toks[b] == hf_ids
            compared += n
        assert compared >= 8, case


def test_qwen25vl_7b_step0_kept_sets_match_hf_warpers(ops):
    """Qwen2.5-VL-7B width, B = 2, 448x448 images + 32 text ids: HF bf16 sdpa's first-step scores (its lm_head logits, as
    generate(output_scores=True) returns them with no processor) through vqa_op_sample_select give the kept sets of the fp64 warpers on
    the same scores, within the mass band, for the reference's T 0.7 / top_p 0.9 at top_k 50 and with top_k off, and top_k 1 draws
    HF's arg-max wherever the maximum is unique."""
    import gc
    import hf_reference as hf
    dev = torch.device("cuda:0")
    cfg = qo.Qwen25VLConfig.qwen25_vl_7b()
    B = 2
    sd = qo.make_synthetic_state_dict(cfg, seed=0, gen_device=dev)
    inp = qo.make_synthetic_inputs(cfg, B, (448, 448), 32, seed=1, ragged=True)
    model = hf.build_hf_qwen(cfg, sd, dtype=torch.bfloat16, device=dev, attn="sdpa")
    del sd
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    rows = []
    with torch.no_grad():
        for b, ids in enumerate(inp["input_ids"]):
            ids = ids.to(dev)
            out = model.generate(input_ids=ids[None], attention_mask=torch.ones(1, len(ids), dtype=torch.long, device=dev),
                                 pixel_values=inp["pixel_patches"][b * P:(b + 1) * P].to(dev, torch.bfloat16),
                                 image_grid_thw=torch.tensor([list(inp["grid_thw"][b])], device=dev),
                                 mm_token_type_ids=(ids == cfg.image_token_id).long()[None], max_new_tokens=1, do_sample=False,
                                 eos_token_id=None, pad_token_id=0, output_scores=True, return_dict_in_generate=True)
            rows.append(out.scores[0][0])
    del model
    gc.collect()
    torch.cuda.empty_cache()
    logits = torch.stack(rows).bfloat16()          # the bf16 lm_head output, exact in bf16
    assert torch.equal(logits.float(), torch.stack(rows).float())
    x = sr.processed_scores(logits, None, 1.0, 0.7)
    for k in (50, 0):
        toks, kept = run_select(ops, logits, [3, 4], 0.7, k, 0.9)
        for b in range(B):
            want, cum, thr = sr.warp_row(x[b], k, 0.9)
            diff = np.nonzero(kept[b] != want)[0]
            print(f"\n[7b step 0] b={b} top_k {k}: {int(want.sum())} kept, {len(diff)} inside the band")
            assert np.all(np.abs(cum[diff] - thr) < BAND)
            assert kept[b][int(toks[b])]
    toks, _ = run_select(ops, logits, [3, 4], 0.7, 1, 0.9)
    for b in range(B):
        top2 = logits[b].float().topk(2).values
        if float(top2[0]) > float(top2[1]):
            assert int(toks[b]) == int(logits[b].float().argmax())

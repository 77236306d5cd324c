"""Qwen2.5-VL path on a real H100: the grouped qkv GEMM and the engine vs the oracle (the head-dim-128 attention has its kernel-level tests
in test_gpu_qwen_kernels.py)."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import qwen25vl_oracle as qo

TINY = dict(hidden=256, heads=2, kv_heads=1, mrope_section=(16, 24, 24))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


def test_gemm_grouped_output_columns(dev):
    """qkv GEMM at the native head width: logical column c -> (c / 80) * 128 + c % 80 (GemmParams::c_group_in); the slot padding is left untouched."""
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import _ptr, _stream_ptr, _check
    lib = _lib.load()
    torch.manual_seed(6)
    M, K, G, gi, go = 700, 256, 9, 80, 128
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    w = (torch.randn(G * gi, K, device=dev) * K ** -0.5).bfloat16()
    b = torch.randn(G * gi, device=dev).bfloat16()
    c = torch.full((M, G * go), -5.0, dtype=torch.bfloat16, device=dev)
    _check(lib.vqa_op_gemm_bf16_grouped(_ptr(a), K, _ptr(w), K, G * gi, _ptr(c), G * go, M, G * gi, K, _ptr(b), gi, go, 0, _stream_ptr(a.device)),
           None, "vqa_op_gemm_bf16_grouped")
    torch.cuda.synchronize()
    ref = (a.float() @ w.float().t() + b.float()).view(M, G, gi)
    got = c.float().view(M, G, go)
    assert float((got[..., :gi] - ref).abs().max()) < 0.03
    assert bool((got[..., gi:] == -5.0).all())


def make_engine(cfg, sd, dev):
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.engine import QwenVLEngine
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    eng = QwenVLEngine(Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(cfg).items() if k in fields}), dev)
    eng.load_state_dict(sd)
    return eng


@pytest.mark.parametrize("hw,n_images", [((84, 56), None), ((112, 112), None), ((56, 84), 2)])
def test_qwen_engine_matches_oracle(dev, hw, n_images):
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=0)
    inp = qo.make_synthetic_inputs(cfg, 4, hw, 12, ragged=True, n_images=n_images)
    o32 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], inp["image_of_sample"],
                            mode="fp32", return_all=True)
    o16 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], inp["image_of_sample"],
                            mode="bf16", return_all=True)
    eng = make_engine(cfg, sd, dev)
    probs = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], [x.tolist() for x in inp["input_ids"]], inp["answer_ids"],
                              inp["image_of_sample"])
    torch.cuda.synchronize()
    p = probs.cpu()
    lp, l32, l16 = torch.log(p), torch.log(o32["scores"]), torch.log(o16["scores"])
    gap = float((l16 - l32).abs().max())
    print(f"\n[qwen {hw}] engine {p.tolist()}\n   oracle fp32 {o32['scores'].tolist()}\n   |dlogp| vs fp32 {float((lp - l32).abs().max()):.3e} vs bf16 "
          f"{float((lp - l16).abs().max()):.3e} | oracle bf16-vs-fp32 {gap:.3e} | launches {eng.last_launch_count()}")
    assert float((lp - l32).abs().max()) <= 2.0 * gap + 2e-2
    assert float((p - o32["scores"]).abs().max()) <= 1e-3 + 2.0 * float((o16["scores"] - o32["scores"]).abs().max())
    # temperature is applied to the fp32 logits before the softmax (qwen2vl_model.py:166)
    pT = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], [x.tolist() for x in inp["input_ids"]], inp["answer_ids"],
                           inp["image_of_sample"], temperature=2.0).cpu()
    refT = torch.stack([qo.answer_probability(o32["logits"][b], inp["answer_ids"][b], 2.0) for b in range(len(pT))])
    assert float((torch.log(pT) - torch.log(refT)).abs().max()) <= 2.0 * gap + 2e-2



@pytest.mark.parametrize("packed,pen", [(False, 1.0), (True, 1.0), (False, 1.3), (True, 1.3)])
def test_qwen_launch_count_equals_captured_graph_nodes(dev, packed, pen):
    """last_launch_count() is what one forward enqueues (the nodes of a CUDA graph that captures it), padded and packed, with and
    without the repetition-penalty bitmap, and then what the top-k of that call enqueues (lm_head and top-k softmax)."""
    from t2v_metrics_b200 import qwen_host
    from test_gpu_clipt5 import captured_node_count
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    inp = qo.make_synthetic_inputs(cfg, 4, (56, 84), 12, ragged=True, n_images=2)
    eng = make_engine(cfg, qo.make_synthetic_state_dict(cfg, seed=0), dev)
    ec = eng.cfg
    grids = [tuple(map(int, g)) for g in inp["grid_thw"]]
    build = qwen_host.build_packed_indices if packed else qwen_host.build_batch_indices
    idx = build([x.tolist() for x in inp["input_ids"]], grids, list(inp["image_of_sample"]), ec.image_token_id, ec.spatial_merge_size,
                ec.tokens_per_second, video_token_id=ec.video_token_id)
    d = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in idx.items()}
    ans = torch.as_tensor(list(map(int, inp["answer_ids"])), dtype=torch.int32).to(dev)
    pix = inp["pixel_patches"].to(dev)
    if packed:
        fn = lambda: eng.score_packed(pix, grids, d, ans, repetition_penalty=pen)
    else:
        fn = lambda: eng.score_tensors(pix, grids, d["input_ids"], d["seq_lens"], d["feat_index"], d["position_ids"], ans, repetition_penalty=pen)
    assert captured_node_count(fn) == eng.last_launch_count()
    assert captured_node_count(lambda: eng.topk_last(5, repetition_penalty=pen)) == eng.last_launch_count() == 2

@pytest.mark.parametrize("frames,hw", [(2, (56, 84)), (4, (84, 56))])
def test_qwen_engine_video_grid(dev, frames, hw):
    """SURVEY 8(d) config 5: a video is a grid with t > 1 temporal patches -- same tower (windows and full attention are per
    temporal patch), video-token run in the prompt, constant temporal rope index scaled by second_per_grid."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=2)
    inp = qo.make_synthetic_inputs(cfg, 3, hw, 10, ragged=True, frames=frames)
    spg = [2.0] * 3
    o32 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], mode="fp32",
                            return_all=True, second_per_grid_ts=spg)
    o16 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], mode="bf16",
                            return_all=True, second_per_grid_ts=spg)
    eng = make_engine(cfg, sd, dev)
    p = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], [x.tolist() for x in inp["input_ids"]], inp["answer_ids"],
                          second_per_grid_ts=spg).cpu()
    lp, l32, l16 = torch.log(p), torch.log(o32["scores"]), torch.log(o16["scores"])
    gap = float((l16 - l32).abs().max())
    print(f"\n[qwen video t={frames} {hw}] engine {p.tolist()} oracle {o32['scores'].tolist()} |dlogp| {float((lp - l32).abs().max()):.3e} "
          f"(oracle bf16-vs-fp32 {gap:.3e})")
    assert float((lp - l32).abs().max()) <= 2.0 * gap + 2e-2


def test_qwen_repetition_penalty(dev):
    """SURVEY F8 / a23: the reference's scores are post-logits-processor. With a repetition penalty the engine applies HF's
    RepetitionPenaltyLogitsProcessor over each sample's own prompt ids inside the lm_head epilogue (bitmap), then 1/T, then the
    full-vocabulary softmax. Sample 0's answer id is taken from its own prompt so the label logit itself is penalised too."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=5)
    inp = qo.make_synthetic_inputs(cfg, 4, (84, 56), 12, ragged=True)
    prompts = [x.tolist() for x in inp["input_ids"]]
    answers = list(map(int, inp["answer_ids"]))
    answers[0] = prompts[0][-1]
    o32 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], answers, inp["image_of_sample"],
                            mode="fp32", return_all=True)
    o16 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], answers, inp["image_of_sample"],
                            mode="bf16", return_all=True)
    gap = float((torch.log(o16["scores"]) - torch.log(o32["scores"])).abs().max())
    eng = make_engine(cfg, sd, dev)
    base = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, answers, inp["image_of_sample"]).cpu()
    for pen, T in ((1.05, 1.0), (1.5, 1.0), (1.3, 0.5), (0.8, 1.0)):
        got = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, answers, inp["image_of_sample"], temperature=T,
                                repetition_penalty=pen).cpu()
        ref = torch.stack([qo.answer_probability(o32["logits"][b], answers[b], T, inp["input_ids"][b], pen) for b in range(4)])
        err = float((torch.log(got) - torch.log(ref)).abs().max())
        print(f"\n[qwen penalty {pen} T {T}] engine {got.tolist()} oracle {ref.tolist()} |dlogp| {err:.3e}")
        assert err <= 2.0 * gap / min(T, 1.0) + 2e-2
    # the penalty must actually move the penalised answer (sample 0) and be a no-op at 1.0
    strong = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, answers, inp["image_of_sample"], repetition_penalty=1.5).cpu()
    assert abs(float(torch.log(strong[0]) - torch.log(base[0]))) > 1e-3
    same = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, answers, inp["image_of_sample"], repetition_penalty=1.0).cpu()
    assert torch.equal(same, base)


def test_qwen_batch_invariance(dev):
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=3)
    inp = qo.make_synthetic_inputs(cfg, 3, (84, 84), 10, ragged=True)
    eng = make_engine(cfg, sd, dev)
    prompts = [x.tolist() for x in inp["input_ids"]]
    full = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"]).cpu()
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    for b in range(3):
        one = eng.score_prompts(inp["pixel_patches"][b * P:(b + 1) * P], [inp["grid_thw"][b]], [prompts[b]], [inp["answer_ids"][b]]).cpu()
        assert abs(float(torch.log(one[0]) - torch.log(full[b]))) < 2e-2


@pytest.mark.parametrize("case", ["images", "video"])
def test_qwen_engine_matches_committed_hf_golden(golden_dir, dev, case):
    """Engine (through the C ABI) against tests/golden/qwen_tiny.pt = outputs of the real transformers model: plain answer probability
    and the post-processor one (repetition penalty 1.3, temperature 0.5). Tolerance: 2x the bf16-vs-fp32 gap of the oracle + 2e-2 in log."""
    from test_qwen_host import load_qwen_golden
    blob, cfg, sd = load_qwen_golden(golden_dir)
    c = blob["cases"][case]
    inp, hf, spg = c["inputs"], c["hf"], c["second_per_grid_ts"]
    o16 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], inp["image_of_sample"],
                            mode="bf16", second_per_grid_ts=spg)
    gap = float((torch.log(o16) - torch.log(hf["probs"])).abs().max())
    eng = make_engine(cfg, sd, dev)
    prompts = [x.tolist() for x in inp["input_ids"]]
    p = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"], inp["image_of_sample"],
                          second_per_grid_ts=spg).cpu()
    e = float((torch.log(p) - torch.log(hf["probs"])).abs().max())
    pp = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"], inp["image_of_sample"], temperature=0.5,
                           repetition_penalty=1.3, second_per_grid_ts=spg).cpu()
    ep = float((torch.log(pp) - torch.log(hf["probs_penalty_1p3_T_0p5"])).abs().max())
    print(f"\n[qwen golden {case}] engine {p.tolist()} HF {hf['probs'].tolist()} |dlogp| {e:.3e}; penalised |dlogp| {ep:.3e}; "
          f"oracle bf16-vs-HF fp32 {gap:.3e}")
    assert e <= 2.0 * gap + 2e-2
    assert ep <= 2.0 * gap / 0.5 + 4e-2      # temperature 0.5 doubles every logit error


def test_qwen_trace_topk(dev):
    """forward_with_trace's top-5 alternatives (reference qwen2vl_model.py:439-447 torch.topk(softmax(scores / T), 5)): the engine's top-k pass
    over the last position against the oracle's fp32 logits, with and without temperature / repetition penalty; the answer probability
    of the scoring path must equal the probability the top-k pass assigns to the same token."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=4)
    inp = qo.make_synthetic_inputs(cfg, 3, (84, 56), 12, ragged=True)
    prompts = [x.tolist() for x in inp["input_ids"]]
    o32 = qo.qwen25vl_score(sd, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"], mode="fp32", return_all=True)
    eng = make_engine(cfg, sd, dev)
    for T, pen in ((1.0, 1.0), (0.5, 1.3)):
        p = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"], temperature=T, repetition_penalty=pen).cpu()
        ids, probs = eng.topk_last(5, temperature=T, repetition_penalty=pen)
        ids, probs = ids.cpu(), probs.cpu()
        assert bool((probs[:, :-1] >= probs[:, 1:]).all()) and bool((ids >= 0).all())
        for b in range(3):
            full = torch.stack([qo.answer_probability(o32["logits"][b], int(t), T, inp["input_ids"][b], pen) for t in ids[b]])
            assert float((torch.log(probs[b]) - torch.log(full)).abs().max()) < 6e-2 / min(T, 1.0), (probs[b], full)
            ref_top = torch.topk(torch.softmax(o32["logits"][b].float(), -1), 1).indices[0] if (T, pen) == (1.0, 1.0) else None
            if ref_top is not None and float(torch.topk(torch.softmax(o32["logits"][b].float(), -1), 2).values.diff().abs()) > 2e-2:
                assert int(ids[b, 0]) == int(ref_top)
        # an answer token that is itself in the top-k list carries exactly the score's probability
        top1 = [int(ids[b, 0]) for b in range(3)]
        p_top = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, top1, temperature=T, repetition_penalty=pen).cpu()
        ids2, probs2 = eng.topk_last(5, temperature=T, repetition_penalty=pen)
        assert torch.equal(ids2.cpu(), ids) and float((probs2.cpu()[:, 0] - p_top).abs().max()) < 1e-5


@pytest.mark.parametrize("pen", [1.0, 1.2])
def test_qwen_kv_prefix_sharing_matches_the_unshared_prefill(dev, pen):
    """SURVEY App. C item 12 / 8(f)1: M x N scoring repeats each image N times (reference score.py:104-106). With share_prefix the
    [chat prefix + vision tokens] of an image go through the language model once and every text's suffix attends to those shared K/V rows;
    causal attention makes the scores identical to the unshared prefill in real arithmetic. On the device the key tiles are cut at
    different places (prefix tiles, then the suffix's own tiles), so the online-softmax reference of a row -- and with it the bf16 rounding
    of P = 2^(s - m) -- can differ: image 0 (prefix longer than one 128-key tile: same first tile, same reference) comes out bit-identical,
    image 1 (17-row prefix) moves by bf16 noise. Bound: twice the oracle's own bf16-vs-fp32 gap on the same inputs."""
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    sd = qo.make_synthetic_state_dict(cfg, seed=6)
    g = torch.Generator().manual_seed(3)
    grids = [(1, 12, 10), (1, 6, 8)]                       # 30 and 12 vision tokens -> prefixes of 34 / 16 rows; with the text > 128 rows for image 0?
    grids = [(1, 24, 22), (1, 6, 8)]                       # 132 vision tokens: the shared prefix spans two 128-key tiles
    patches = torch.randn(sum(t * h * w for t, h, w in grids), cfg.patch_dim, generator=g)
    ntok = [t * h * w // 4 for t, h, w in grids]
    prompts, img = [], []
    for i in (0, 1):
        for k in range(3):
            prompts.append([5, 6, 7, 8] + [cfg.image_token_id] * ntok[i] + [9] + torch.randint(0, 500, (5 + 3 * k,), generator=g).tolist())
            img.append(i)
    answers = [9, 11, 13, 9, 11, 500]
    eng = make_engine(cfg, sd, dev)
    plain = eng.score_prompts(patches, grids, prompts, answers, image_of_sample=img, repetition_penalty=pen, share_prefix=False).cpu()
    shared = eng.score_prompts(patches, grids, prompts, answers, image_of_sample=img, repetition_penalty=pen, share_prefix=True).cpu()
    ids_s, p_s = eng.topk_last(3, repetition_penalty=pen)
    auto = eng.score_prompts(patches, grids, prompts, answers, image_of_sample=img, repetition_penalty=pen).cpu()
    print(f"\n[prefix sharing pen={pen}] plain {plain.tolist()} shared {shared.tolist()}")
    assert torch.equal(shared, auto)
    o32 = qo.qwen25vl_score(sd, cfg, patches, grids, [torch.tensor(p) for p in prompts], answers, img, mode="fp32", repetition_penalty=pen)
    o16 = qo.qwen25vl_score(sd, cfg, patches, grids, [torch.tensor(p) for p in prompts], answers, img, mode="bf16", repetition_penalty=pen)
    gap = float((torch.log(o16) - torch.log(o32)).abs().max())
    d = (torch.log(shared) - torch.log(plain)).abs()
    print(f"   |dlog p| shared vs plain {d.tolist()}  oracle bf16-vs-fp32 gap {gap:.3e}")
    assert float(d[:3].max()) < 1e-4            # image 0: identical first key tile -> identical softmax reference
    assert float(d.max()) <= 2.0 * gap + 2e-3
    assert float((torch.log(shared) - torch.log(o32)).abs().max()) <= 2.0 * gap + 2e-2
    assert float((torch.log(plain) - torch.log(o32)).abs().max()) <= 2.0 * gap + 2e-2
    # trace top-k works after a packed call too
    eng.score_prompts(patches, grids, prompts, answers, image_of_sample=img, repetition_penalty=pen, share_prefix=False)
    ids_p, p_p = eng.topk_last(3, repetition_penalty=pen)
    assert torch.equal(ids_s.cpu()[:, 0], ids_p.cpu()[:, 0]) or float((p_s.cpu() - p_p.cpu()).abs().max()) < 1e-2

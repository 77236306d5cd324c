"""Qwen2.5-VL-3B at production width on a real H100: all 36 decoder and 32 vision layers, tied lm_head, 8 query heads per K/V head,
against the real transformers Qwen2_5_VLForConditionalGeneration (tie_word_embeddings=True) in bf16 with sdpa on the same GPU and weights,
as test_gpu_fullwidth.py and test_gpu_qwen_generate.py do for the 7B: the calibrated scores at 1e-3, and greedy generation."""
import dataclasses
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import qwen25vl_oracle as qo
from qwen_tied import EMBED, build_hf_qwen_tied, tied_state_dict

TOL = 1e-3


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def configs():
    """(oracle config with the 3B's dims, the engine's table entry)."""
    from t2v_metrics_b200.config import QWEN25VL_MODELS
    ecfg = QWEN25VL_MODELS["qwen2.5-vl-3b"]["config"]()
    fields = {f.name for f in dataclasses.fields(qo.Qwen25VLConfig)}
    return qo.Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(ecfg).items() if k in fields}), ecfg


def test_qwen25vl_3b_matches_reference_bf16_on_this_gpu(dev):
    """B = 2, 448x448 images (256 vision tokens) + 64 text ids: the reference recipe (generate(max_new_tokens=1, output_scores=True) per
    sample) on the tied HF model vs ONE engine prefill. The answer row is calibrated on HF's final hidden states; with tied weights that
    row is also the answer token's embedding, which no prompt contains."""
    import hf_reference as hf
    from t2v_metrics_b200.engine import QwenVLEngine
    cfg, ecfg = configs()
    B, answer = 2, 9454
    sd = tied_state_dict(cfg, seed=0, gen_device=dev)
    inp = qo.make_synthetic_inputs(cfg, B, (448, 448), 64, seed=1, ragged=True, answer_id=answer)
    assert all(answer not in x.tolist() for x in inp["input_ids"])
    model = build_hf_qwen_tied(cfg, sd, dtype=torch.bfloat16, device=dev, attn="sdpa")
    score = lambda m, T=1.0: hf.hf_qwen_reference_scores(m, cfg, inp["pixel_patches"], inp["grid_thw"], inp["input_ids"], inp["answer_ids"],
                                                          temperature=T, return_hidden=True)
    _, hid = score(model)
    row = hf.calibrate_rows(hid, model.lm_head.weight, answer, torch.tensor([-1.5, 1.5]))
    model.lm_head.weight.data[answer] = row.to(dev)
    assert torch.equal(model.model.language_model.embed_tokens.weight[answer], row.to(dev))
    sd[EMBED][answer] = row.to(sd[EMBED].device)
    ref, hid = score(model)
    refT, _ = score(model, 0.7)
    del model
    _free()
    eng = QwenVLEngine(ecfg, dev)
    eng.load_state_dict(sd)
    assert eng._weights["llm.lm_head"].data_ptr() == eng._weights["llm.embed"].data_ptr()
    prompts = [x.tolist() for x in inp["input_ids"]]
    p = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"])
    torch.cuda.synchronize()
    S = max(len(x) for x in prompts)
    dbg = eng.debug_tensors(B, S, inp["pixel_patches"].shape[0])
    h = dbg["last_hidden"].float().cpu()
    hrel = float((h - hid.cpu()).norm() / hid.cpu().norm())
    pT = eng.score_prompts(inp["pixel_patches"], inp["grid_thw"], prompts, inp["answer_ids"], temperature=0.7).cpu()
    p = p.cpu()
    err, errT = float((p - ref).abs().max()), float((pT - refT).abs().max())
    print(f"\n[qwen-3b] engine {p.tolist()}  HF bf16 sdpa GPU {ref.tolist()}  max|dp| {err:.3e}; T=0.7: engine {pT.tolist()} HF {refT.tolist()} "
          f"max|dp| {errT:.3e}\n[qwen-3b] last hidden state rel.err {hrel:.2e} | launches {eng.last_launch_count()}")
    del sd, eng
    _free()
    assert float(ref.min()) > 0.08 and float(ref.max()) < 0.92 and float(ref.max() - ref.min()) > 0.4
    assert err <= TOL and errT <= 2 * TOL, (p, ref, pT, refT)


def test_qwen25vl_3b_generate_matches_reference_bf16_on_this_gpu(dev):
    """B = 2, 448x448 images + 32 text ids, 16 new tokens: the engine's decode loop (split-K decode GEMMs, group-8 decode attention, tied
    lm_head) against HF bf16 sdpa generate(do_sample=False) per sample. As for the 7B: at every step where the engine's path still equals
    HF's, the engine's token scores within 0.25 of HF's best processed score at that step."""
    from t2v_metrics_b200.engine import QwenVLEngine
    cfg, ecfg = configs()
    B, N = 2, 16
    sd = tied_state_dict(cfg, seed=0, gen_device=dev)
    inp = qo.make_synthetic_inputs(cfg, B, (448, 448), 32, seed=1, ragged=True)
    model = build_hf_qwen_tied(cfg, sd, dtype=torch.bfloat16, device=dev, attn="sdpa")
    P = inp["grid_thw"][0][1] * inp["grid_thw"][0][2]
    ref_ids, ref_scores = [], []
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
    _free()
    eng = QwenVLEngine(ecfg, dev)
    eng.load_state_dict(sd)
    toks = eng.generate_prompts(inp["pixel_patches"], inp["grid_thw"], [x.tolist() for x in inp["input_ids"]], N, ())
    compared = 0
    for b in range(B):
        scores = ref_scores[b]
        top2 = scores.topk(2, dim=-1).values
        shared = next((t for t in range(N) if toks[b][t] != ref_ids[b][t]), N)
        print(f"\n[qwen-3b generate] b={b} engine {toks[b]}\n    HF bf16 {ref_ids[b]}\n    HF margins "
              f"{[round(float(x), 3) for x in top2[:, 0] - top2[:, 1]]} shared prefix {shared}")
        for t in range(min(shared + 1, N)):
            assert float(scores[t].max() - scores[t, toks[b][t]]) <= 0.25, (b, t)
        compared += min(shared + 1, N)
    del sd, eng
    _free()
    assert compared >= 4

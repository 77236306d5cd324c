"""Qwen2.5-VL video inputs on a real H100: frame-stack pre-processing on the device bit for bit against the CPU restatement, and the
plugin's forward / forward_with_trace / generate / k = 4 rollout on 4-D .npy stacks against the committed HF video golden."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

from oracle import qwen25vl_oracle as qo
from t2v_metrics_b200 import qwen_host
from t2v_metrics_b200.models.vqascore_models.qwen_utils import (qwen_image_to_patches, qwen_video_to_patches, default_question_template,
                                                                default_answer_template)
from test_qwen_video_host import CharTokenizer, load_video_golden


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


def _items(seed=7):
    """Stacks of 4, 5 (odd), 2 resized and 3 larger resized frames, a still image and a 1-frame video, in one call."""
    rng = np.random.default_rng(seed)
    u8 = lambda *s: rng.integers(0, 256, s, dtype=np.uint8)
    return [u8(4, 56, 84, 3), u8(5, 84, 112, 3), u8(123, 77, 3), u8(2, 50, 90, 3), u8(3, 300, 500, 3), u8(1, 61, 97, 3)]


def _reference(items):
    rows = [qwen_video_to_patches(a) if a.ndim == 4 else qwen_image_to_patches(Image.fromarray(a)) for a in items]
    return torch.cat([r[0] for r in rows]), [tuple(r[1]) for r in rows]


@pytest.mark.parametrize("dtype,on_device", [(torch.float32, False), (torch.bfloat16, False), (torch.float32, True)])
def test_device_video_preprocess_is_bit_exact(dev, dtype, on_device):
    from t2v_metrics_b200.engine import qwen_preprocess_video_u8
    items = _items()
    ref, grids = _reference(items)
    src = [torch.from_numpy(a).to(dev) if on_device else torch.from_numpy(a) for a in items]
    got, g = qwen_preprocess_video_u8(src, dev, out_dtype=dtype)
    assert g == grids and grids[0] == (2, 4, 6) and grids[1] == (3, 6, 8) and grids[2][0] == 1 and grids[5][0] == 1
    assert torch.equal(got.cpu(), ref.to(dtype))


def test_device_video_preprocess_is_one_kernel_launch(dev):
    """The whole mixed call, driven through the C entry point under stream capture, is the table upload plus ONE kernel."""
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import CLIP_MEAN, CLIP_STD, _ptr
    lib = _lib.load()
    items = _items(seed=8)
    ref, grids = _reference(items)
    n = len(items)
    nf = [a.shape[0] if a.ndim == 4 else 1 for a in items]
    hs, ws, vid = [a.shape[-3] for a in items], [a.shape[-2] for a in items], [int(a.ndim == 4) for a in items]
    offs, o = [], 0
    for a, k in zip(items, nf):
        offs += [o + f * a[..., 0].size // k * 3 for f in range(k)]
        o += a.size
    src = torch.from_numpy(np.concatenate([a.reshape(-1) for a in items])).to(dev)
    I32 = lambda v: (C.c_int32 * n)(*v)
    args = (I32(nf), I32(hs), I32(ws), I32(vid))
    rows, need = C.c_int64(0), C.c_size_t(0)
    thw = (C.c_int32 * (3 * n))()
    assert lib.vqa_qwen_preprocess_video_plan(*args, n, 14, 2, 2, 56 * 56, 14 * 14 * 4 * 1280, thw, C.byref(rows), C.byref(need)) == 0
    assert [tuple(thw[3 * i:3 * i + 3]) for i in range(n)] == grids and rows.value == ref.shape[0]
    out = torch.full((rows.value, 1176), float("nan"), device=dev)
    wsb = torch.empty(need.value, dtype=torch.uint8, device=dev)
    staging = torch.empty(need.value, dtype=torch.uint8, pin_memory=True)

    def call():      # on the current stream, which is the capturing one inside torch.cuda.graph
        rc = lib.vqa_qwen_preprocess_video(_ptr(src), (C.c_int64 * len(offs))(*offs), *args, n, 14, 2, 2, 56 * 56, 14 * 14 * 4 * 1280,
                                           (C.c_float * 3)(*CLIP_MEAN), (C.c_float * 3)(*CLIP_STD), _ptr(out), _lib.VQA_DTYPE_F32, _ptr(wsb),
                                           need.value, staging.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        assert rc == 0, _lib.last_error(None)
    call()
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), ref)
    out.fill_(float("nan"))
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        call()
    nodes = C.c_size_t(0)
    assert C.CDLL("libcuda.so.1").cuGraphGetNodes(C.c_void_p(graph.raw_cuda_graph()), None, C.byref(nodes)) == 0
    assert nodes.value == 2
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), ref)


# ------------------------------------------------------------------------------------------------ plugin against the HF video golden
@pytest.fixture(scope="module")
def golden(golden_dir, dev, tmp_path_factory):
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    blob, ocfg, sd = load_video_golden(golden_dir)
    d = tmp_path_factory.mktemp("video")
    paths = []
    for i, s in enumerate(blob["stacks"]):
        np.save(d / f"v{i}.npy", s["frames"].numpy())
        paths.append(str(d / f"v{i}.npy"))
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    cfg = Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(ocfg).items() if k in fields})
    model = Qwen2VLModel("qwen2.5-vl-7b", device=str(dev), tokenizer=CharTokenizer(), state_dict=dict(sd), config=cfg,
                         checkpoint=str(d / "none.bin"))
    return blob, ocfg, sd, model, paths


def _oracle_gap(blob, ocfg, sd, i):
    """The oracle's bf16-vs-HF-fp32 gap of stack i's scoring prompt: logits and log-probability."""
    s = blob["stacks"][i]
    o = qo.qwen25vl_score(sd, ocfg, s["patches"], [tuple(s["grid_thw"])], [torch.tensor(s["score_prompt"])], [s["answer_ids"][0]],
                          mode="bf16", return_all=True, second_per_grid_ts=[s["second_per_grid_ts"]])
    return float((o["logits"][0] - s["logits"]).abs().max()), abs(math.log(float(o["scores"][0])) - math.log(s["probs"]))


def test_plugin_forward_on_frame_stacks_matches_the_hf_golden(golden):
    blob, ocfg, sd, model, paths = golden
    texts = blob["texts"]
    got = model.forward(paths, texts)
    pen = model.forward(paths, texts, temperature=0.5, repetition_penalty=1.3)
    assert torch.equal(model.forward(paths, texts, fps=4.0), got)
    for i, s in enumerate(blob["stacks"]):
        _, gap = _oracle_gap(blob, ocfg, sd, i)
        e = abs(math.log(float(got[i])) - math.log(s["probs"]))
        ep = abs(math.log(float(pen[i])) - math.log(s["probs_penalty_1p3_T_0p5"]))
        print(f"\n[video golden {i}] engine {float(got[i]):.6e} HF {s['probs']:.6e} |dlogp| {e:.3e}; penalised {ep:.3e}; oracle gap {gap:.3e}")
        assert e <= 2.0 * gap + 2e-2
        assert ep <= 2.0 * gap / 0.5 + 4e-2


def test_plugin_trace_top5_equals_hf(golden):
    """Top-5 ids of the last position against HF's, at every rank whose neighbouring logit gaps exceed twice the oracle's bf16 gap."""
    blob, ocfg, sd, model, paths = golden
    _, traces = model.forward_with_trace(paths, blob["texts"])
    compared = 0
    for i, (s, tr) in enumerate(zip(blob["stacks"], traces)):
        thr = 2.0 * _oracle_gap(blob, ocfg, sd, i)[0] + 1e-3
        v, hf_ids = s["logits"].topk(6)
        ids = [a["token_id"] for a in tr["token_details"][0]["top_alternatives"]]
        for r in range(5):
            if (r == 0 or float(v[r - 1] - v[r]) > thr) and float(v[r] - v[r + 1]) > thr:
                assert ids[r] == int(hf_ids[r]), (i, r, ids, hf_ids.tolist())
                compared += 1
    assert compared >= 5


def _decisive(margins, thr=1e-2):
    return next((t for t, m in enumerate(margins.tolist()) if m < thr), len(margins))


def test_plugin_generate_on_frame_stacks_equals_the_golden(golden):
    blob, ocfg, sd, model, paths = golden
    out = model.generate(paths, blob["texts"], max_new_tokens=blob["gen_steps"])
    compared = 0
    for s, text in zip(blob["stacks"], out):
        n = _decisive(s["generate_margins"])
        print(f"\n[video generate] engine {text!r} HF {s['generate_ids']} decisive {n}")
        assert text.split()[:n] == [str(t) for t in s["generate_ids"][:n]]
        compared += n
    assert compared >= 12


def test_plugin_rollout_on_frame_stacks_matches_the_golden(golden):
    """k = 4 greedy rollout of the scoring prompt: tokens equal HF's over the decisive steps, and there each answer probability is within
    the single-prefill bound of HF's."""
    blob, ocfg, sd, model, paths = golden
    res = model._rollout(paths, blob["texts"], default_question_template, default_answer_template, blob["rollout_steps"], 1.0, 1.0,
                         "forward", 0)
    scores = model.forward(paths, blob["texts"], max_new_tokens=blob["rollout_steps"])
    full = 0
    for i, (s, r) in enumerate(zip(blob["stacks"], res)):
        n = _decisive(s["rollout_margins"])
        _, gap = _oracle_gap(blob, ocfg, sd, i)
        hf = qwen_host.rollout_answer_score(s["rollout_ids"], s["rollout_probs"].log(), s["answer_ids"], {638, 639}, "forward")
        print(f"\n[video rollout {i}] engine {r['tokens']} HF {s['rollout_ids']} decisive {n} probs {r['probs']} HF {hf['probs']}")
        assert r["tokens"][:n] == s["rollout_ids"][:n]
        assert float(scores[i]) == pytest.approx(r["score"], rel=1e-6)
        if n == len(s["rollout_ids"]):
            full += 1
            assert r["steps"] == hf["steps"]
            assert max(abs(math.log(a) - math.log(b)) for a, b in zip(r["probs"], hf["probs"])) <= 2.0 * gap + 2e-2
    assert full >= 2


def test_score_forward_over_videos_equals_pairwise_calls_and_prefix_sharing(golden):
    """Score.forward over 2 videos x 3 texts (one plugin call, each video encoded once, prefixes shared) equals one call per pair, and
    the engine's prefix-shared prefill equals the unshared one within twice the oracle's bf16 gap."""
    import t2v_metrics_b200 as t2v
    blob, ocfg, sd, model, paths = golden
    scorer = t2v.VQAScore(model="qwen2.5-vl-7b", device="cuda", tokenizer=CharTokenizer(), state_dict=dict(sd), config=model.cfg,
                          checkpoint=model._checkpoint)
    model = scorer.model
    texts = ["a red car", "two dogs on a sofa", "x"]
    out = scorer(images=paths[:2], texts=texts).cpu()
    pair = torch.tensor([[float(model.forward([p], [t])[0]) for t in texts] for p in paths[:2]])
    gap = max(_oracle_gap(blob, ocfg, sd, i)[1] for i in (0, 1))
    print(f"\n[video Score.forward] batched {out.tolist()} pairwise {pair.tolist()}")
    assert float((out.log() - pair.log()).abs().max()) <= 2.0 * gap + 1e-6
    from t2v_metrics_b200.models.vqascore_models.qwen_utils import build_prompt_ids
    patches, grids = model.load_images(paths[:2])
    prompts = [build_prompt_ids(model.tokenizer, default_question_template.format(t), math.prod(grids[v]) // 4, ocfg.video_token_id)
               for v in (0, 1) for t in texts]
    kw = dict(image_of_sample=[0, 0, 0, 1, 1, 1], second_per_grid_ts=[2 / 24] * 2)
    plain = model.engine.score_prompts(patches, grids, prompts, [89] * 6, share_prefix=False, **kw).cpu()
    shared = model.engine.score_prompts(patches, grids, prompts, [89] * 6, share_prefix=True, **kw).cpu()
    assert torch.equal(shared, out.view(-1))
    assert float((plain.log() - shared.log()).abs().max()) <= 2.0 * gap + 1e-6

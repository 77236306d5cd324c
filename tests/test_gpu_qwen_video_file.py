"""Qwen2.5-VL video FILES on a real H100: the device's antialiased bicubic resize against torchvision on the host CPU (equal except at
rounding ties), its patch rows bit for bit against the restatement built from the device's own uint8 frames, one kernel per slice, and
the plugin's forward / forward_with_trace / generate / k = 4 rollout on the committed clip against the HF golden. The bit-exact tests of
the device resize, against a host restatement of its fp32 arithmetic under every row-tile plan, are in test_gpu_qwen_video_aa_exact.py;
the torchvision comparison here stays the check against the reference's own implementation."""
import ctypes as C
import dataclasses
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

from oracle import qwen25vl_oracle as qo
from t2v_metrics_b200 import qwen_host
from t2v_metrics_b200.models.vqascore_models import qwen_utils as qu
from t2v_metrics_b200.models.vqascore_models.qwen_utils import default_answer_template, default_question_template
from test_qwen_video_host import CharTokenizer
from test_qwen_video_file_host import load_file_golden, smooth_frames, write_clip, golden_patches


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


def device_levels(rows, grid, patch=14, temporal=2, merge=2):
    """Patch rows (fp32, values of the normalisation table) -> the uint8 frames [t*temporal, rh, rw, 3] behind them; every value must be
    one of the table's."""
    from t2v_metrics_b200.engine import CLIP_MEAN, CLIP_STD
    table = (torch.arange(256, dtype=torch.float32)[None] / 255.0 - torch.tensor(CLIP_MEAN)[:, None]) / torch.tensor(CLIP_STD)[:, None]
    t, gh, gw = grid
    x = rows.view(t, gh // merge, gw // merge, merge, merge, 3, temporal, patch, patch).permute(0, 6, 5, 1, 3, 7, 2, 4, 8)
    x = x.reshape(t * temporal, 3, gh * patch, gw * patch)
    lv = torch.stack([torch.searchsorted(table[c], x[:, c].contiguous()) for c in range(3)], 1).clamp(max=255)
    assert torch.equal(torch.stack([table[c][lv[:, c]] for c in range(3)], 1), x), "a value outside the normalisation table"
    return lv.to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def torch_fp32(frames, size):
    """torch's fp32 resize before rounding (what torchvision rounds)."""
    x = torch.from_numpy(frames).permute(0, 3, 1, 2).float()
    return torch.nn.functional.interpolate(x, size=list(size), mode="bicubic", antialias=True, align_corners=False).permute(0, 2, 3, 1)


CASES = [((480, 640), (336, 448)), ((360, 640), (252, 448)), ((240, 320), (280, 364)), ((97, 61), (392, 252)), ((1080, 1920), (280, 504)),
         ((333, 501), (308, 476)), ((64, 96), (280, 392))]


@pytest.mark.parametrize("src,size", CASES)
def test_device_resize_equals_torchvision_except_at_rounding_ties(dev, src, size):
    from t2v_metrics_b200.engine import qwen_preprocess_video_file_u8
    n = 3
    frames = np.random.default_rng(src[0] * 3 + src[1]).integers(0, 256, (n, *src, 3), dtype=np.uint8)
    rows, grid = qwen_preprocess_video_file_u8(torch.from_numpy(frames), size, dev)
    assert grid == ((n + 1) // 2, size[0] // 14, size[1] // 14)
    got = device_levels(rows.cpu(), grid)[:n]
    want, _, _ = qu.qwen_video_file_to_patches(frames, size)
    diff = got.int() - want.int()
    bad = diff != 0
    exact = torch_fp32(frames, size)[bad]
    print(f"\n[aa resize {src} -> {size}] {int(bad.sum())} of {bad.numel()} elements differ from torchvision; "
          f"max |fp32 - (k + 0.5)| there {float((exact - exact.floor() - 0.5).abs().max()) if bad.any() else 0.0:.2e}")
    assert int(diff.abs().max()) <= 1
    assert bool(((exact - exact.floor() - 0.5).abs() <= 1e-3).all())
    # the patch rows are exactly the restatement's layout of the device's own frames, also for the padded odd last frame
    ref, g = qu._video_patch_rows(got.permute(0, 3, 1, 2).float(), 14, 2, 2)
    assert g == grid and torch.equal(rows.cpu(), ref)


@pytest.mark.parametrize("dtype,on_device,slice_frames", [(torch.float32, False, 2), (torch.bfloat16, False, 3), (torch.float32, True, 1)])
def test_sliced_calls_equal_the_restatement_in_fp32_and_bf16(dev, monkeypatch, dtype, on_device, slice_frames):
    from t2v_metrics_b200 import engine
    frames = smooth_frames(7, 360, 640, seed=1)
    size = (280, 504)
    whole, grid = engine.qwen_preprocess_video_file_u8(torch.from_numpy(frames), size, dev)
    ref, g = qu._video_patch_rows(device_levels(whole.cpu(), grid)[:7].permute(0, 3, 1, 2).float(), 14, 2, 2)
    assert g == grid == (4, 20, 36) and torch.equal(whole.cpu(), ref)
    monkeypatch.setattr(engine, "VIDEO_SLICE_BYTES", slice_frames * 360 * 640 * 3)
    src = torch.from_numpy(frames).to(dev) if on_device else torch.from_numpy(frames)
    got, _ = engine.qwen_preprocess_video_file_u8(src, size, dev, out_dtype=dtype)
    assert torch.equal(got.cpu(), ref.to(dtype))
    # an iterable of slices of uneven sizes
    got, _ = engine.qwen_preprocess_video_file_u8((torch.from_numpy(frames[a:b]) for a, b in ((0, 1), (1, 5), (5, 7))), size, dev,
                                                  n_frames=7, out_dtype=dtype)
    assert torch.equal(got.cpu(), ref.to(dtype))


def test_one_slice_is_the_table_upload_plus_one_kernel(dev):
    from t2v_metrics_b200 import _lib
    from t2v_metrics_b200.engine import CLIP_MEAN, CLIP_STD, _aa_bicubic_taps, _ptr, qwen_preprocess_video_file_u8
    lib = _lib.load()
    frames = np.random.default_rng(5).integers(0, 256, (4, 240, 320, 3), dtype=np.uint8)
    size = (280, 364)
    ref, grid = qwen_preprocess_video_file_u8(torch.from_numpy(frames), size, dev)
    (fh, wh, th), (fv, wv, tv) = _aa_bicubic_taps(320, size[1]), _aa_bicubic_taps(240, size[0])
    i32 = lambda t: C.cast(t.data_ptr(), C.POINTER(C.c_int32))
    f32 = lambda t: C.cast(t.data_ptr(), C.POINTER(C.c_float))
    rows, need = C.c_int64(0), C.c_size_t(0)
    assert lib.vqa_qwen_preprocess_video_aa_plan(240, 320, *size, i32(fh), th, i32(fv), tv, 14, 2, 2, 4, C.byref(rows), C.byref(need)) == 0
    assert rows.value == ref.shape[0]
    src = torch.from_numpy(frames).to(dev)
    out = torch.full_like(ref, float("nan"))
    wsb = torch.empty(need.value, dtype=torch.uint8, device=dev)
    staging = torch.empty(need.value, dtype=torch.uint8, pin_memory=True)

    def call():
        rc = lib.vqa_qwen_preprocess_video_aa(_ptr(src), 4, 0, 4, 240, 320, *size, i32(fh), f32(wh), th, i32(fv), f32(wv), tv, 14, 2, 2,
                                              (C.c_float * 3)(*CLIP_MEAN), (C.c_float * 3)(*CLIP_STD), _ptr(out), _lib.VQA_DTYPE_F32,
                                              _ptr(wsb), need.value, staging.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        assert rc == 0, _lib.last_error(None)
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        call()
    nodes = C.c_size_t(0)
    assert C.CDLL("libcuda.so.1").cuGraphGetNodes(C.c_void_p(graph.raw_cuda_graph()), None, C.byref(nodes)) == 0
    assert nodes.value == 2
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------ plugin against the HF file golden
@pytest.fixture(scope="module")
def golden(golden_dir, dev, tmp_path_factory):
    from t2v_metrics_b200.config import Qwen25VLConfig
    from t2v_metrics_b200.models.vqascore_models.qwen2vl_model import Qwen2VLModel
    blob, ocfg, sd = load_file_golden(golden_dir)
    d = tmp_path_factory.mktemp("videofile")
    clip = str(d / ("clip" + blob["clip_ext"]))
    with open(clip, "wb") as f:
        f.write(blob["clip"])
    fields = {f.name for f in dataclasses.fields(Qwen25VLConfig)}
    cfg = Qwen25VLConfig(**{k: v for k, v in dataclasses.asdict(ocfg).items() if k in fields})
    model = Qwen2VLModel("qwen2.5-vl-7b", device=str(dev), tokenizer=CharTokenizer(), state_dict=dict(sd), config=cfg,
                         checkpoint=str(d / "none.bin"), video_reader="opencv")
    gaps = {}
    for key, r in blob["runs"].items():
        patches = golden_patches(clip, r)
        o = qo.qwen25vl_score(sd, ocfg, patches, [tuple(r["grid_thw"])], [torch.tensor(r["score_prompt"])], [r["answer_ids"][0]],
                              mode="bf16", return_all=True, second_per_grid_ts=[r["second_per_grid_ts"]])
        gaps[key] = (float((o["logits"][0] - r["logits"]).abs().max()), abs(math.log(float(o["scores"][0])) - math.log(r["probs"])))
    return blob, model, clip, gaps, d


def test_plugin_forward_on_a_video_file_matches_the_hf_golden(golden):
    blob, model, clip, gaps, _ = golden
    for fps, key in ((None, "8.0"), (8.0, "8.0"), ("dynamic", "dynamic")):
        got = float(model.forward([clip], [blob["text"]], fps=fps)[0])
        e = abs(math.log(got) - math.log(blob["runs"][key]["probs"]))
        print(f"\n[video file fps={fps}] engine {got:.6e} HF {blob['runs'][key]['probs']:.6e} |dlogp| {e:.3e} oracle gap {gaps[key][1]:.3e}")
        assert e <= 2.0 * gaps[key][1] + 2e-2


def test_plugin_trace_top5_on_a_video_file_equals_hf(golden):
    blob, model, clip, gaps, _ = golden
    r = blob["runs"]["8.0"]
    _, (tr,) = model.forward_with_trace([clip], [blob["text"]], fps=8.0)
    thr = 2.0 * gaps["8.0"][0] + 1e-3
    v, hf_ids = r["logits"].topk(6)
    ids = [a["token_id"] for a in tr["token_details"][0]["top_alternatives"]]
    compared = 0
    for k in range(5):
        if (k == 0 or float(v[k - 1] - v[k]) > thr) and float(v[k] - v[k + 1]) > thr:
            assert ids[k] == int(hf_ids[k]), (k, ids, hf_ids.tolist())
            compared += 1
    print(f"\n[video file trace] engine {ids} HF {hf_ids.tolist()[:5]} compared {compared}")
    assert compared >= 2


def _decisive(margins, thr=1e-2):
    return next((t for t, m in enumerate(margins.tolist()) if m < thr), len(margins))


def test_plugin_generate_and_rollout_on_a_video_file_equal_the_golden(golden):
    blob, model, clip, gaps, _ = golden
    r = blob["runs"]["8.0"]
    (text,) = model.generate([clip], [blob["text"]], max_new_tokens=blob["gen_steps"], fps=8.0)
    n = _decisive(r["generate_margins"])
    print(f"\n[video file generate] engine {text!r} HF {r['generate_ids']} decisive {n}")
    assert text.split()[:n] == [str(t) for t in r["generate_ids"][:n]] and n >= 3
    (res,) = model._rollout([clip], [blob["text"]], default_question_template, default_answer_template, blob["rollout_steps"], 1.0, 1.0,
                            "forward", 0, 8.0)
    score = float(model.forward([clip], [blob["text"]], max_new_tokens=blob["rollout_steps"], fps=8.0)[0])
    n = _decisive(r["rollout_margins"])
    hf = qwen_host.rollout_answer_score(r["rollout_ids"], r["rollout_probs"].log(), r["answer_ids"], {638, 639}, "forward")
    print(f"\n[video file rollout] engine {res['tokens']} HF {r['rollout_ids']} decisive {n} probs {res['probs']} HF {hf['probs']}")
    assert res["tokens"][:n] == r["rollout_ids"][:n] and score == pytest.approx(res["score"], rel=1e-6)
    if n == len(r["rollout_ids"]):
        assert res["steps"] == hf["steps"]
        assert max(abs(math.log(a) - math.log(b)) for a, b in zip(res["probs"], hf["probs"])) <= 2.0 * gaps["8.0"][1] + 2e-2


def test_score_forward_over_files_equals_pairwise_calls_and_mixes_with_stills_and_stacks(golden):
    blob, model, clip, gaps, d = golden
    other = str(d / "other.mkv")
    write_clip(other, smooth_frames(9, 120, 160, seed=7), 6.0)
    from t2v_metrics_b200.score import Score

    class S(Score):                  # the Score front end around the golden's plugin (video_mode "direct", an OpenCV reader)
        def prepare_scoremodel(self, name, device, cache_dir, **kw):
            return model

        def list_all_models(self):
            return ["qwen2.5-vl-7b"]
    scorer = S("qwen2.5-vl-7b", device="cuda")
    texts = ["a red car", "two dogs on a sofa", "x"]
    out = scorer(images=[clip, other], texts=texts).cpu()
    pair = torch.tensor([[float(model.forward([p], [t])[0]) for t in texts] for p in (clip, other)])
    print(f"\n[video file Score.forward] batched {out.tolist()} pairwise {pair.tolist()}")
    assert float((out.log() - pair.log()).abs().max()) <= 2.0 * gaps["8.0"][1] + 1e-6
    # a file, a still and a frame stack in one call score as they do alone
    img, stack = str(d / "still.png"), str(d / "stack.npy")
    Image.fromarray(smooth_frames(1, 100, 140, seed=9)[0]).save(img)
    np.save(stack, smooth_frames(3, 84, 112, seed=11))
    mixed = model.forward([clip, img, stack, clip], ["a", "b", "c", "d"])
    alone = torch.cat([model.forward([p], [t]) for p, t in ((clip, "a"), (img, "b"), (stack, "c"), (clip, "d"))])
    assert float((mixed.log() - alone.log()).abs().max()) <= 2.0 * gaps["8.0"][1] + 1e-6

"""Qwen2.5-VL video FILES, CPU side: qwen_vl_utils' frame sampling and pixel budget (qwen_utils.qwen_video_file_plan) against a literal
restatement, the OpenCV reader on synthesized .mp4 / .avi / .mkv clips, the file restatement (torchvision resize + processor layout)
against the installed Qwen2VLVideoProcessor, the processor's second_per_grid_ts for a file's frames, the plugin's wiring of files onto a
stand-in engine, the refusal without a reader, and Score.forward / batch_forward passing files through only to a plugin that decodes."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import qwen25vl_oracle as qo
from t2v_metrics_b200 import engine as eng_mod
from t2v_metrics_b200.models.vqascore_models import qwen2vl_model as qm
from t2v_metrics_b200.models.vqascore_models import qwen_utils as qu
from test_qwen_host import TINY
from test_qwen_video_host import CharTokenizer, SPG_VIDEO, _Engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def vl_utils_fetch_plan(ele, total_frames, video_fps, height, width, total_pixels=qu.VIDEO_TOTAL_PIXELS):
    """qwen_vl_utils 0.0.8 smart_nframes / _read_video_* / fetch_video, transcribed line by line for the test."""
    round_by_factor = lambda n, f: round(n / f) * f
    ceil_by_factor = lambda n, f: math.ceil(n / f) * f
    floor_by_factor = lambda n, f: math.floor(n / f) * f
    fps = ele.get("fps", 2.0)
    min_frames = ceil_by_factor(ele.get("min_frames", 4), 2)
    max_frames = floor_by_factor(ele.get("max_frames", min(768, total_frames)), 2)
    nframes = total_frames / video_fps * fps
    nframes = min(min(max(nframes, min_frames), max_frames), total_frames)
    nframes = floor_by_factor(nframes, 2)
    if not (2 <= nframes and nframes <= total_frames):
        raise ValueError(f"nframes should in interval [2, {total_frames}], but got {nframes}.")
    idx = torch.linspace(0, total_frames - 1, nframes).round().long().tolist()
    sample_fps = nframes / max(total_frames, 1e-6) * video_fps
    min_pixels = ele.get("min_pixels", 128 * 28 * 28)
    max_pixels = max(min(768 * 28 * 28, total_pixels / nframes * 2), int(min_pixels * 1.05))
    max_pixels = min(ele.get("max_pixels", max_pixels), max_pixels)
    # qwen_vl_utils smart_resize
    h_bar, w_bar = max(28, round_by_factor(height, 28)), max(28, round_by_factor(width, 28))
    if h_bar * w_bar > max_pixels:
        beta = math.sqrt((height * width) / max_pixels)
        h_bar, w_bar = floor_by_factor(height / beta, 28), floor_by_factor(width / beta, 28)
    elif h_bar * w_bar < min_pixels:
        beta = math.sqrt(min_pixels / (height * width))
        h_bar, w_bar = ceil_by_factor(height * beta, 28), ceil_by_factor(width * beta, 28)
    return idx, sample_fps, (h_bar, w_bar)


def element(fps):
    """The reference's video element for a file (qwen2vl_model.py:135-144)."""
    ele = {"type": "video", "video": "x.mp4", "max_pixels": 360 * 420}
    if fps != "dynamic":
        ele["fps"] = 8.0 if fps is None else fps
    return ele


@pytest.mark.parametrize("fps", [8.0, 2.0, "dynamic", None, 30.0])
@pytest.mark.parametrize("total,video_fps,h,w", [(504, 24.0, 360, 640), (24, 12.0, 96, 128), (300, 29.97, 1080, 1920),
                                                 (7, 25.0, 240, 320), (95, 30.0, 480, 360), (5000, 24.0, 720, 1280)])
def test_planner_reproduces_qwen_vl_utils(fps, total, video_fps, h, w):
    want = vl_utils_fetch_plan(element(fps), total, video_fps, h, w)
    got = qu.qwen_video_file_plan(total, video_fps, h, w, fps=None if fps == "dynamic" else (8.0 if fps is None else fps),
                                  max_pixels=qm.VIDEO_FILE_MAX_PIXELS)
    assert got[0] == want[0] and got[1] == want[1] and tuple(got[2]) == tuple(want[2])


def test_planner_on_the_readme_clip_shape():
    """A 21 s, 24 fps, 640x360 clip: 168 frames at fps 8 and 42 at qwen_vl_utils' 2.0, resized to 280x504 under 360*420 pixels."""
    idx, sfps, size = qu.qwen_video_file_plan(504, 24.0, 360, 640, fps=8.0, max_pixels=qm.VIDEO_FILE_MAX_PIXELS)
    assert len(idx) == 168 and idx[0] == 0 and idx[-1] == 503 and sfps == pytest.approx(8.0) and size == (280, 504)
    idx, sfps, size = qu.qwen_video_file_plan(504, 24.0, 360, 640, fps=None, max_pixels=qm.VIDEO_FILE_MAX_PIXELS)
    assert len(idx) == 42 and sfps == pytest.approx(2.0) and size == (280, 504)


def test_planner_short_clips_and_caps():
    with pytest.raises(ValueError, match="nframes"):
        qu.qwen_video_file_plan(1, 24.0, 64, 64, fps=8.0)
    with pytest.raises(ValueError, match="nframes"):
        qu.qwen_video_file_plan(0, 24.0, 64, 64, fps=8.0)
    assert qu.qwen_video_file_plan(2, 24.0, 64, 64, fps=8.0)[0] == [0, 1]
    assert qu.qwen_video_file_plan(3, 30.0, 64, 64, fps=8.0)[0] == [0, 2]       # 4 minimum frames, floored to the even 2 <= 3
    idx = qu.qwen_video_file_plan(100000, 24.0, 360, 640, fps=8.0)[0]           # the 768-frame cap
    assert len(idx) == 768 and idx[-1] == 99999
    # VIDEO_TOTAL_PIXELS: total_pixels / nframes * 2 caps the budget, down to int(min_pixels * 1.05)
    for total_pixels in (168 * 120000 // 2, 1000):
        want = vl_utils_fetch_plan({"fps": 8.0}, 504, 24.0, 720, 1280, total_pixels=total_pixels)
        got = qu.qwen_video_file_plan(504, 24.0, 720, 1280, fps=8.0, total_pixels=total_pixels)
        assert tuple(got[2]) == tuple(want[2])
        assert got[2][0] * got[2][1] <= max(total_pixels / 168 * 2, int(qu.VIDEO_MIN_PIXELS * 1.05))
    env = dict(os.environ, VIDEO_MAX_PIXELS="1234567.0")
    out = subprocess.run([sys.executable, "-c", "from t2v_metrics_b200.models.vqascore_models import qwen_utils as q; print(q.VIDEO_TOTAL_PIXELS)"],
                         cwd=ROOT, env=env, capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "1234567"


# ------------------------------------------------------------------------------------------------ OpenCV reader
def write_clip(path, frames, fps):
    import cv2
    codec = {".mp4": "mp4v", ".avi": "MJPG", ".mkv": "MJPG"}[os.path.splitext(path)[1]]
    w = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*codec), fps, (frames.shape[2], frames.shape[1]))
    for f in frames:
        w.write(np.ascontiguousarray(f[..., ::-1]))
    w.release()


def smooth_frames(n, h, w, seed=0):
    """Smooth, distinct frames (lossy codecs keep them close): moving colour gradients."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = [np.stack([128 + 100 * np.sin(x / 9 + f / 2 + seed), 128 + 100 * np.cos(y / 7 - f / 3), 128 + 90 * np.sin((x + y) / 13 + f)], -1)
           for f in range(n)]
    return np.clip(np.stack(out), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("ext", [".mp4", ".avi", ".mkv"])
def test_opencv_reader_returns_the_frames_written(tmp_path, ext):
    pytest.importorskip("cv2")
    frames = smooth_frames(10, 64, 96)
    path = tmp_path / ("clip" + ext)
    write_clip(path, frames, 12.0)
    total, fps, get = qu.OpenCVVideoReader().open(str(path))
    assert total == 10 and fps == pytest.approx(12.0)
    first = get([0])
    got = np.concatenate([first, get([0, 3, 4]), get([7, 9])])          # continues where it stopped; a repeated index is re-served
    assert got.dtype == np.uint8 and got.shape == (6, 64, 96, 3)
    want = frames[[0, 0, 3, 4, 7, 9]].astype(np.float64)
    err = np.abs(got.astype(np.float64) - want).mean(axis=(1, 2, 3))
    assert err.max() < 6, err                                              # lossy codecs, RGB order (a BGR swap is ~80 levels off)
    for k, i in enumerate([0, 0, 3, 4, 7, 9]):                             # each frame is nearest to the one written at its index
        d = np.abs(frames.astype(np.float64) - got[k].astype(np.float64)).mean(axis=(1, 2, 3))
        assert int(d.argmin()) == i
    assert np.array_equal(get([2]), qu.OpenCVVideoReader().open(str(path))[2]([2]))   # a backwards index reopens the stream


def test_opencv_reader_refuses_unreadable_files(tmp_path):
    pytest.importorskip("cv2")
    bad = tmp_path / "bad.mp4"
    bad.write_bytes(b"not a video")
    with pytest.raises(ValueError):
        qu.OpenCVVideoReader().open(str(bad))


# ------------------------------------------------------------------------------------------------ restatement and processor
@pytest.mark.parametrize("n,h,w,size", [(4, 360, 640, (280, 504)), (3, 240, 320, (280, 364)), (2, 97, 61, (392, 252)),
                                        (4, 480, 640, (336, 448))])
def test_file_restatement_matches_the_installed_processor(n, h, w, size):
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms import functional as TF
    from transformers import Qwen2VLVideoProcessor
    frames = np.random.default_rng(n * 7 + h).integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    resized, rows, grid = qu.qwen_video_file_to_patches(frames, size)
    # fetch_video's tensor (resize(BICUBIC, antialias=True).float()) handed to the processor with do_resize=False
    video = TF.resize(torch.from_numpy(frames).permute(0, 3, 1, 2), list(size), interpolation=InterpolationMode.BICUBIC, antialias=True)
    assert torch.equal(resized.permute(0, 3, 1, 2), video)
    ref = Qwen2VLVideoProcessor()(videos=[video.float()], do_resize=False, return_tensors="pt", fps=8.0)
    assert list(grid) == ref["video_grid_thw"][0].tolist() == [math.ceil(n / 2), size[0] // 14, size[1] // 14]
    assert rows.shape == ref["pixel_values_videos"].shape
    assert float((rows - ref["pixel_values_videos"]).abs().max()) <= 1e-6


def test_second_per_grid_ts_of_a_file_is_the_processors():
    """fetch_video hands the processor a float [T, 3, H, W] tensor without metadata and the sample fps as `fps=`; the processor's
    sampled_fps is then 24 (video_utils.py:108-112), so a file's second_per_grid_ts is 2/24 like a frame stack's."""
    from transformers import Qwen2VLVideoProcessor
    video = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (4, 3, 56, 84))).float()
    for kw in ({}, {"fps": 8.0}, {"fps": 2.0}, {"fps": 0.5}):
        meta = Qwen2VLVideoProcessor()(videos=[video], do_resize=False, return_tensors="pt", return_metadata=True, **kw)["video_metadata"][0]
        assert 2 / meta.sampled_fps == SPG_VIDEO == qo.Qwen25VLConfig.tiny(**TINY).temporal_patch_size / qm.HF_FRAME_LIST_FPS


# ------------------------------------------------------------------------------------------------ the committed file golden
def load_file_golden(golden_dir):
    """tests/golden/qwen_video_file_tiny.pt (tools/make_golden_qwen_video_file.py); the weights are regenerated from the seed and pinned
    by their checksum."""
    import hashlib
    blob = torch.load(os.path.join(golden_dir, "qwen_video_file_tiny.pt"), weights_only=False)
    cfg = qo.Qwen25VLConfig(**blob["config"])
    sd = qo.make_synthetic_state_dict(cfg, seed=blob["weights_seed"])
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().view(torch.uint8).numpy().tobytes())
    assert h.hexdigest() == blob["weights_sha256"], "synthetic weights differ from the ones the golden was generated with"
    return blob, cfg, sd


def golden_patches(clip_path, run):
    """The golden clip decoded by the OpenCV reader at the run's indices, through the host restatement."""
    total, fps, get = qu.OpenCVVideoReader().open(clip_path)
    return qu.qwen_video_file_to_patches(get(run["indices"]), tuple(run["size"]))[1]


@pytest.mark.parametrize("key,fps", [("8.0", 8.0), ("dynamic", None)])
def test_planner_reader_and_oracle_reproduce_the_committed_file_golden(golden_dir, tmp_path, key, fps):
    pytest.importorskip("cv2")
    blob, cfg, sd = load_file_golden(golden_dir)
    r = blob["runs"][key]
    clip = tmp_path / ("clip" + blob["clip_ext"])
    clip.write_bytes(blob["clip"])
    total, vfps, get = qu.OpenCVVideoReader().open(str(clip))
    h, w = get([0]).shape[1:3]
    idx, _, size = qu.qwen_video_file_plan(total, vfps, h, w, fps=fps, max_pixels=qm.VIDEO_FILE_MAX_PIXELS)
    assert idx == r["indices"] and list(size) == r["size"] and r["second_per_grid_ts"] == SPG_VIDEO
    patches = golden_patches(str(clip), r)
    t, gh, gw = r["grid_thw"]
    assert patches.shape[0] == t * gh * gw
    o = qo.qwen25vl_score(sd, cfg, patches, [tuple(r["grid_thw"])], [torch.tensor(r["score_prompt"])], [r["answer_ids"][0]], mode="fp32",
                          return_all=True, second_per_grid_ts=[SPG_VIDEO])
    assert float((o["logits"][0] - r["logits"]).abs().max()) < 2e-4
    assert abs(float(o["scores"][0]) - r["probs"]) < 1e-6


# ------------------------------------------------------------------------------------------------ plugin wiring with a stand-in engine
class _Reader:
    """Stand-in decoder: frame i of a clip is filled with level i; clip sizes and lengths by name. Records every get()."""
    CLIPS = {"a": (48, 24.0, 360, 640), "b": (10, 10.0, 96, 128)}

    def __init__(self):
        self.opened, self.gets = [], []

    def open(self, path):
        name = os.path.basename(path)[:-4]
        total, fps, h, w = self.CLIPS[name]
        self.opened.append(name)

        def get(indices):
            self.gets.append((name, list(indices)))
            return np.stack([np.full((h, w, 3), i, np.uint8) for i in indices])
        return total, fps, get


def _file_plugin(monkeypatch, engine, reader):
    """The real plugin with a stand-in engine, tokenizer and reader; the two device pre-processing entry points replaced by stand-ins
    whose rows name the item (files: 100 + clip index, stills / stacks: the number in the file name)."""
    p = qm.Qwen2VLModel.__new__(qm.Qwen2VLModel)
    p.engine, p.tokenizer, p.cfg, p.repetition_penalty = engine, CharTokenizer(), qo.Qwen25VLConfig.tiny(**TINY), 1.1
    p.model_name, p._checkpoint, p.video_reader = "qwen2.5-vl-7b", "/nonexistent/model.safetensors", reader
    p.min_pixels, p.max_pixels = qm.QWEN_VL_UTILS_MIN_PIXELS, qm.QWEN_VL_UTILS_MAX_PIXELS
    engine.device = torch.device("cpu")
    seen = []

    def file_pre(slices, size, device, n_frames, **kw):
        got = [s for s in slices]
        frames = torch.cat(got)
        seen.append(dict(n=n_frames, size=tuple(size), frames=frames[:, 0, 0, 0].tolist(), slices=len(got)))
        t, gh, gw = (n_frames + 1) // 2, size[0] // 14, size[1] // 14
        return torch.full((t * gh * gw, 4), 100.0 + len(seen)), (t, gh, gw)

    def still_pre(items, device, *a, **kw):
        grids = [((it.shape[0] + 1) // 2 if it.dim() == 4 else 1, 4, 4) for it in items]
        return torch.cat([torch.full((math.prod(g), 4), float(i)) for i, g in enumerate(grids)]), grids

    monkeypatch.setattr(eng_mod, "qwen_preprocess_video_file_u8", file_pre)
    monkeypatch.setattr(eng_mod, "qwen_preprocess_u8", still_pre)
    monkeypatch.setattr(eng_mod, "qwen_preprocess_video_u8", still_pre)
    return p, seen


def _paths(tmp_path):
    rng = np.random.default_rng(0)
    img, stack = tmp_path / "img.png", tmp_path / "stack.npy"
    Image.fromarray(rng.integers(0, 256, (56, 56, 3), dtype=np.uint8)).save(img)
    np.save(stack, rng.integers(0, 256, (3, 56, 56, 3), dtype=np.uint8))
    return str(tmp_path / "a.mp4"), str(tmp_path / "b.mkv"), str(img), str(stack)


@pytest.mark.parametrize("fps", [None, 8.0, "dynamic", 2.0])
def test_files_mix_with_stills_and_stacks_in_one_engine_call(monkeypatch, tmp_path, fps):
    a, b, img, stack = _paths(tmp_path)
    reader, engine = _Reader(), _Engine()
    p, seen = _file_plugin(monkeypatch, engine, reader)
    images = [a, img, a, stack, b]
    out = p.forward(images, ["t0", "t1", "t2", "t3", "t4"], fps=fps)
    (c,) = engine.calls
    assert reader.opened == ["a", "b"]                                      # each distinct file decoded once
    plans = []
    for name in ("a", "b"):
        total, vfps, h, w = _Reader.CLIPS[name]
        plans.append(qu.qwen_video_file_plan(total, vfps, h, w, fps=None if fps == "dynamic" else (8.0 if fps is None else fps),
                                             max_pixels=qm.VIDEO_FILE_MAX_PIXELS))
    assert [s["frames"] for s in seen] == [pl[0] for pl in plans] and [s["size"] for s in seen] == [tuple(pl[2]) for pl in plans]
    file_grids = [((len(pl[0]) + 1) // 2, pl[2][0] // 14, pl[2][1] // 14) for pl in plans]
    assert c["grids"] == [file_grids[0], (1, 4, 4), (2, 4, 4), file_grids[1]]
    assert c["kw"]["image_of_sample"] == [0, 1, 0, 2, 3]
    assert c["kw"]["second_per_grid_ts"] == [SPG_VIDEO, 1.0, SPG_VIDEO, SPG_VIDEO]
    # rows in item order: file a, still, stack, file b
    rows = [0]
    for g in c["grids"]:
        rows.append(rows[-1] + math.prod(g))
    assert [float(c["pixels"][r, 0]) for r in rows[:-1]] == [101.0, 0.0, 1.0, 102.0]
    for b_, item in enumerate(c["kw"]["image_of_sample"]):
        tok = p.cfg.image_token_id if item == 1 else p.cfg.video_token_id
        run = [t for t in c["prompts"][b_] if t in (p.cfg.video_token_id, p.cfg.image_token_id)]
        assert run == [tok] * (math.prod(c["grids"][item]) // 4)
    assert out.tolist() == torch.tensor([(len(q) % 97) / 100 for q in c["prompts"]]).tolist()


def test_fps_changes_a_files_frames_and_not_a_stacks(monkeypatch, tmp_path):
    a, _, _, stack = _paths(tmp_path)
    grids = {}
    for fps in (8.0, "dynamic"):
        engine = _Engine()
        p, _ = _file_plugin(monkeypatch, engine, _Reader())
        p.forward([a, stack], ["x", "y"], fps=fps)
        grids[fps] = engine.calls[0]["grids"]
    assert grids[8.0][0] == (8, 20, 36) and grids["dynamic"][0] == (2, 20, 36)   # 16 and 4 of 48 frames at 24 fps
    assert grids[8.0][1] == grids["dynamic"][1]


def test_large_clips_go_to_the_device_in_slices(monkeypatch, tmp_path):
    a = _paths(tmp_path)[0]
    engine = _Engine()
    p, seen = _file_plugin(monkeypatch, engine, _Reader())
    monkeypatch.setattr(eng_mod, "VIDEO_SLICE_BYTES", 3 * 360 * 640 * 3)        # three 640x360 frames per slice
    p.forward([a], ["x"])
    (s,) = seen
    assert s["n"] == 16 and s["slices"] == 6 and s["frames"] == qu.qwen_video_file_plan(48, 24.0, 360, 640, 8.0)[0]


@pytest.mark.parametrize("op", ["forward", "trace", "generate", "rollout"])
def test_calls_with_files_split_under_the_workspace_budget(monkeypatch, tmp_path, op):
    a, b, img, stack = _paths(tmp_path)
    engine = _Engine(per_pair=1000)
    p, _ = _file_plugin(monkeypatch, engine, _Reader())
    p.VIDEO_WORKSPACE_BUDGET = p.ROLLOUT_WORKSPACE_BUDGET = 2500              # 5 pairs -> 3 -> 2 per call
    images, texts = [a, img, b, stack, a], ["p", "q", "r", "s", "t"]
    if op == "generate":
        p.generate(images, texts, max_new_tokens=3)
    elif op == "trace":
        p.forward_with_trace(images, texts)
    elif op == "rollout":
        p.forward(images, texts, max_new_tokens=2)
    else:
        p.forward(images, texts)
    assert [len(c["prompts"]) for c in engine.calls] == [2, 2, 1]
    assert [c["kw"]["second_per_grid_ts"] for c in engine.calls] == [[SPG_VIDEO, 1.0], [SPG_VIDEO, SPG_VIDEO], [SPG_VIDEO]]


def test_without_a_reader_files_are_refused_before_any_launch(monkeypatch, tmp_path):
    a, _, img, _ = _paths(tmp_path)

    engine = _Engine()
    p, seen = _file_plugin(monkeypatch, engine, None)
    for call in (lambda: p.forward([img, a], ["x", "y"]), lambda: p.forward_with_trace([a], ["x"]),
                 lambda: p.generate([a], ["x"]), lambda: p.forward([a], ["x"], max_new_tokens=3)):
        with pytest.raises(NotImplementedError, match="4-D .npy"):
            call()
    assert seen == [] and engine.calls == []


# ------------------------------------------------------------------------------------------------ Score
class _ScoreModel:
    def __init__(self, video_mode, reader):
        self.video_mode, self.video_reader, self.calls = video_mode, reader, []

    def forward(self, images, texts, **kw):
        self.calls.append((list(images), list(texts), kw))
        return torch.tensor([float(os.path.basename(i)[1]) + float(t[1:]) / 10 for i, t in zip(images, texts)])


def _score(model):
    from t2v_metrics_b200.score import Score

    class S(Score):
        def prepare_scoremodel(self, name, device, cache_dir, **kw):
            return model

        def list_all_models(self):
            return ["fake"]
    return S("fake", device="cpu")


def test_score_forward_passes_files_only_to_a_plugin_that_decodes_them():
    files, texts = ["v1.mp4", "v2.avi"], ["t1", "t2", "t3"]
    sc = _score(_ScoreModel("direct", object()))
    got = sc(images=files, texts=texts, fps=4.0)
    assert torch.allclose(got, torch.tensor([[1.1, 1.2, 1.3], [2.1, 2.2, 2.3]]))
    assert sc.model.calls == [(["v1.mp4"] * 3 + ["v2.avi"] * 3, texts * 2, {"fps": 4.0})]
    got = sc.batch_forward([{"videos": ["v1.mp4", "v2.mkv"], "texts": ["t1"]}, {"videos": ["v2.mp4", "v1.mov"], "texts": ["t3"]}],
                           batch_size=2)
    assert torch.allclose(got, torch.tensor([[[1.1], [2.1]], [[2.3], [1.3]]]))
    for model in (_ScoreModel("direct", None), _ScoreModel("concat", object())):
        sc = _score(model)
        with pytest.raises(NotImplementedError):
            sc(images=files, texts=texts)
        with pytest.raises(NotImplementedError):
            sc.batch_forward([{"videos": ["v1.mp4"], "texts": ["t1"]}])
        assert model.calls == []


@pytest.mark.parametrize("in_size,out_size", [(120, 308), (360, 280), (1080, 280), (640, 504), (61, 252), (96, 392), (280, 280)])
def test_resize_taps_are_torchs_weights_in_monotonic_windows(in_size, out_size):
    """engine._aa_bicubic_taps: scattered back, the windows give torch's whole weight matrix bit for bit; window starts never decrease
    and stay inside the axis (the device kernel refuses anything else). 120 -> 308 has windows whose first tap weighs exactly 0."""
    first, w, taps = eng_mod._aa_bicubic_taps(in_size, out_size)
    assert (first[1:] >= first[:-1]).all() and int(first.min()) >= 0 and int(first.max()) + taps <= in_size
    eye = torch.eye(in_size)[None, :, None, :]
    want = torch.nn.functional.interpolate(eye, size=(1, out_size), mode="bicubic", antialias=True, align_corners=False)[0, :, 0, :].t()
    got = torch.zeros_like(want).scatter_(1, first[:, None].long() + torch.arange(taps), w)
    assert torch.equal(got, want)

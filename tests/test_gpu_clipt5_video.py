"""CLIP-FlanT5 video scoring by frame concatenation on the GPU: the column-tiled device resize of wide canvases is bit-exact against the
CPU PIL path, one launch per upload slice, and Score.forward on the fixture videos equals Score.forward on the reference's canvases
(tests/golden/clipt5_video) and sits within the golden tolerance of the oracle's scores of those canvases."""
import dataclasses
import io
import os
import tempfile
import types

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import clipt5_oracle as orc
from preprocess_ref import canvas, pil_reference
from t2v_metrics_b200.models.vqascore_models.mm_utils import clip_preprocess

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clipt5_video")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda", 0)


def test_two_pass_restatement_equals_the_pil_path():
    for w, h in ((5190, 360), (300, 4000)):
        a = canvas(w, h, 3)
        assert torch.equal(pil_reference(a), clip_preprocess(Image.fromarray(a), 336))


WIDE = [(5190, 360), (10310, 720), (15430, 1080), (65500, 64), (64, 65500)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_wide_canvases_bit_exact_vs_pil(dev, dtype):
    from t2v_metrics_b200.engine import clip_preprocess_u8
    rng = np.random.default_rng(7)
    sizes = WIDE + [(int(rng.integers(9000, 30000)), int(rng.integers(200, 1200))) for _ in range(2)] + \
        [(int(rng.integers(100, 900)), int(rng.integers(9000, 20000)))] + [(512, 512)]
    arrs = [canvas(w, h, i) for i, (w, h) in enumerate(sizes)]
    got = clip_preprocess_u8([torch.from_numpy(a) for a in arrs], 336, dev, out_dtype=dtype)       # one launch, a 512^2 still among them
    torch.cuda.synchronize()
    for i, a in enumerate(arrs):
        ref = (clip_preprocess(Image.fromarray(a), 336) if max(a.shape) <= 16000 else pil_reference(a)).to(dtype)
        assert torch.equal(got[i].cpu(), ref), f"{sizes[i]} {dtype}: max diff {float((got[i].cpu().float() - ref.float()).abs().max())}"


def test_one_launch_per_upload_slice(dev, monkeypatch):
    from t2v_metrics_b200 import engine
    arrs = [torch.from_numpy(canvas(10310, 720, i)) for i in range(3)] + [torch.from_numpy(canvas(512, 512, 9))]
    whole = engine.clip_preprocess_u8_sliced(arrs, 336, dev)
    monkeypatch.setattr(engine, "CLIP_SLICE_BYTES", 10310 * 720 * 3 * 2)        # slices of 2, then 1 + the still
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        sliced = engine.clip_preprocess_u8_sliced(arrs, 336, dev)
        torch.cuda.synchronize()
    launches = [e for e in prof.events() if "image_preprocess_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    assert len(launches) == 2
    assert torch.equal(sliced, whole)


def _scorer(golden_dir):
    import t2v_metrics_b200 as t2v
    from t2v_metrics_b200.config import ClipT5Config
    blob = torch.load(os.path.join(golden_dir, "clipt5_tiny.pt"), weights_only=False)
    cfg = orc.ClipT5Config.tiny(**blob["config"])
    sd = orc.golden_state_dict(blob, cfg)
    ref_gap = float((blob["hf_bf16"]["scores"] - blob["hf_fp32"]["scores"]).abs().max())

    class Tok:                      # the stand-in tokenizer tools/make_golden_clipt5_video.py scored the canvases with
        pad_token_id = 0

        def __call__(self, chunk):
            return types.SimpleNamespace(input_ids=[3 + (sum(map(ord, w)) % 400) for w in chunk.split()] + [1])
    return t2v.VQAScore(model="clip-flant5-xl", device="cuda", cache_dir=tempfile.mkdtemp(), tokenizer=Tok(), state_dict=sd,
                        config=ClipT5Config(**dataclasses.asdict(cfg))), ref_gap


def test_score_forward_on_videos_equals_the_reference_canvases(dev, golden_dir, tmp_path):
    gold = torch.load(os.path.join(GOLD, "canvases.pt"), weights_only=False)
    texts = gold["texts"]
    scorer, ref_gap = _scorer(golden_dir)
    tol = 1e-3 + 2.0 * ref_gap
    for nf in sorted({c["num_frames"] for c in gold["cases"]}):
        cases = [c for c in gold["cases"] if c["num_frames"] == nf]
        videos = [os.path.join(GOLD, c["video"]) for c in cases]
        pngs = []
        for i, c in enumerate(cases):
            p = str(tmp_path / f"canvas_{nf}_{i}.png")
            open(p, "wb").write(c["canvas_png"])
            pngs.append(p)
        got = scorer(images=videos, texts=texts, num_frames=nf).cpu()
        want = scorer(images=pngs, texts=texts).cpu()
        assert torch.equal(got, want), (nf, got, want)
        oracle = torch.stack([c["oracle_bf16"] for c in cases])
        err = float((got - oracle).abs().max())
        print(f"\n[num_frames {nf}] scores {got.tolist()} | vs oracle bf16 {err:.2e} (tol {tol:.2e})")
        assert err <= tol


def test_several_texts_build_one_canvas_per_video(dev, golden_dir, monkeypatch):
    from t2v_metrics_b200.models.vqascore_models import clip_t5_model
    scorer, _ = _scorer(golden_dir)
    built = []
    real = clip_t5_model.video_canvas
    monkeypatch.setattr(clip_t5_model, "video_canvas", lambda p, n: built.append(p) or real(p, n))
    videos = [os.path.join(GOLD, "clip40.avi"), os.path.join(GOLD, "clip40.mp4")]
    out = scorer(images=videos, texts=["a", "b c", "d e f"], num_frames=4)
    assert out.shape == (2, 3) and sorted(built) == sorted(videos)


def test_batch_forward_over_videos_equals_per_pair_calls(dev, golden_dir):
    scorer, _ = _scorer(golden_dir)
    v = [os.path.join(GOLD, n) for n in ("clip40.avi", "clip40.mp4", "clip5.avi")]
    data = [{"videos": [v[0], v[1]], "texts": ["a dog", "red square"]}, {"videos": [v[2], v[0]], "texts": ["cats", "moving"]}]
    got = scorer.batch_forward(data, batch_size=2).cpu()
    for s, item in enumerate(data):
        for i, vid in enumerate(item["videos"]):
            for j, t in enumerate(item["texts"]):
                one = scorer.model.forward([vid], [t], num_frames=4)
                assert float((got[s, i, j] - one[0]).abs()) <= 2e-4, (s, i, j)

"""CLIP-FlanT5 video scoring by frame concatenation, host side: the canvas of every fixture equals the one the reference's own functions
make (tests/golden/clipt5_video, from tools/make_golden_clipt5_video.py), the error cases, the Score wiring with a stand-in plugin, and
the column-tiled plan of the device resize for wide canvases."""
import ctypes as C
import io
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

from t2v_metrics_b200.models.vqascore_models import mm_utils

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clipt5_video")


def golden_cases():
    return torch.load(os.path.join(GOLD, "canvases.pt"), weights_only=False)["cases"]


def canvas_of(case):
    return np.asarray(Image.open(io.BytesIO(case["canvas_png"])))


@pytest.mark.parametrize("video", ["clip40.avi", "clip40.mp4", "clip5.avi"])
def test_host_canvas_equals_the_reference(video):
    cases = [c for c in golden_cases() if c["video"] == video]
    assert sorted(c["num_frames"] for c in cases) == [1, 4, 8, 12, 50]
    for c in cases:
        got = mm_utils.video_canvas(os.path.join(GOLD, video), c["num_frames"])
        want = canvas_of(c)
        assert got.dtype == np.uint8 and got.shape == tuple(c["canvas_shape"])
        assert np.array_equal(got, want), (video, c["num_frames"])


def test_canvas_layout():
    """Width = frame widths + 10 px per gap, height = the tallest frame, black below the shorter one and in the gaps."""
    frames = [np.full((16, 24, 3), 200, np.uint8), np.full((32, 16, 3), 100, np.uint8)]
    got = mm_utils.concat_frames_rgb(frames)
    assert got.shape == (32, 24 + 10 + 16, 3)
    assert int(got[24:, :16].max()) <= 16 and int(got[:, 27:31].max()) <= 16 and int(got[4:28, 40:46].min()) >= 80


def _write_video(path, n, w, h, fourcc="MJPG"):
    import cv2
    wr = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*fourcc), 10, (w, h))
    assert wr.isOpened()
    for i in range(n):
        wr.write(np.full((h, w, 3), (i * 20) % 256, np.uint8))
    wr.release()
    return str(path)


def test_error_cases(tmp_path):
    bad = tmp_path / "broken.mp4"
    bad.write_bytes(b"not a video")
    with pytest.raises(ValueError, match="no frame"):
        mm_utils.video_canvas(str(bad), 4)
    with pytest.raises(ValueError, match="num_frames"):
        mm_utils.video_canvas(os.path.join(GOLD, "clip40.avi"), 0)
    wide = _write_video(tmp_path / "wide.avi", 40, 2000, 16)
    with pytest.raises(ValueError, match="80390x16"):          # 40 x 2000 + 39 x 10
        mm_utils.video_canvas(wide, 40)


# ------------------------------------------------------------------------------------------------ Score wiring
class _Plugin:
    """Stand-in CLIPT5Model: records its calls, scores pair i of a call as 1 + i / 10."""
    video_mode = "concat"
    builds_video_canvases = True

    def __init__(self):
        self.calls = []

    def forward(self, images, texts, **kw):
        self.calls.append((list(images), list(texts), kw))
        return torch.tensor([1.0 + i / 10 for i in range(len(images))])


def _score(model):
    from t2v_metrics_b200.score import Score

    class S(Score):
        def prepare_scoremodel(self, *a, **k):
            return model

        def list_all_models(self):
            return ["fake"]
    return S("fake", device="cpu")


def test_score_passes_videos_and_num_frames_to_a_canvas_building_plugin():
    sc = _score(_Plugin())
    got = sc(images=["a.mp4", "b.MKV"], texts=["t1", "t2"], num_frames=6)
    assert got.shape == (2, 2)
    assert sc.model.calls == [(["a.mp4", "a.mp4", "b.MKV", "b.MKV"], ["t1", "t2", "t1", "t2"], {"num_frames": 6})]
    sc.model.calls.clear()
    sc(images=["a.mp4"], texts=["t1"])
    assert sc.model.calls[0][2] == {"num_frames": 8}


def test_image_only_calls_carry_no_num_frames():
    sc = _score(_Plugin())
    sc(images=["a.png", "b.jpg"], texts=["t"], num_frames=3)
    sc.batch_forward([{"images": ["a.png"], "texts": ["t"]}])
    assert [c[2] for c in sc.model.calls] == [{}, {}]


def test_mixed_call_sends_videos_and_images_in_one_plugin_call():
    sc = _score(_Plugin())
    sc(images=["a.png", "v.avi"], texts=["t"])
    assert sc.model.calls == [(["a.png", "v.avi"], ["t", "t"], {"num_frames": 8})]


def test_batch_forward_over_videos_passes_num_frames_4():
    sc = _score(_Plugin())
    got = sc.batch_forward([{"videos": ["v1.mp4", "v2.avi"], "texts": ["t1"]}, {"videos": ["v3.mp4", "v4.mov"], "texts": ["t2"]}],
                           batch_size=2)
    assert got.shape == (2, 2, 1)
    assert [c[2] for c in sc.model.calls] == [{"num_frames": 4}, {"num_frames": 4}]
    assert [c[0] for c in sc.model.calls] == [["v1.mp4", "v3.mp4"], ["v2.avi", "v4.mov"]]


def test_a_concat_plugin_without_canvases_still_refuses_videos():
    p = _Plugin()
    p.builds_video_canvases = False
    sc = _score(p)
    with pytest.raises(NotImplementedError):
        sc(images=["v.mp4"], texts=["t"])
    assert p.calls == []


def test_clipt5_plugin_declares_canvases_and_refuses_videos_in_generate():
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import CLIPT5Model
    assert CLIPT5Model.video_mode == "concat" and CLIPT5Model.builds_video_canvases
    m = CLIPT5Model.__new__(CLIPT5Model)
    with pytest.raises(NotImplementedError):
        m.generate(["v.mp4"], ["t"])


def test_plugin_forward_refuses_num_frames_0_before_device_work():
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import CLIPT5Model
    m = CLIPT5Model.__new__(CLIPT5Model)
    with pytest.raises(ValueError, match="num_frames"):
        m.forward([os.path.join(GOLD, "clip40.avi")], ["t"], num_frames=0)


# ------------------------------------------------------------------------------------------------ the device resize's plan
def _ws_bytes(w, h, pad=1, size=336):
    from t2v_metrics_b200 import _lib
    return _lib.load().vqa_clip_preprocess_workspace_bytes((C.c_int32 * 1)(h), (C.c_int32 * 1)(w), 1, size, pad)


@pytest.mark.parametrize("w,h", [(65500, 720), (720, 65500), (65500, 65500), (10310, 720), (15430, 1080), (65500, 64), (64, 65500),
                                 (9000, 720)])
def test_wide_canvases_are_accepted_with_pad(w, h):
    assert _ws_bytes(w, h) > 0


@pytest.mark.parametrize("w,h", [(65501, 720), (720, 65501), (65501, 65501)])
def test_canvases_over_65500_are_refused(w, h):
    from t2v_metrics_b200 import _lib
    assert _ws_bytes(w, h) == 0
    assert "too large" in _lib.last_error(None)


@pytest.mark.parametrize("in_size,first,count", [(10310, 0, 336), (15430, 100, 68), (65500, 315, 21), (5190, 0, 336)])
def test_column_tile_tables_equal_pillow(in_size, first, count):
    """The horizontal table of one column tile of a wide padded canvas (outputs [first, first + count) of in_size -> 336), replayed on
    the host, resizes a random row exactly as Pillow does."""
    from t2v_metrics_b200 import _lib
    lib = _lib.load()
    ks = lib.vqa_resample_table(in_size, 336, first, count, None, None)
    b = (C.c_int32 * (2 * count))()
    k = (C.c_int32 * (count * ks))()
    assert lib.vqa_resample_table(in_size, 336, first, count, b, k) == ks
    bounds = np.frombuffer(b, np.int32).reshape(count, 2)
    kk = np.frombuffer(k, np.int32).reshape(count, ks).astype(np.int64)
    row = np.random.default_rng(in_size).integers(0, 256, (1, in_size), dtype=np.uint8)
    got = np.empty(count, np.int64)
    for i, (x0, n) in enumerate(bounds):
        acc = int((row[0, x0:x0 + n].astype(np.int64) * kk[i, :n]).sum()) + (1 << 21)
        got[i] = min(max(acc >> 22, 0), 255)
    want = np.asarray(Image.fromarray(row, "L").resize((336, 1), Image.BICUBIC))[0, first:first + count]
    assert np.array_equal(got, want)

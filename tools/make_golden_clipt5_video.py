"""Generate tests/golden/clipt5_video/ : small video fixtures and the canvases the reference makes of them for CLIP-FlanT5.

  T2V_METRICS_REF=<checkout of linzhiqiu/t2v_metrics> python tools/make_golden_clipt5_video.py

The fixtures are synthesized here (written once, then kept): a 96x64 MJPG .avi and a 96x64 mp4v .mp4 of 40 frames, and a 5-frame
MJPG .avi shorter than most frame counts asked for. For each fixture and num_frames in NUM_FRAMES the canvas is made by the reference's
own functions, executed from the checkout: extract_frames into a temporary directory, cv2.imread of the frame files in name order
(temporal order; the reference's os.listdir order is not defined), concatenate_images_horizontal(dist_images=10), cv2.imwrite of the
canvas and PIL's Image.open(...).convert("RGB") of that file, as the reference's score.py:78-98 and CLIPT5Model.load_images do. The
canvases are stored as PNG bytes (lossless). The CPU oracle's scores of those canvases (oracle/clipt5_oracle.py at the width of tests/golden/clipt5_tiny.pt, mode "bf16" and "fp32")
are stored beside them for TEXTS with the question and answer templates of the plugin and the stand-in tokenizer of the tests.
"""
import io
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv2
import numpy as np
import torch
from PIL import Image

from oracle import clipt5_oracle as orc

OUT = os.path.join(ROOT, "tests", "golden", "clipt5_video")
FIXTURES = {"clip40.avi": ("MJPG", 40), "clip40.mp4": ("mp4v", 40), "clip5.avi": ("MJPG", 5)}
NUM_FRAMES = (1, 4, 8, 12, 50)
TEXTS = ["a red square moving right", "two cats on a sofa"]


class Tok:
    """Stand-in with the T5 tokenizer's contract (ids + trailing </s> = 1), as tests/test_gpu_clipt5.py's plugin test uses."""
    pad_token_id = 0

    def __call__(self, chunk):
        return types.SimpleNamespace(input_ids=[3 + (sum(map(ord, w)) % 400) for w in chunk.split()] + [1])


def synth(path, fourcc, n, w=96, h=64, fps=10):
    """A gradient background, a square that moves right and a frame-number stripe: every frame differs from its neighbours."""
    wr = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*fourcc), fps, (w, h))
    assert wr.isOpened(), fourcc
    y, x = np.mgrid[0:h, 0:w]
    for i in range(n):
        f = np.stack([(x * 255 // (w - 1)), (y * 255 // (h - 1)), np.full_like(x, (i * 37) % 256)], -1).astype(np.uint8)
        s = 4 + (i * 2) % (w - 24)
        f[20:40, s:s + 16] = (0, 0, 255)
        f[h - 6:, : (i * w) // n + 1] = 255
        wr.write(f)
    wr.release()


def load_reference(ref_root):
    ref_mm = os.path.join(ref_root, "t2v_metrics", "models", "vqascore_models", "mm_utils.py")
    src = open(ref_mm).read().replace("from ...constants import", "from _ref_constants import")
    consts = types.ModuleType("_ref_constants")
    exec(open(os.path.join(ref_root, "t2v_metrics", "constants.py")).read(), consts.__dict__)
    sys.modules["_ref_constants"] = consts
    mod = types.ModuleType("_ref_mm_utils")
    exec(compile(src, ref_mm, "exec"), mod.__dict__)
    return mod


def reference_canvas(mod, video, num_frames):
    with tempfile.TemporaryDirectory() as tmp:
        frames_dir = os.path.join(tmp, f"temp_{os.path.basename(video)}")
        mod.extract_frames(video, num_frames, frames_dir)
        frames = [cv2.imread(os.path.join(frames_dir, f)) for f in sorted(os.listdir(frames_dir)) if f.endswith(".jpg")]
        canvas = mod.concatenate_images_horizontal(frames, dist_images=10)
        path = os.path.join(tmp, f"concat_{os.path.basename(video)}.jpg")
        cv2.imwrite(path, canvas)
        return np.asarray(Image.open(path).convert("RGB"), dtype=np.uint8).copy()


def oracle_inputs(cfg, n_images):
    """input_ids / lens / labels of every (canvas, text) pair, built as CLIPT5Model._tokenize builds them."""
    from t2v_metrics_b200.constants import CONTEXT_LEN, IGNORE_INDEX
    from t2v_metrics_b200.models.vqascore_models.clip_t5_model import (default_answer_template, default_question_template,
                                                                        format_question, prompt_token_ids)
    from t2v_metrics_b200.models.vqascore_models.mm_utils import t5_tokenizer_image_token
    texts = TEXTS * n_images
    ids = prompt_token_ids(Tok(), [format_question(default_question_template.format(t)) for t in texts], CONTEXT_LEN, cfg.vocab, {})
    labs = [t5_tokenizer_image_token(default_answer_template.format(t), Tok()) for t in texts]
    L, T = max(map(len, ids)), max(map(len, labs))
    input_ids = torch.zeros(len(ids), L, dtype=torch.long)
    labels = torch.full((len(ids), T), IGNORE_INDEX, dtype=torch.long)
    for i, (a, b) in enumerate(zip(ids, labs)):
        input_ids[i, :len(a)] = torch.tensor(a)
        labels[i, :len(b)] = torch.tensor(b)
    lens = torch.tensor([len(a) for a in ids])
    image_index = torch.arange(n_images).repeat_interleave(len(TEXTS))
    return input_ids, lens, labels, image_index


def main():
    ref_root = os.environ.get("T2V_METRICS_REF", "")
    if not ref_root:
        sys.exit("set T2V_METRICS_REF to a checkout of the reference")
    os.makedirs(OUT, exist_ok=True)
    for name, (fourcc, n) in FIXTURES.items():
        if not os.path.exists(os.path.join(OUT, name)):
            synth(os.path.join(OUT, name), fourcc, n)
    mod = load_reference(ref_root)
    blob_tiny = torch.load(os.path.join(ROOT, "tests", "golden", "clipt5_tiny.pt"), weights_only=False)
    cfg = orc.ClipT5Config.tiny(**blob_tiny["config"])
    sd = orc.golden_state_dict(blob_tiny, cfg)
    cases, canvases = [], []
    for name in FIXTURES:
        for nf in NUM_FRAMES:
            canvas = reference_canvas(mod, os.path.join(OUT, name), nf)
            png = io.BytesIO()
            Image.fromarray(canvas).save(png, format="PNG", optimize=True)
            assert np.array_equal(np.asarray(Image.open(io.BytesIO(png.getvalue()))), canvas)
            cases.append(dict(video=name, num_frames=nf, canvas_png=png.getvalue(), canvas_shape=canvas.shape))
            print(name, nf, canvas.shape, len(png.getvalue()), "PNG bytes")
            canvases.append(canvas)
    pixels = torch.stack([orc.clip_preprocess(Image.fromarray(c), cfg.image_size) for c in canvases])
    input_ids, lens, labels, image_index = oracle_inputs(cfg, len(cases))
    scores = {mode: orc.clipt5_score(sd, cfg, pixels, input_ids, lens, labels, image_index, mode=mode).view(len(cases), len(TEXTS))
              for mode in ("bf16", "fp32")}
    for i, c in enumerate(cases):
        c["oracle_bf16"], c["oracle_fp32"] = scores["bf16"][i], scores["fp32"][i]
    torch.save(dict(cases=cases, texts=TEXTS, weights="clipt5_tiny.pt", opencv_version=cv2.__version__,
                    pillow_version=Image.__version__), os.path.join(OUT, "canvases.pt"))
    print("oracle bf16", scores["bf16"].tolist())


if __name__ == "__main__":
    main()

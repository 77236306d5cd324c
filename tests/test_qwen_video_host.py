"""Qwen2.5-VL video inputs (4-D .npy frame stacks), CPU side: the restated fetch_video + video processor against the installed
Qwen2VLVideoProcessor, the processor's second_per_grid_ts and the rope positions it gives, the oracle against the committed HF video
golden, and the plugin's wiring onto the engine (token runs, per-grid second_per_grid_ts, order, duplicates, budget splits, refusals)
with a stand-in engine."""
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import qwen25vl_oracle as qo
from t2v_metrics_b200 import qwen_host
from t2v_metrics_b200.models.vqascore_models import qwen2vl_model as qm
from t2v_metrics_b200.models.vqascore_models.qwen_utils import (build_prompt_ids, default_question_template, qwen_video_to_patches,
                                                                smart_resize)
from test_qwen_host import TINY, hf_model

SPG_VIDEO = 2 / 24


class CharTokenizer:
    """Stand-in tokenizer: characters -> code points (mod 500); ids >= 630 are special (eos 639, pad 638)."""
    eos_token_id, pad_token_id, bos_token_id = 639, 638, None

    def encode(self, s, add_special_tokens=False):
        return [ord(ch) % 500 for ch in s]

    def decode(self, ids, skip_special_tokens=False, clean_up_tokenization_spaces=True):
        return " ".join(str(int(i)) for i in ids if not (skip_special_tokens and int(i) >= 630))


def processor_patches(frames, **kw):
    """The installed processor on the frames as the reference hands them over: PIL frames resized like still images (fetch_image), the
    count padded to an even number with the last frame (fetch_video), then do_resize=False."""
    from transformers import Qwen2VLVideoProcessor
    ims = []
    for f in frames:
        im = Image.fromarray(f, "RGB")
        rh, rw = smart_resize(im.height, im.width, 28, qm.QWEN_VL_UTILS_MIN_PIXELS, qm.QWEN_VL_UTILS_MAX_PIXELS)
        ims.append(im.resize((rw, rh), resample=Image.BICUBIC))
    ims += [ims[-1]] * (len(ims) % 2)
    return Qwen2VLVideoProcessor()(videos=[ims], do_resize=False, return_tensors="pt", return_metadata=True, **kw)


@pytest.mark.parametrize("n,h,w", [(4, 56, 84), (5, 112, 168), (3, 84, 56), (1, 56, 56), (2, 50, 90), (3, 61, 97)])
def test_video_restatement_matches_the_installed_processor(n, h, w):
    frames = np.random.default_rng(n * 1000 + h).integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    got, grid = qwen_video_to_patches(frames, min_pixels=qm.QWEN_VL_UTILS_MIN_PIXELS, max_pixels=qm.QWEN_VL_UTILS_MAX_PIXELS)
    ref = processor_patches(frames)
    assert list(grid) == ref["video_grid_thw"][0].tolist() and grid[0] == math.ceil(n / 2)
    assert got.shape == ref["pixel_values_videos"].shape
    assert float((got - ref["pixel_values_videos"]).abs().max()) <= 1e-6


def test_second_per_grid_ts_is_the_processors_and_gives_its_rope_positions():
    """A frame list has no fps, so the processor's sampled_fps is 24 whatever fps is passed (video_utils.py:108-111) and
    second_per_grid_ts = 2/24 (processing_qwen2_5_vl.py:103-113); with it every video token has temporal position 0 in the installed
    get_rope_index, and qwen_host reproduces those positions."""
    frames = np.random.default_rng(0).integers(0, 256, (4, 56, 84, 3), dtype=np.uint8)
    for kw in ({}, {"fps": 2.0}, {"fps": 8.0}):
        assert processor_patches(frames, **kw)["video_metadata"][0].sampled_fps == qm.HF_FRAME_LIST_FPS
    cfg = qo.Qwen25VLConfig.tiny(**TINY)
    assert cfg.temporal_patch_size / qm.HF_FRAME_LIST_FPS == SPG_VIDEO
    m = hf_model(cfg)
    grid = [(2, 4, 6)]
    ids = torch.tensor(build_prompt_ids(CharTokenizer(), "Q", 2 * 4 * 6 // 4, cfg.video_token_id))
    hf_pos, _ = m.model.get_rope_index(ids[None], torch.where(ids == cfg.video_token_id, 2, 0)[None], video_grid_thw=torch.tensor(grid),
                                       second_per_grid_ts=torch.tensor([SPG_VIDEO]), attention_mask=torch.ones(1, len(ids), dtype=torch.long))
    mine = qwen_host.mrope_position_ids(ids.tolist(), grid, cfg.image_token_id, cfg.spatial_merge_size, cfg.tokens_per_second,
                                        cfg.video_token_id, [SPG_VIDEO])
    assert torch.equal(mine, hf_pos[:, 0])
    assert int(mine[0][ids == cfg.video_token_id].max()) == 0


def load_video_golden(golden_dir):
    """tests/golden/qwen_video_tiny.pt (tools/make_golden_qwen_video.py); the weights are regenerated from the seed and pinned by their
    checksum. The processor's patches are stored as uint8 levels + its fp32 value per (channel, level) and rebuilt here as `patches`."""
    import hashlib
    blob = torch.load(os.path.join(golden_dir, "qwen_video_tiny.pt"), weights_only=False)
    cfg = qo.Qwen25VLConfig(**blob["config"])
    sd = qo.make_synthetic_state_dict(cfg, seed=blob["weights_seed"])
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().view(torch.uint8).numpy().tobytes())
    assert h.hexdigest() == blob["weights_sha256"], "synthetic weights differ from the ones the golden was generated with"
    for s in blob["stacks"]:
        lv = s["patch_levels"].long()
        s["patches"] = s["patch_table"][torch.arange(lv.shape[1]) // (lv.shape[1] // 3), lv]
    return blob, cfg, sd


@pytest.mark.parametrize("i", [0, 1, 2])
def test_oracle_and_restatement_reproduce_the_committed_video_golden(golden_dir, i):
    blob, cfg, sd = load_video_golden(golden_dir)
    s = blob["stacks"][i]
    got, grid = qwen_video_to_patches(s["frames"].numpy(), min_pixels=qm.QWEN_VL_UTILS_MIN_PIXELS, max_pixels=qm.QWEN_VL_UTILS_MAX_PIXELS)
    assert list(grid) == s["grid_thw"] and float((got - s["patches"]).abs().max()) <= 1e-6
    assert s["second_per_grid_ts"] == SPG_VIDEO
    t, gh, gw = grid
    assert s["score_prompt"] == build_prompt_ids(CharTokenizer(), default_question_template.format(blob["texts"][i]), t * gh * gw // 4,
                                                 cfg.video_token_id)
    ids = [torch.tensor(s["score_prompt"])]
    o = qo.qwen25vl_score(sd, cfg, s["patches"], [tuple(grid)], ids, [s["answer_ids"][0]], mode="fp32", return_all=True,
                          second_per_grid_ts=[SPG_VIDEO])
    assert float((o["logits"][0] - s["logits"]).abs().max()) < 5e-5
    assert abs(float(o["scores"][0]) - s["probs"]) < 1e-6


# ------------------------------------------------------------------------------------------------ plugin wiring with a stand-in engine
class _Engine:
    """Records every call. score_prompts: probability = (prompt length mod 97) / 100; workspace bytes = pairs x `per_pair`."""

    def __init__(self, per_pair=0):
        self.calls, self.per_pair = [], per_pair

    def score_workspace_bytes(self, batch, seq_len, n_patches):
        return batch * self.per_pair

    def generate_workspace_bytes(self, batch, seq_len, n_patches, max_new_tokens):
        return batch * self.per_pair

    def score_prompts(self, pixel_patches, grid_thw, prompts, answer_ids, **kw):
        self.calls.append(dict(op="score", pixels=pixel_patches, grids=list(grid_thw), prompts=prompts, answers=answer_ids, kw=kw))
        return torch.tensor([(len(p) % 97) / 100 for p in prompts])

    def topk_last(self, k, temperature=1.0, repetition_penalty=1.0):
        B = len(self.calls[-1]["prompts"])
        return torch.tensor([[len(p) % 500 + j for j in range(k)] for p in self.calls[-1]["prompts"]]), torch.full((B, k), 0.5)

    def generate_prompts(self, pixel_patches, grid_thw, prompts, max_new_tokens, eos_ids, **kw):
        self.calls.append(dict(op="generate", pixels=pixel_patches, grids=list(grid_thw), prompts=prompts, kw=kw))
        return [[len(p) % 500] for p in prompts]

    def rollout_scores(self, pixel_patches, grid_thw, prompts, answer_ids, max_new_tokens, eos_ids, **kw):
        self.calls.append(dict(op="rollout", pixels=pixel_patches, grids=list(grid_thw), prompts=prompts, kw=kw))
        B, n = len(prompts), max(len(a) for a in answer_ids)
        return dict(tokens=[[5] * max_new_tokens for _ in prompts], logp=torch.full((B, max_new_tokens, n), -0.5))


def _files(tmp_path):
    """vid0.npy: 5 frames of 56x84 (grid 3x4x6), img1.png: 56x56 (1x4x4), img2.npy: 3-D 84x56 (1x6x4), vid3.npy: 1 frame (1x4x4)."""
    rng = np.random.default_rng(0)
    paths = dict(vid0=tmp_path / "vid0.npy", img1=tmp_path / "img1.png", img2=tmp_path / "img2.npy", vid3=tmp_path / "vid3.npy")
    np.save(paths["vid0"], rng.integers(0, 256, (5, 56, 84, 3), dtype=np.uint8))
    Image.fromarray(rng.integers(0, 256, (56, 56, 3), dtype=np.uint8)).save(paths["img1"])
    np.save(paths["img2"], rng.integers(0, 256, (84, 56, 3), dtype=np.uint8))
    np.save(paths["vid3"], rng.integers(0, 256, (1, 56, 56, 3), dtype=np.uint8))
    return {k: str(v) for k, v in paths.items()}


GRIDS = dict(vid0=(3, 4, 6), img1=(1, 4, 4), img2=(1, 6, 4), vid3=(1, 4, 4))


def _plugin(engine):
    p = qm.Qwen2VLModel.__new__(qm.Qwen2VLModel)
    p.engine, p.tokenizer, p.cfg, p.repetition_penalty = engine, CharTokenizer(), qo.Qwen25VLConfig.tiny(**TINY), 1.1
    p.model_name, p._checkpoint = "qwen2.5-vl-7b", "/nonexistent/model.safetensors"
    name = lambda x: os.path.basename(x)[:-4]
    # item rows hold the item's number, so the rows an engine call receives name the items
    p.load_images = lambda paths: (torch.cat([torch.full((math.prod(GRIDS[name(x)]), 4), float(name(x)[3:])) for x in paths]),
                                   [GRIDS[name(x)] for x in paths])
    return p


def _check_call(c, images, sel, cfg):
    """One engine call: each item it uses once, the right token run per prompt and the per-grid second_per_grid_ts."""
    names = [os.path.basename(images[i])[:-4] for i in sel]
    items = sorted(set(names), key=names.index)
    assert len(c["grids"]) == len(items)
    rows = [0]
    for g in c["grids"]:
        rows.append(rows[-1] + math.prod(g))
    spg = c["kw"].get("second_per_grid_ts")
    for b, nm in enumerate(names):
        g = c["kw"]["image_of_sample"][b]
        assert c["grids"][g] == GRIDS[nm] and float(c["pixels"][rows[g], 0]) == float(nm[3:])
        video = nm.startswith("vid")
        tok = cfg.video_token_id if video else cfg.image_token_id
        run = [t for t in c["prompts"][b] if t in (cfg.video_token_id, cfg.image_token_id)]
        assert run == [tok] * (math.prod(GRIDS[nm]) // 4)
        assert spg[g] == (SPG_VIDEO if video else 1.0)


def test_mixed_call_is_one_engine_call_in_order_with_duplicates_encoded_once(tmp_path):
    f = _files(tmp_path)
    eng = _Engine()
    p = _plugin(eng)
    images = [f["vid0"], f["img1"], f["vid0"], f["img2"], f["vid3"]]
    texts = ["a cat", "dogs", "a hat on a mat", "x", "a long text about a red car"]
    out = p.forward(images, texts)
    (c,) = eng.calls
    _check_call(c, images, range(5), p.cfg)
    assert c["kw"]["image_of_sample"] == [0, 1, 0, 2, 3]
    assert out.tolist() == torch.tensor([(len(q) % 97) / 100 for q in c["prompts"]]).tolist()
    assert c["answers"] == [ord("Y") % 500] * 5
    # a 1-frame video has the grid of a still image but video tokens and 2/24
    assert c["grids"][3] == GRIDS["img1"] and c["kw"]["second_per_grid_ts"][3] == SPG_VIDEO
    # fps does not change a .npy stack's scores
    assert torch.equal(p.forward(images, texts, fps=8.0), out)


@pytest.mark.parametrize("op", ["forward", "trace", "generate"])
def test_calls_with_a_video_split_under_the_workspace_budget(tmp_path, op):
    f = _files(tmp_path)
    eng = _Engine(per_pair=1000)
    p = _plugin(eng)
    p.VIDEO_WORKSPACE_BUDGET = 2500                    # 5 pairs -> 3 -> 2 per call
    images = [f["vid0"], f["img1"], f["vid0"], f["img2"], f["vid3"]]
    texts = ["a cat", "dogs", "a hat on a mat", "x", "a long text about a red car"]
    if op == "generate":
        out = p.generate(images, texts, max_new_tokens=3)
    elif op == "trace":
        out, traces = p.forward_with_trace(images, texts)
    else:
        out = p.forward(images, texts)
    assert [len(c["prompts"]) for c in eng.calls] == [2, 2, 1]
    for c, sel in zip(eng.calls, ([0, 1], [2, 3], [4])):
        _check_call(c, images, sel, p.cfg)
    prompts = [q for c in eng.calls for q in c["prompts"]]
    if op == "generate":
        assert out == [str(len(q) % 500) for q in prompts]
    else:
        assert out.tolist() == torch.tensor([(len(q) % 97) / 100 for q in prompts]).tolist()
    if op == "trace":
        assert [t["token_details"][0]["top_alternatives"][0]["token_id"] for t in traces] == [len(q) % 500 for q in prompts]


def test_rollout_scoring_of_a_video_passes_its_second_per_grid_ts(tmp_path):
    f = _files(tmp_path)
    eng = _Engine()
    p = _plugin(eng)
    images = [f["img1"], f["vid0"]]
    p.forward(images, ["a", "b"], max_new_tokens=3)
    (c,) = eng.calls
    assert c["op"] == "rollout" and c["kw"]["second_per_grid_ts"] == [1.0, SPG_VIDEO]
    assert [t for t in c["prompts"][1] if t == p.cfg.video_token_id] == [p.cfg.video_token_id] * 18


def test_image_only_calls_make_the_engine_call_they_always_made(tmp_path):
    f = _files(tmp_path)
    eng = _Engine(per_pair=1 << 40)                   # over any budget: image-only calls are never split
    p = _plugin(eng)
    images, texts = [f["img1"], f["img2"], f["img1"]], ["a", "bb", "ccc"]
    p.forward(images, texts, temperature=0.5)
    p.generate(images, texts, max_new_tokens=2)
    patches, grids = p.load_images([f["img1"], f["img2"]])
    q = [build_prompt_ids(p.tokenizer, default_question_template.format(t), math.prod(grids[g]) // 4, p.cfg.image_token_id)
         for t, g in zip(texts, (0, 1, 0))]
    s, g = eng.calls
    assert torch.equal(s["pixels"], patches) and s["grids"] == grids and s["prompts"] == q and s["answers"] == [89] * 3
    assert s["kw"] == dict(image_of_sample=[0, 1, 0], temperature=0.5, repetition_penalty=1.1)
    assert g["prompts"] == [build_prompt_ids(p.tokenizer, t, math.prod(grids[i]) // 4, p.cfg.image_token_id) for t, i in zip(texts, (0, 1, 0))]
    assert g["grids"] == grids and g["kw"] == dict(image_of_sample=[0, 1, 0], repetition_penalty=1.1)


def test_video_files_are_refused_and_other_array_ranks_raise(tmp_path):
    p = qm.Qwen2VLModel.__new__(qm.Qwen2VLModel)
    for ext in (".mp4", ".avi", ".MOV", ".mkv"):
        with pytest.raises(NotImplementedError, match="4-D .npy"):
            p.load_images([str(tmp_path / ("clip" + ext))])
    for shape in [(4, 4), (2, 2, 4, 4, 3)]:
        path = str(tmp_path / f"a{len(shape)}.npy")
        np.save(path, np.zeros(shape, dtype=np.uint8))
        with pytest.raises(ValueError, match="Unexpected shape"):
            p.load_images([path])

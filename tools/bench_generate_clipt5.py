"""Greedy generation with CLIP-FlanT5 on one H100: clip-flant5-xxl width with synthetic weights drawn on the device, 512x512 images
(CLIP pre-processing to 336x336) and 32 text ids per prompt, B in {1, 8, 32, 64}, 64 new tokens with no EOS ids so every run decodes the
same number of steps. One JSON line per batch size: prefill ms, median / p10 / p90 of the decode step (CUDA events around each graph
replay), generated tokens/s, launches per step, algorithmic bytes per step and the whole-step rate they give against the 3.35 TB/s
HBM3 data-sheet figure, per-category device time of one profiled step, and the GPU name and power limit read in the same run.

Bytes per step: every decoder weight read once (self-attention qkv / o, cross-attention q, Wk^T, Wv, o, gated FFN wi / wo, norms), the
lm_head, the encoder output the absorbed cross-attention reads twice per layer (scores against x, context against x^T), and the K/V rows
the step's self-attention reads (mean over the steps).

The baseline is HF T5ForConditionalGeneration.generate(inputs_embeds=<spliced prompt>, do_sample=False) in bf16 under autocast with its
K/V cache, one sample at a time, min_new_tokens = max_new_tokens, on the same GPU and weights (measured once, on --hf-samples).

  python tools/bench_generate_clipt5.py [--batches 1,8,32,64] [--new 64] [--no-hf] [--out results.jsonl]
"""
import argparse
import copy
import dataclasses
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from oracle import clipt5_oracle as orc
from bench_generate import HBM_PEAK, gpu_identity


def decoder_weight_bytes(cfg):
    D, inner, dff = cfg.d_model, cfg.n_heads * cfg.d_kv, cfg.d_ff
    per_layer = 3 * inner * D + D * inner + inner * D + 2 * inner * D + D * inner + 2 * dff * D + D * dff + 3 * D
    return 2.0 * (cfg.dec_layers * per_layer + D)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,64")
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--text", type=int, default=32)
    ap.add_argument("--image", type=int, default=512)
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--hf-samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_generate_clipt5.py measures on a CUDA device; there is none")
    from t2v_metrics_b200.config import ClipT5Config
    from t2v_metrics_b200.engine import ClipT5Engine, clip_preprocess_u8
    dev = torch.device("cuda:0")
    gpu, power = gpu_identity()
    cfg = orc.ClipT5Config.xxl()
    N = a.new
    sd = orc.make_synthetic_state_dict(cfg, seed=0, device=dev, gen_device=dev)
    eng = ClipT5Engine(ClipT5Config(**dataclasses.asdict(cfg)), dev)
    eng.load_state_dict(sd)
    W = decoder_weight_bytes(cfg)
    LM = 2.0 * cfg.vocab * cfg.d_model
    g = torch.Generator().manual_seed(2)
    lines = []

    def batch_inputs(B):
        inp = orc.make_synthetic_inputs(cfg, B, a.text, seed=1)
        raw = torch.randint(0, 256, (B, a.image, a.image, 3), dtype=torch.uint8, generator=g)
        pixels = clip_preprocess_u8(raw, cfg.image_size, dev)
        i32 = lambda t: t.to(dev, torch.int32).contiguous()
        return inp, pixels, i32(inp["input_ids"]), i32(inp["text_lens"])

    for B in [int(x) for x in a.batches.split(",")]:
        inp, pixels, ids, lens = batch_inputs(B)
        eng.generate_tensors(pixels, ids, lens, N, ())          # warm-up: loads modules, captures the step graph
        st = eng.generate_begin(pixels, ids, lens, N, ())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        pre = []
        for _ in range(3):
            e0.record()
            st["prefill"]()
            e1.record()
            torch.cuda.synchronize()
            pre.append(e0.elapsed_time(e1))
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(N - 1)]
        t0 = time.perf_counter()
        for s, e in evs:
            s.record()
            st["graph"].replay()
            e.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        steps = torch.tensor([s.elapsed_time(e) for s, e in evs])
        assert bool((st["lengths"].cpu() == N).all())
        st["prefill"]()
        eng.generate_step(st)
        launches = eng.last_launch_count()
        eng.set_profile(True)
        eng.generate_step(st)
        torch.cuda.synchronize()
        prof = eng.read_profile()
        eng.set_profile(False)
        S = inp["input_ids"].shape[1] - 1 + cfg.num_patches
        enc = 2.0 * cfg.dec_layers * B * S * cfg.d_model * 2                  # x and x^T read once each per layer
        kv = 2.0 * cfg.dec_layers * B * cfg.n_heads * cfg.d_kv * 2 * (1 + N) / 2     # K and V rows a step attends to, mean over the steps
        total = W + LM + enc + kv
        med = float(steps.median())
        line = dict(workload="clip-flant5-xxl greedy generate", gpu=gpu, power_limit=power, batch=B, image=a.image, text_tokens=a.text,
                    encoder_tokens=S, new_tokens=N, prefill_ms=round(min(pre), 3), step_ms_median=round(med, 4),
                    step_ms_p10=round(float(steps.quantile(0.1)), 4), step_ms_p90=round(float(steps.quantile(0.9)), 4),
                    decode_tokens_per_s=round(B * (N - 1) / wall, 1), launches_per_step=launches, step_bytes=total,
                    step_decoder_weight_bytes=W, step_lm_head_bytes=LM, step_encoder_output_bytes=enc, step_kv_bytes=kv,
                    whole_step_GBps=round(total / (med * 1e-3) / 1e9, 1), whole_step_share_of_hbm_peak=round(total / (med * 1e-3) / HBM_PEAK, 3),
                    step_device_ms_by_category={k: round(v[0], 4) for k, v in prof.items()},
                    step_scopes_by_category={k: v[2] for k, v in prof.items()})
        print(json.dumps(line), flush=True)
        lines.append(line)
        del st
    del eng
    torch.cuda.empty_cache()
    if not a.no_hf:
        import hf_reference as hf
        vision, proj, t5 = hf.build_hf_modules(cfg, sd, dtype=torch.bfloat16, device=dev, assign=True)
        t5.config.use_cache = True
        gcfg = copy.deepcopy(t5.generation_config)
        gcfg.eos_token_id, gcfg.max_length, gcfg.do_sample, gcfg.num_beams, gcfg.use_cache = None, None, False, 1, True
        inp, pixels, _, _ = batch_inputs(a.hf_samples)

        def run(b, n):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                feats = vision(pixels[b:b + 1].to(torch.bfloat16), output_hidden_states=True).hidden_states[-2][:, 1:]
                img = proj(feats.to(torch.bfloat16))
                ids = inp["input_ids"][b, :int(inp["text_lens"][b])].to(dev)
                s = int((ids == orc.IMAGE_TOKEN_INDEX).nonzero()[0])
                emb = torch.cat([t5.shared(ids[:s]).to(img.dtype), img[0], t5.shared(ids[s + 1:]).to(img.dtype)])[None]
                return t5.generate(inputs_embeds=emb, attention_mask=torch.ones(1, emb.shape[1], dtype=torch.long, device=dev),
                                   generation_config=gcfg, max_new_tokens=n, min_new_tokens=n)
        run(0, 4)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in range(a.hf_samples):
            run(b, N)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        line = dict(workload="HF T5 generate(do_sample=False) bf16 autocast, K/V cache, one sample at a time", gpu=gpu, power_limit=power,
                    samples=a.hf_samples, image=a.image, text_tokens=a.text, new_tokens=N, seconds=round(dt, 3),
                    tokens_per_s=round(a.hf_samples * N / dt, 1))
        print(json.dumps(line), flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

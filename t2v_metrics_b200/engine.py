"""Tensor-level entry to the H100 engine: PyTorch tensors in, PyTorch tensors out, everything in between is
libvqa_b200.so (hand-written sm_90a kernels) reached through ctypes. PyTorch only supplies device memory and the
current CUDA stream.

`ClipT5Engine.score_tensors` is what `bench.py` and the plugin (`models/clip_t5_model.py`) call; it replaces the
`self.model(input_ids, images=..., labels=...)` + CrossEntropy loop of the reference's v3.0 CLIPT5Model.forward.
"""
from __future__ import annotations

import collections
import functools
import ctypes as C
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .config import ClipT5Config

IMAGE_TOKEN_INDEX = -200  # t2v_metrics/constants.py:7
IGNORE_INDEX = -100       # t2v_metrics/constants.py:6
ATTN_KEY_TILE = 128       # key rows per tile of the head-dim-128 attention kernel (attention_sm90.cuh)


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream_ptr(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _dtype_code(dtype: torch.dtype) -> int:
    """The vqa_dtype of an fp32 or bf16 tensor."""
    return _lib.VQA_DTYPE_F32 if dtype == torch.float32 else _lib.VQA_DTYPE_BF16


def _check(rc: int, handle=None, what: str = ""):
    if rc != 0:
        raise RuntimeError(f"libvqa_b200 {what} failed (status {rc}): {_lib.last_error(handle)}")


def _call(name: str, *args):
    """Call `name` in libvqa_b200.so; a non-zero status raises RuntimeError naming it."""
    _check(getattr(_lib.load(), name)(*args), None, name)


def _size_query(name: str, ctype, head: tuple, tail: tuple) -> int:
    """Call `name` without scratch (NULL, 0 bytes between `head` and `tail`). It stops at its scratch check with VQA_ERR_WORKSPACE and
    reports through the pointer after the scratch arguments the size (or split count) it needs, which this returns. Any other status is
    an argument error and raises."""
    value = ctype(0)
    rc = getattr(_lib.load(), name)(*head, None, 0, C.byref(value), *tail)
    if rc != _lib.VQA_ERR_WORKSPACE:
        raise RuntimeError(f"libvqa_b200 {name} without scratch returned status {rc}, not VQA_ERR_WORKSPACE: {_lib.last_error(None)}")
    return int(value.value)


def fold_norm_gain(weight: torch.Tensor, gamma: torch.Tensor) -> torch.Tensor:
    """W . diag(gamma) in fp32, rounded to bf16 once: the weight the fused-norm GEMMs use (their epilogue supplies rsqrt(mean(x^2) + eps))."""
    return (weight.float() * gamma.float()[None, :]).to(torch.bfloat16).contiguous()


def convert_state_dict(sd: Dict[str, torch.Tensor], cfg: ClipT5Config, device, fuse_norms: bool = False) -> Dict[str, torch.Tensor]:
    """HF-named CLIP-FlanT5 weights (CLIPVisionModel under `vision_tower.`, `mm_projector.*`,
    T5ForConditionalGeneration names) -> the engine's fused bf16 layout:
      * q/k/v projections concatenated row-wise ([3*inner, d]) so one GEMM produces the packed QKV buffer;
      * wi_0 / wi_1 concatenated ([2*d_ff, d]) for the gated-GELU epilogue; cross-attention k/v concatenated;
      * the Conv2d patch embedding flattened to [D, 3*ps*ps] and zero-padded along K to a multiple of 64.
    Mirrors `model.to(device, dtype=torch.bfloat16)` (mm_utils.py:228)."""
    out: Dict[str, torch.Tensor] = {}

    def put(name, t):
        out[name] = t.detach().to(device=device, dtype=torch.bfloat16).contiguous()

    v = "vision_tower.vision_model."
    D = cfg.vit_hidden
    k_real = 3 * cfg.patch_size * cfg.patch_size
    kpad = (k_real + 63) // 64 * 64
    pw = sd[v + "embeddings.patch_embedding.weight"].reshape(D, k_real)
    pw_pad = torch.zeros(D, kpad, dtype=pw.dtype, device=pw.device)
    pw_pad[:, :k_real] = pw
    put("vit.patch_embed.weight", pw_pad)
    put("vit.class_embedding", sd[v + "embeddings.class_embedding"])
    put("vit.position_embedding", sd[v + "embeddings.position_embedding.weight"])
    put("vit.pre_ln.weight", sd[v + "pre_layrnorm.weight"])
    put("vit.pre_ln.bias", sd[v + "pre_layrnorm.bias"])
    for l in range(cfg.vit_layers - 1):
        p, q = v + f"encoder.layers.{l}.", f"vit.layers.{l}."
        put(q + "ln1.weight", sd[p + "layer_norm1.weight"]); put(q + "ln1.bias", sd[p + "layer_norm1.bias"])
        put(q + "ln2.weight", sd[p + "layer_norm2.weight"]); put(q + "ln2.bias", sd[p + "layer_norm2.bias"])
        put(q + "qkv.weight", torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], dim=0))
        put(q + "qkv.bias", torch.cat([sd[p + f"self_attn.{n}_proj.bias"] for n in "qkv"], dim=0))
        put(q + "out.weight", sd[p + "self_attn.out_proj.weight"]); put(q + "out.bias", sd[p + "self_attn.out_proj.bias"])
        put(q + "fc1.weight", sd[p + "mlp.fc1.weight"]); put(q + "fc1.bias", sd[p + "mlp.fc1.bias"])
        put(q + "fc2.weight", sd[p + "mlp.fc2.weight"]); put(q + "fc2.bias", sd[p + "mlp.fc2.bias"])
    for i in (0, 2):
        put(f"proj.{i}.weight", sd[f"mm_projector.{i}.weight"]); put(f"proj.{i}.bias", sd[f"mm_projector.{i}.bias"])
    put("t5.shared", sd["shared.weight"])
    put("t5.lm_head", sd["lm_head.weight"])  # untied from `shared` for FlanT5 (SURVEY F6)
    put("t5.enc.rel_bias", sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"])
    put("t5.dec.rel_bias", sd["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"])
    put("t5.enc.final_ln", sd["encoder.final_layer_norm.weight"])
    put("t5.dec.final_ln", sd["decoder.final_layer_norm.weight"])
    for l in range(cfg.enc_layers):
        p, q = f"encoder.block.{l}.layer.", f"t5.enc.{l}."
        a = p + "0.SelfAttention."
        put(q + "ln0", sd[p + "0.layer_norm.weight"])
        put(q + "qkv", torch.cat([sd[a + f"{n}.weight"] for n in "qkv"], dim=0))
        put(q + "o", sd[a + "o.weight"])
        put(q + "ln1", sd[p + "1.layer_norm.weight"])
        put(q + "wi", torch.cat([sd[p + "1.DenseReluDense.wi_0.weight"], sd[p + "1.DenseReluDense.wi_1.weight"]], dim=0))
        put(q + "wo", sd[p + "1.DenseReluDense.wo.weight"])
        if fuse_norms:
            out[q + "qkv_g"] = fold_norm_gain(out[q + "qkv"], out[q + "ln0"])
            out[q + "wi_g"] = fold_norm_gain(out[q + "wi"], out[q + "ln1"])
    for l in range(cfg.dec_layers):
        p, q = f"decoder.block.{l}.layer.", f"t5.dec.{l}."
        a, c = p + "0.SelfAttention.", p + "1.EncDecAttention."
        put(q + "ln0", sd[p + "0.layer_norm.weight"])
        put(q + "qkv", torch.cat([sd[a + f"{n}.weight"] for n in "qkv"], dim=0))
        put(q + "o", sd[a + "o.weight"])
        put(q + "ln1", sd[p + "1.layer_norm.weight"])
        put(q + "cq", sd[c + "q.weight"])
        put(q + "ckv", torch.cat([sd[c + "k.weight"], sd[c + "v.weight"]], dim=0))
        put(q + "ckT", sd[c + "k.weight"].t())   # Wk^T for the absorbed cross-attention
        put(q + "co", sd[c + "o.weight"])
        put(q + "ln2", sd[p + "2.layer_norm.weight"])
        put(q + "wi", torch.cat([sd[p + "2.DenseReluDense.wi_0.weight"], sd[p + "2.DenseReluDense.wi_1.weight"]], dim=0))
        put(q + "wo", sd[p + "2.DenseReluDense.wo.weight"])
    return out


class _Engine:
    """What both engines share: one library handle on one device, weight binding, profiling, the scoring workspace, and greedy
    generation (its own workspace, one state per call shape, the decode loop)."""

    MAX_GEN_GRAPHS = 8

    def __init__(self, cfg, device, create: str, config):
        """create: the vqa_create_* entry point that makes the handle from the config struct `config`."""
        if not torch.cuda.is_available():
            raise RuntimeError(f"{type(self).__name__} needs a CUDA device (sm_90a); there is no CPU path")
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device)
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self._h = C.c_void_p()
        with torch.cuda.device(idx):
            _check(getattr(self.lib, create)(C.byref(config), idx, C.byref(self._h)), None, create)
        self._weights: Dict[str, torch.Tensor] = {}
        self._workspace: Optional[torch.Tensor] = None
        self._graphs: Dict[tuple, tuple] = {}      # CUDA graphs of whole scoring forwards, keyed by the call's shapes
        self._gen_workspace: Optional[torch.Tensor] = None
        self._gen_states: "collections.OrderedDict[tuple, dict]" = collections.OrderedDict()   # per generation call shape, LRU order
        self._gen_flag = torch.zeros(1, dtype=torch.int32, pin_memory=True)                   # the decode loop's all-finished read-back

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            self.lib.vqa_destroy(h)
            self._h = C.c_void_p()

    def _run(self, name: str, *args):
        """Call the handle entry point `name` (the handle is its first argument) with the engine's device current -- the library launches
        on the current device, and a process may drive several GPUs -- and raise on a non-zero status."""
        with torch.cuda.device(self.device):
            rc = getattr(self.lib, name)(self._h, *args)
        _check(rc, self._h, name)

    def _grow(self, attr: str, need: int, dependents: dict) -> torch.Tensor:
        """The workspace self.<attr>, reallocated when it holds fewer than `need` bytes. The captured graphs or generation states in
        `dependents` point into the old one and are dropped with it."""
        if getattr(self, attr) is None or getattr(self, attr).numel() < need:
            dependents.clear()
            setattr(self, attr, None)        # free the old workspace before allocating the larger one
            setattr(self, attr, torch.empty(need, dtype=torch.uint8, device=self.device))
        return getattr(self, attr)

    # ---- weights
    def bind_engine_tensors(self, tensors: Dict[str, torch.Tensor]):
        arr = (_lib.VqaTensor * len(tensors))()
        keep = []
        for i, (name, t) in enumerate(tensors.items()):
            assert t.is_cuda and t.dtype == torch.bfloat16 and t.is_contiguous(), name
            nb = name.encode()
            keep.append(nb)
            arr[i].name = nb
            arr[i].data = t.data_ptr()
            for d in range(4):
                arr[i].shape[d] = t.shape[d] if d < t.dim() else 1
            arr[i].ndim = t.dim()
            arr[i].dtype = _lib.VQA_DTYPE_BF16
        self._run("vqa_bind_weights", arr, len(tensors))
        self._weights.update(tensors)  # keep the borrowed memory alive
        self._run("vqa_finalize_weights")

    # ---- launch count and profiling
    def last_launch_count(self) -> int:
        return int(self.lib.vqa_last_launch_count(self._h))

    def set_profile(self, enable: bool):
        self._run("vqa_set_profile", 1 if enable else 0)

    def read_profile(self):
        """After torch.cuda.synchronize(): {category: (device_ms, algorithmic_flops, scopes, algorithmic_bytes)} of the last call."""
        ms = (C.c_float * 4)()
        fl = (C.c_double * 4)()
        by = (C.c_double * 4)()
        sc = (C.c_int64 * 4)()
        self._run("vqa_profile_read", ms, fl, by, sc)
        names = ("gemm", "attention", "norm", "other")
        return {n: (float(ms[i]), float(fl[i]), int(sc[i]), float(by[i])) for i, n in enumerate(names)}

    # ---- greedy generation
    def _gen_state(self, key: tuple, need: int, make) -> dict:
        """The generation state of call shape `key`, made by make() on first use, with the generation workspace grown to `need` bytes.
        The MAX_GEN_GRAPHS most recently used states (each with its captured step graph) are kept."""
        self._grow("_gen_workspace", need, self._gen_states)
        st = self._gen_states.get(key)
        if st is None:
            st = self._gen_states[key] = make()
            while len(self._gen_states) > self.MAX_GEN_GRAPHS:
                self._gen_states.popitem(last=False)         # least recently used shape first
        self._gen_states.move_to_end(key)
        return st

    def _decode_loop(self, st: dict, use_graph: bool, check_every: int):
        """Decode steps (generate_step) after generate_begin until every prompt has finished: a CUDA graph of the step captured once per
        state, replayed. The host reads the all-finished flag through pinned memory every `check_every` steps. Returns (each prompt's
        generated ids, lengths [B] on the host)."""
        flag = self._gen_flag
        ev = torch.cuda.Event()

        def finished() -> bool:
            flag.copy_(st["all_done"], non_blocking=True)
            ev.record()
            ev.synchronize()
            return bool(flag[0])

        for step in range(1, st["max_new"]):
            if (step - 1) % check_every == 0 and finished():
                break
            if not use_graph:
                self.generate_step(st)
            elif st["graph"] is None:
                self.generate_step(st)             # the first step runs directly (module loading, kernel attributes), then is captured
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    self.generate_step(st)
                st["graph"] = graph
            else:
                st["graph"].replay()
        tokens, lengths = st["tokens"].cpu(), st["lengths"].cpu()
        return [tokens[b, :int(lengths[b])].tolist() for b in range(st["B"])], lengths


class ClipT5Engine(_Engine):
    """One engine = one model replica on one GPU (one process per GPU; SURVEY section 8e)."""

    def __init__(self, cfg: ClipT5Config, device="cuda:0", emulate_bf16_rounding: bool = True,
                 cross_attention_mode: str = "absorbed", round_attention_scores: bool = False, fuse_norms: bool = False):
        """round_attention_scores: form the bf16 score tensors of the reference's eager attention before the softmax (off: fp32 scores --
        closer to the exact result, and measured no closer to the bf16 reference, DESIGN.md section 4). fuse_norms: fold the encoder's
        T5LayerNorms into the GEMMs around them (no normalised copy of the residual stream; a different, equally valid rounding point)."""
        c = _lib.VqaClipT5Config(
            image_size=cfg.image_size, patch_size=cfg.patch_size, vit_hidden=cfg.vit_hidden, vit_heads=cfg.vit_heads,
            vit_mlp=cfg.vit_mlp, vit_layers_run=cfg.vit_layers - 1, vit_ln_eps=cfg.vit_ln_eps, d_model=cfg.d_model,
            n_heads=cfg.n_heads, d_ff=cfg.d_ff, enc_layers=cfg.enc_layers, dec_layers=cfg.dec_layers, vocab=cfg.vocab,
            rel_buckets=cfg.rel_buckets, rel_max_distance=cfg.rel_max_distance, t5_ln_eps=cfg.t5_ln_eps,
            image_token_id=IMAGE_TOKEN_INDEX, pad_token_id=cfg.pad_token_id, decoder_start_id=cfg.decoder_start_id,
            emulate_bf16_rounding=(1 if emulate_bf16_rounding else 0) | (2 if round_attention_scores else 0) | (4 if fuse_norms else 0),
            cross_attention_mode={"absorbed": 0, "reference": 1}[cross_attention_mode])
        self.fuse_norms = bool(fuse_norms)
        if cfg.d_kv != 64:
            raise ValueError("the engine's attention kernels are specialised for d_kv == 64")
        super().__init__(cfg, device, "vqa_create_clipt5", c)

    # ---- weights
    def bind_engine_tensors(self, tensors: Dict[str, torch.Tensor]):
        if self.fuse_norms and "t5.enc.0.qkv" in tensors and "t5.enc.0.qkv_g" not in tensors:
            tensors = dict(tensors)       # engine-layout weights without the folded copies (synthetic / shared dicts): derive them
            for l in range(self.cfg.enc_layers):
                q = f"t5.enc.{l}."
                tensors[q + "qkv_g"] = fold_norm_gain(tensors[q + "qkv"], tensors[q + "ln0"])
                tensors[q + "wi_g"] = fold_norm_gain(tensors[q + "wi"], tensors[q + "ln1"])
        super().bind_engine_tensors(tensors)

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        self.bind_engine_tensors(convert_state_dict(sd, self.cfg, self.device, fuse_norms=self.fuse_norms))

    # ---- forward
    @staticmethod
    def _check_inputs(pixel_values: torch.Tensor, image_index: Optional[torch.Tensor], input_ids: torch.Tensor, *int32_tensors):
        assert pixel_values.is_cuda and pixel_values.dim() == 4 and pixel_values.is_contiguous()
        assert pixel_values.dtype in (torch.float32, torch.bfloat16)
        for t in (input_ids, *int32_tensors):
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()
        if image_index is not None:
            assert image_index.is_cuda and image_index.dtype == torch.int32 and image_index.shape == (input_ids.shape[0],)

    def workspace_bytes(self, batch: int, n_images: int, text_len: int, label_len: int) -> int:
        return int(self.lib.vqa_clipt5_workspace_bytes(self._h, batch, n_images, text_len, label_len))

    def score_tensors(self, pixel_values: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor,
                      labels: torch.Tensor, image_index: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None, return_logprobs: bool = False):
        """pixel_values [NI,3,H,W] fp32/bf16 cuda; input_ids [B,L] int32 (-200 = image slot); text_lens [B] int32;
        labels [B,T] int32 (-100 = ignore); image_index [B] int32 or None. Returns scores [B] fp32 on the device
        (enqueued on the current stream; no synchronisation)."""
        dev = self.device
        self._check_inputs(pixel_values, image_index, input_ids, text_lens, labels)
        B, L = input_ids.shape
        T = labels.shape[1]
        NI = pixel_values.shape[0]
        ws = self._grow("_workspace", self.workspace_bytes(B, NI, L, T), self._graphs)
        if out is None:
            out = torch.empty(B, dtype=torch.float32, device=dev)
        logp = torch.zeros(B, T, dtype=torch.float32, device=dev) if return_logprobs else None   # ignored (-100) positions stay 0
        self._run("vqa_clipt5_score", _ptr(pixel_values), _dtype_code(pixel_values.dtype), NI, _ptr(image_index), _ptr(input_ids),
                  _ptr(text_lens), _ptr(labels), B, L, T, _ptr(out), _ptr(logp), _ptr(ws), ws.numel(), _stream_ptr(dev))
        return (out, logp) if return_logprobs else out

    MAX_GRAPHS = 16

    def score_tensors_graphed(self, pixel_values: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor, labels: torch.Tensor,
                              image_index: Optional[torch.Tensor] = None) -> torch.Tensor:
        """score_tensors replayed from a CUDA graph captured once per call shape (SURVEY 7 step 6): the forward is ~700 launches whose
        host-side cost (launch + argument marshalling) is the floor of small-batch calls such as the M x N API with a handful of pairs.
        Inputs are copied into the graph's static buffers; the returned scores tensor is the graph's output buffer (valid until the next
        replay of the same shape)."""
        key = (tuple(pixel_values.shape), pixel_values.dtype, tuple(input_ids.shape), int(labels.shape[1]), image_index is not None)
        entry = self._graphs.get(key)
        if entry is None:
            static = [t.clone() if t is not None else None for t in (pixel_values, input_ids, text_lens, labels, image_index)]
            self.score_tensors(static[0], static[1], static[2], static[3], image_index=static[4])      # sizes the workspace, sets kernel attributes
            torch.cuda.synchronize(self.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self.score_tensors(static[0], static[1], static[2], static[3], image_index=static[4])
            entry = self._graphs[key] = (graph, static, out)
            while len(self._graphs) > self.MAX_GRAPHS:          # oldest shape first (dict order = insertion order)
                self._graphs.pop(next(iter(self._graphs)))
        graph, static, out = entry
        for dst, src in zip(static, (pixel_values, input_ids, text_lens, labels, image_index)):
            if dst is not None:
                dst.copy_(src, non_blocking=True)
        graph.replay()
        return out

    def score_host(self, pixel_values: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor,
                   labels: torch.Tensor, image_index: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Host tensors in, host tensor out: H2D copies of this step's inputs (use pinned memory for async copies),
        one engine call, D2H of the scores. This is the end-to-end call bench.py's `e2e` times."""
        dev = self.device
        d = [t.to(dev, non_blocking=True) if t is not None else None
             for t in (pixel_values, input_ids, text_lens, labels, image_index)]
        scores = self.score_tensors(d[0], d[1], d[2], d[3], image_index=d[4])
        return scores.cpu()

    def score_images_u8(self, images_u8, input_ids: torch.Tensor, text_lens: torch.Tensor, labels: torch.Tensor,
                        image_index: Optional[torch.Tensor] = None, pad: bool = True) -> torch.Tensor:
        """End to end from DECODED images: uint8 HWC host (pinned) or device tensors -> device pre-processing kernel -> scores on
        the host. The reference does the resize + normalise per image on the CPU (a4 in SURVEY 8a) before its forward."""
        dev = self.device
        pixels = clip_preprocess_u8(images_u8, self.cfg.image_size, dev, pad=pad)
        d = [t.to(dev, non_blocking=True) if t is not None else None for t in (input_ids, text_lens, labels, image_index)]
        return self.score_tensors(pixels, d[0], d[1], d[2], image_index=d[3]).cpu()

    def debug_tensors(self, batch: int, n_images: int, text_len: int, label_len: int) -> Dict[str, torch.Tensor]:
        """Views into the workspace of the LAST call with these sizes (synchronise first): encoder / decoder outputs after their
        final norms, projector output, residual streams. Parity investigations only."""
        off = (C.c_size_t * 6)()
        self._run("vqa_clipt5_debug_layout", batch, n_images, text_len, label_len, off, 6)
        cfg = self.cfg
        S = text_len - 1 + cfg.num_patches
        ws = self._workspace

        def view(o, rows, cols):
            return ws[o:o + rows * cols * 2].view(torch.bfloat16).view(rows, cols)
        return dict(enc_out=view(off[0], batch * S, cfg.d_model).view(batch, S, cfg.d_model),
                    dec_out=view(off[1], batch * label_len, cfg.d_model).view(batch, label_len, cfg.d_model),
                    proj=view(off[2], n_images * (cfg.num_patches + 1), cfg.d_model).view(n_images, cfg.num_patches + 1, cfg.d_model),
                    vit_hidden=ws[off[5]:off[5] + n_images * (cfg.num_patches + 1) * cfg.vit_hidden * 4].view(torch.float32)
                    .view(n_images, cfg.num_patches + 1, cfg.vit_hidden))

    # ------------------------------------------------------------------------------------------ greedy generation
    def generate_begin(self, pixel_values: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor, max_new_tokens: int,
                       eos_ids: Sequence[int], image_index: Optional[torch.Tensor] = None, sample: Optional[dict] = None,
                       prompt_index: Optional[torch.Tensor] = None) -> dict:
        """The prefill of a greedy generation (vqa_clipt5_generate_prefill): the encoder pass of score_tensors over the same inputs (no
        labels), then the decoder start token and the first token. Returns the generation state that generate_step() advances: device
        tensors `tokens` [B, max_new_tokens] (-1 after a prompt's last token), `lengths` [B] and `all_done` [1], all owned by the state of
        this call shape. The generation workspace is separate from the scoring one, so scoring graphs are never invalidated by it.
        sample = dict(seeds=[one int per sequence], temperature=T, top_k=k, top_p=p) makes it a sampled generation
        (vqa_clipt5_generate_*_sampled) of B = len(seeds) sequences over the input_ids.shape[0] prompts: with fewer prompts than
        sequences, prompt_index (int32 [B] on the device) names each slot's prompt, and slot b < input_ids.shape[0] must be prompt b. The
        seeds go to a device buffer of the state before each prefill, so one captured step graph serves every seed."""
        dev = self.device
        self._check_inputs(pixel_values, image_index, input_ids, text_lens)
        n_prompts, L = input_ids.shape
        B = n_prompts
        NI = pixel_values.shape[0]
        max_new = int(max_new_tokens)
        eos = [int(e) for e in eos_ids]
        key = (B, NI, L, max_new, len(eos))
        if sample is not None:
            seeds = [int(x) for x in sample["seeds"]]
            B = len(seeds)
            if not all(0 <= x < 1 << 64 for x in seeds):
                raise ValueError("sampling needs one seed in [0, 2^64) per sequence")
            if B < n_prompts or (B > n_prompts and prompt_index is None):
                raise ValueError(f"{B} sequences over {n_prompts} prompts: need at least one sequence per prompt and, with more, prompt_index")
            if prompt_index is not None:
                assert prompt_index.is_cuda and prompt_index.dtype == torch.int32 and prompt_index.shape == (B,)
            smp_t, smp_k, smp_p = float(sample["temperature"]), int(sample["top_k"]), float(sample["top_p"])
            key = (B, NI, L, max_new, len(eos), "sample", smp_t, smp_k, smp_p)
        need = int(self.lib.vqa_clipt5_generate_workspace_bytes(self._h, B, NI, L, max_new))
        if need == 0:
            raise ValueError(f"bad generation size: batch {B}, images {NI}, prompt length {L}, max_new_tokens {max_new}")
        i32 = lambda *shape: torch.empty(*shape, dtype=torch.int32, device=dev)

        def make() -> dict:
            st = dict(B=B, NI=NI, L=L, max_new=max_new, n_eos=len(eos), eos=i32(max(len(eos), 1)), tokens=i32(B, max_new), lengths=i32(B),
                      all_done=i32(1), graph=None, sample=None)
            if sample is not None:
                sm = st["sample"] = dict(seeds=torch.empty(B, dtype=torch.int64, device=dev))
                sm["struct"] = _lib.VqaQwen25VLSampling(seeds=_ptr(sm["seeds"]), temperature=smp_t, top_k=smp_k, top_p=smp_p)
            return st
        st = self._gen_state(key, need, make)
        if eos:
            st["eos"].copy_(torch.as_tensor(eos, dtype=torch.int32), non_blocking=True)
        if st["sample"] is not None:
            # uint64 seeds in an int64 buffer: the same 8 bytes
            st["sample"]["seeds"].copy_(torch.tensor([x - (1 << 64) if x >= 1 << 63 else x for x in seeds], dtype=torch.int64), non_blocking=True)
        pdt = _dtype_code(pixel_values.dtype)

        def prefill():
            ws = self._gen_workspace
            head = (_ptr(pixel_values), pdt, NI, _ptr(image_index), _ptr(input_ids), _ptr(text_lens), B, L, _ptr(st["eos"]), len(eos), max_new,
                    _ptr(st["tokens"]), _ptr(st["lengths"]), _ptr(st["all_done"]))
            if st["sample"] is None:
                self._run("vqa_clipt5_generate_prefill", *head, _ptr(ws), ws.numel(), _stream_ptr(dev))
            else:
                self._run("vqa_clipt5_generate_prefill_sampled", *head, n_prompts, _ptr(prompt_index), C.byref(st["sample"]["struct"]), _ptr(ws),
                          ws.numel(), _stream_ptr(dev))
        st["prefill"] = prefill          # relaunches this prefill on the same device inputs (no host work)
        prefill()
        return st

    def generate_step(self, st: dict):
        """One decode step of the generation `st` (vqa_clipt5_generate_step, or _step_sampled), launched directly."""
        ws = self._gen_workspace
        head = (st["B"], st["NI"], st["L"], _ptr(st["eos"]), st["n_eos"], st["max_new"], _ptr(st["tokens"]), _ptr(st["lengths"]), _ptr(st["all_done"]))
        if st["sample"] is None:
            self._run("vqa_clipt5_generate_step", *head, _ptr(ws), ws.numel(), _stream_ptr(self.device))
        else:
            self._run("vqa_clipt5_generate_step_sampled", *head, C.byref(st["sample"]["struct"]), _ptr(ws), ws.numel(), _stream_ptr(self.device))

    def generate_tensors(self, pixel_values: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor, max_new_tokens: int,
                         eos_ids: Sequence[int], image_index: Optional[torch.Tensor] = None, use_graph: bool = True, check_every: int = 16):
        """Greedy generation (HF generate(do_sample=False, num_beams=1)) for a batch of prompts laid out as for score_tensors: one prefill,
        then decode steps replayed from a CUDA graph captured once per (batch, images, prompt length, max_new_tokens) and kept for the
        MAX_GEN_GRAPHS most recently used shapes. The host reads the all-finished flag through pinned memory every `check_every` steps and
        never synchronises in between. Returns each prompt's generated ids, the EOS id included when one ended it."""
        st = self.generate_begin(pixel_values, input_ids, text_lens, max_new_tokens, eos_ids, image_index)
        return self._decode_loop(st, use_graph, check_every)[0]

    def sample_tensors(self, pixel_values: torch.Tensor, input_ids: torch.Tensor, text_lens: torch.Tensor, max_new_tokens: int,
                       eos_ids: Sequence[int], seeds: Sequence[int], temperature: float, top_k: int, top_p: float,
                       image_index: Optional[torch.Tensor] = None, prompt_of_sample: Optional[Sequence[int]] = None, use_graph: bool = True,
                       check_every: int = 16):
        """Sampled generation (HF generate(do_sample=True) with the temperature, top_k and top_p warpers) of len(seeds) samples over the
        input_ids.shape[0] prompts laid out as for generate_tensors: sample s continues prompt prompt_of_sample[s] (None: sample s is
        prompt s) under seeds[s] (an integer in [0, 2^64)). Each prompt is encoded once however many samples it has, and sample s's tokens
        depend on its seed, prompt and the sizes only. Every prompt needs at least one sample. One prefill, then decode steps replayed from
        a CUDA graph captured once per (call shape, temperature, top_k, top_p). Returns each sample's generated ids in the caller's order,
        the EOS id included when one ended it."""
        n_prompts, B = input_ids.shape[0], len(seeds)
        owner = list(range(B)) if prompt_of_sample is None else [int(p) for p in prompt_of_sample]
        if len(owner) != B or not all(0 <= p < n_prompts for p in owner):
            raise ValueError(f"prompt_of_sample needs one prompt in [0, {n_prompts}) per sample ({B} samples)")
        firsts = {}
        for s, p in enumerate(owner):
            firsts.setdefault(p, s)
        if len(firsts) != n_prompts:
            raise ValueError(f"prompts {sorted(set(range(n_prompts)) - set(firsts))} have no sample")
        # slot p < n_prompts is prompt p's first sample (the encoded prompt itself); the other samples follow in the caller's order
        order = [firsts[p] for p in range(n_prompts)] + [s for s in range(B) if firsts[owner[s]] != s]
        prompt_index = None
        if B > n_prompts:
            prompt_index = torch.tensor([owner[s] for s in order], dtype=torch.int32).to(self.device)
        st = self.generate_begin(pixel_values, input_ids, text_lens, max_new_tokens, eos_ids, image_index, prompt_index=prompt_index,
                                 sample=dict(seeds=[int(seeds[s]) for s in order], temperature=temperature, top_k=top_k, top_p=top_p))
        ids = self._decode_loop(st, use_graph, check_every)[0]
        out: list = [None] * B
        for slot, s in enumerate(order):
            out[s] = ids[slot]
        return out


# ------------------------------------------------------------------------------------------------ single-kernel ops
class ops:
    """Kernel-level calls through the same C ABI (used by tests and bench.py's roofline probe)."""

    EPI = dict(store=0, quick_gelu=1, gelu=2, gated_gelu=3, relu=5, gated_silu=6)
    GATED = (3, 6)          # W = [gate; up] `gate_up_offset` rows apart, C has N / 2 columns

    @staticmethod
    def gemm(a: torch.Tensor, w: torch.Tensor, bias=None, residual=None, epilogue="store", variant=0, out=None,
             gate_up_offset=0):
        M, K = a.shape
        n_rows = w.shape[0]
        epi = ops.EPI[epilogue]
        gated = epi in ops.GATED
        n_out = n_rows // 2 if gated else n_rows
        if out is None:
            out = torch.empty(M, n_out, dtype=torch.bfloat16, device=a.device)
        _call("vqa_op_gemm_bf16", _ptr(a), a.stride(0), _ptr(w), w.stride(0), n_rows, _ptr(out), out.stride(0), M, n_rows, K, _ptr(bias),
              _ptr(residual), residual.stride(0) if residual is not None else 0, epi, gate_up_offset if gated else 0, variant,
              _stream_ptr(a.device))
        return out

    @staticmethod
    def gemm_normfuse(a: torch.Tensor, w: torch.Tensor, residual=None, epilogue="store", gate_up_offset=0, ssq_in=None, ssq_out=None,
                      norm_dim: int = 0, eps: float = 1e-6, out=None):
        """GEMM with the fused-RMSNorm hooks (see include/vqa_b200.h). ssq_in / ssq_out: fp32 [M, stride] cuda, stride % 4 == 0.
        Returns (C, number of ssq_out slots written)."""
        M, K = a.shape
        n_rows = w.shape[0]
        epi = ops.EPI[epilogue]
        gated = epi in ops.GATED
        n_out = n_rows // 2 if gated else n_rows
        if out is None:
            out = torch.empty(M, n_out, dtype=torch.bfloat16, device=a.device)
        buf = ssq_in if ssq_in is not None else ssq_out
        parts = C.c_int32(0)
        _call("vqa_op_gemm_bf16_normfuse", _ptr(a), a.stride(0), _ptr(w), w.stride(0), n_rows, _ptr(out), out.stride(0), M, n_rows, K,
              _ptr(residual), residual.stride(0) if residual is not None else 0, epi, gate_up_offset if gated else 0, _ptr(ssq_in),
              _ptr(ssq_out), buf.shape[1], norm_dim or K, float(eps), C.byref(parts), _stream_ptr(a.device))
        return out, int(parts.value)

    @staticmethod
    def lmhead_logprob(h: torch.Tensor, w: torch.Tensor, labels: torch.Tensor, temperature: float = 1.0, pen_bitmap=None,
                       repetition_penalty: float = 1.0):
        """The Qwen2.5-VL score's lm_head: log softmax(penalised bf16 logits / temperature)[labels] of h [M, K] against w [N, K], without
        materialising the logits. pen_bitmap int32 [M, ceil(N / 32)] or None. Returns fp32 [M]."""
        M, K = h.shape
        N = w.shape[0]
        out = torch.empty(M, dtype=torch.float32, device=h.device)
        st = _stream_ptr(h.device)
        args = (_ptr(h), h.stride(0), _ptr(w), w.stride(0), M, N, K, _ptr(labels), float(temperature), _ptr(pen_bitmap), float(repetition_penalty),
                _ptr(out))
        need = _size_query("vqa_op_lmhead_logprob", C.c_size_t, args, (st,))
        scratch = torch.empty((need + 3) // 4, dtype=torch.float32, device=h.device)
        _call("vqa_op_lmhead_logprob", *args, _ptr(scratch), scratch.numel() * 4, None, st)
        return out

    @staticmethod
    def attention(qkv: torch.Tensor, B: int, S: int, H: int, seq_lens=None, bias_table=None, scale=1.0,
                  bias_const_from: int = 0, round_scores: bool = False):
        """bias_const_from > 0 promises that bias_table[h] is constant for |key - query| >= bias_const_from on either side (T5:
        relative_attention_max_distance); 0 makes no assumption. round_scores: form the reference's bf16 score tensors before the softmax."""
        out = torch.empty(B * S, H * 64, dtype=torch.bfloat16, device=qkv.device)
        _call("vqa_op_attention_d64", _ptr(qkv), _ptr(out), B, S, H, _ptr(seq_lens), _ptr(bias_table), float(scale), int(bias_const_from),
              1 if round_scores else 0, _stream_ptr(qkv.device))
        return out

    @staticmethod
    def answer_logprob(logits: torch.Tensor, answer_ids: torch.Tensor, answer_counts: torch.Tensor, lengths: torch.Tensor, done: torch.Tensor,
                       max_new: int, temperature: float = 1.0, penalty_bitmap=None, repetition_penalty: float = 1.0, top_k: int = 0,
                       out_logp=None, out_topk_ids=None, out_topk_probs=None):
        """The per-step kernel of a scored rollout on given bf16 logits [B, V] (int32 answer_ids [B, n_max], answer_counts / lengths /
        done [B]; penalty_bitmap int32 [B, ceil(V / 32)] or None). Writes row lengths[b] of out_logp [B, max_new, n_max] and, with
        top_k > 0, of out_topk_ids / out_topk_probs [B, max_new, top_k]; returns the three outputs (allocated NaN / -1 when not given)."""
        B, V = logits.shape
        n_max = answer_ids.shape[1]
        dev = logits.device
        if out_logp is None:
            out_logp = torch.full((B, max_new, n_max), float("nan"), dtype=torch.float32, device=dev)
        if top_k > 0 and out_topk_ids is None:
            out_topk_ids = torch.full((B, max_new, top_k), -1, dtype=torch.int32, device=dev)
            out_topk_probs = torch.full((B, max_new, top_k), float("nan"), dtype=torch.float32, device=dev)
        _call("vqa_op_answer_logprob", _ptr(logits), B, V, _ptr(penalty_bitmap), float(repetition_penalty), float(temperature), _ptr(answer_ids),
              _ptr(answer_counts), n_max, max_new, _ptr(lengths), _ptr(done), top_k, _ptr(out_logp), _ptr(out_topk_ids), _ptr(out_topk_probs),
              _stream_ptr(dev))
        return out_logp, out_topk_ids, out_topk_probs

    @staticmethod
    def kv_cache_write(qkv: torch.Tensor, k_col0: int, v_col0: int, kv_heads: int, S: int, seq_lens: torch.Tensor, kc: torch.Tensor,
                       vc: torch.Tensor, gen_len=None):
        """The Qwen2.5-VL K/V cache write on packed rows qkv [B * S, ld] into kc / vc [B, kv_heads, cap, 128] (in place). gen_len None:
        prefill, row s < seq_lens[b] to slot s; gen_len int32 [B] (S == 1): decode, to slot seq_lens[b] + gen_len[b] - 1."""
        B, cap = kc.shape[0], kc.shape[2]
        _call("vqa_op_kv_cache_write", _ptr(qkv), qkv.stride(0), k_col0, v_col0, kv_heads, B, S, _ptr(seq_lens), _ptr(gen_len), _ptr(kc),
              _ptr(vc), cap, _stream_ptr(qkv.device))

    @staticmethod
    def decode_attention(q: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, seq_lens: torch.Tensor, gen_len: torch.Tensor, q_heads: int,
                         scale: float, splits: int = 0, out=None):
        """Flash-decoding attention of query rows q [B, >= q_heads * 128] (row stride q.stride(0)) over kc / vc [B, kv_heads, cap, 128],
        sequence b over slots [0, seq_lens[b] + gen_len[b]). splits == 0: the generation's rule. Returns (out [B, q_heads * 128] or the given
        out, splits used)."""
        B, kv_heads, cap = kc.shape[0], kc.shape[1], kc.shape[2]
        if out is None:
            out = torch.empty(B, q_heads * 128, dtype=torch.bfloat16, device=q.device)
        st = _stream_ptr(q.device)
        args = (_ptr(q), q.stride(0), _ptr(kc), _ptr(vc), cap, _ptr(seq_lens), _ptr(gen_len), B, q_heads, kv_heads, float(scale))
        if splits == 0:      # the rule's split count
            splits = _size_query("vqa_op_decode_attention_d128", C.c_int32, (*args, 0), (_ptr(out), out.stride(0), st))
        ws = torch.empty(max(1, B * q_heads * splits * 130), dtype=torch.float32, device=q.device)
        used = C.c_int32(0)
        _call("vqa_op_decode_attention_d128", *args, splits, _ptr(ws), ws.numel() * 4, C.byref(used), _ptr(out), out.stride(0), st)
        return out, int(used.value)

    @staticmethod
    def greedy_select(logits: torch.Tensor, tokens: torch.Tensor, lengths: torch.Tensor, done: torch.Tensor, n_done: torch.Tensor,
                      all_done: torch.Tensor, next_ids: torch.Tensor, eos_ids=None, pen_bitmap=None, repetition_penalty: float = 1.0,
                      first_pos=None, pos3=None):
        """One greedy selection step on bf16 logits [B, V] and the caller's int32 state (in place): tokens [B, max_new], lengths / done /
        next_ids [B], n_done / all_done [1], pen_bitmap [B, ceil(V / 32)] or None, first_pos [B] and pos3 [3, B] or both None."""
        B, V = logits.shape
        n_eos = eos_ids.numel() if eos_ids is not None else 0
        _call("vqa_op_greedy_select", _ptr(logits), B, V, _ptr(pen_bitmap), float(repetition_penalty), _ptr(eos_ids), n_eos, tokens.shape[1],
              _ptr(first_pos), _ptr(tokens), _ptr(lengths), _ptr(done), _ptr(n_done), _ptr(all_done), _ptr(next_ids), _ptr(pos3),
              _stream_ptr(logits.device))

    @staticmethod
    def sample_select(logits: torch.Tensor, seeds: torch.Tensor, temperature: float, top_k: int, top_p: float, tokens: torch.Tensor,
                      lengths: torch.Tensor, done: torch.Tensor, n_done: torch.Tensor, all_done: torch.Tensor, next_ids: torch.Tensor, eos_ids=None,
                      pen_bitmap=None, repetition_penalty: float = 1.0, first_pos=None, pos3=None, kept=None):
        """One sampled selection step (vqa_op_sample_select): greedy_select's state and arguments, plus int64 seeds [B] on the device and
        the warpers' (temperature, top_k, top_p; top_p goes to the kernel as the double it is, so its threshold is HF's fp32(1 - top_p)).
        kept: None or int32 [B, ceil(V / 32)] that receives each unfinished row's kept-id bitmap."""
        B, V = logits.shape
        n_eos = eos_ids.numel() if eos_ids is not None else 0
        smp = _lib.VqaQwen25VLSampling(seeds=_ptr(seeds), temperature=float(temperature), top_k=int(top_k), top_p=float(top_p))
        _call("vqa_op_sample_select", _ptr(logits), B, V, _ptr(pen_bitmap), float(repetition_penalty), _ptr(eos_ids), n_eos, tokens.shape[1],
              _ptr(first_pos), _ptr(tokens), _ptr(lengths), _ptr(done), _ptr(n_done), _ptr(all_done), _ptr(next_ids), _ptr(pos3), C.byref(smp),
              _ptr(kept), _stream_ptr(logits.device))

    @staticmethod
    def clipt5_expand_prompts(xn: torch.Tensor, xt: torch.Tensor, seq_lens: torch.Tensor, n_prompts: int, prompt_index=None):
        """The encoder sharing of the sampled CLIP-FlanT5 prefill (vqa_op_clipt5_expand_prompts), in place: slots b >= n_prompts of xn
        bf16 [B, S, d_model], xt bf16 [B, d_model, Sp] and seq_lens int32 [B] become copies of slot prompt_index[b] (int32 [B])."""
        B, S, D = xn.shape
        assert xt.shape == (B, D, (S + 7) // 8 * 8) and seq_lens.shape == (B,)
        _call("vqa_op_clipt5_expand_prompts", _ptr(xn), _ptr(xt), _ptr(seq_lens), _ptr(prompt_index), int(n_prompts), B, S, D,
              _stream_ptr(xn.device))

    @staticmethod
    def t5_bucket_lut(bidirectional: bool, num_buckets: int, max_distance: int) -> torch.Tensor:
        """The engine's relative-position bucket table (host): int32 [2 * max_distance + 1], entry rel + max_distance."""
        out = torch.empty(2 * max_distance + 1, dtype=torch.int32)
        _call("vqa_t5_bucket_lut", 1 if bidirectional else 0, num_buckets, max_distance, C.cast(out.data_ptr(), C.POINTER(C.c_int32)))
        return out

    @staticmethod
    def t5_decoder_self_attn(qkv: torch.Tensor, B: int, T: int, H: int, rel_emb: torch.Tensor, bucket_lut: torch.Tensor, max_distance: int,
                             round_scores: bool = False):
        """The scoring path's T5 decoder self-attention: qkv [B * T, 3 * H * 64] -> [B * T, H * 64]; bucket_lut on the device."""
        out = torch.empty(B * T, H * 64, dtype=torch.bfloat16, device=qkv.device)
        _call("vqa_op_t5_decoder_self_attn", _ptr(qkv), _ptr(out), _ptr(rel_emb), _ptr(bucket_lut), max_distance, B, T, H,
              1 if round_scores else 0, _stream_ptr(qkv.device))
        return out

    @staticmethod
    def t5_decode_self_attn(qkv: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, lengths: torch.Tensor, rel_emb: torch.Tensor,
                            bucket_lut: torch.Tensor, max_distance: int, round_scores: bool = False, out=None):
        """One cached T5 decoder self-attention layer of a generation step: the row qkv [B, 3 * H * 64] of sequence b is appended to
        kc / vc [B, H, cap, 64] at min(lengths[b], cap - 1) (in place) and attends to the slots up to it. Returns out [B, H * 64]."""
        B, H, cap = kc.shape[0], kc.shape[1], kc.shape[2]
        if out is None:
            out = torch.empty(B, H * 64, dtype=torch.bfloat16, device=qkv.device)
        _call("vqa_op_t5_decode_self_attn", _ptr(qkv), _ptr(kc), _ptr(vc), cap, _ptr(lengths), _ptr(out), _ptr(rel_emb), _ptr(bucket_lut),
              max_distance, B, H, 1 if round_scores else 0, _stream_ptr(qkv.device))
        return out

    @staticmethod
    def norm(x: torch.Tensor, gamma: torch.Tensor, eps=1e-6, out=None):
        """T5LayerNorm / Qwen RMSNorm of the rows of x [rows, D] bf16: gamma * bf16(x * rsqrt(mean(x^2) + eps))."""
        y = torch.empty_like(x) if out is None else out
        _call("vqa_op_norm", _ptr(x), _ptr(gamma), _ptr(y), x.shape[0], x.shape[1], float(eps), _stream_ptr(x.device))
        return y

    @staticmethod
    def patchify(pixels: torch.Tensor, patch: int, kpad: int, out=None):
        """The patch gather of the CLIP tower: pixels [n, 3, S, S] fp32 / bf16 -> bf16 [n * (S / patch)^2, kpad]."""
        n, S = pixels.shape[0], pixels.shape[2]
        if out is None:
            out = torch.empty(n * (S // patch) ** 2, kpad, dtype=torch.bfloat16, device=pixels.device)
        _call("vqa_op_patchify", _ptr(pixels), _dtype_code(pixels.dtype), n, S, patch, kpad, _ptr(out), _stream_ptr(pixels.device))
        return out

    @staticmethod
    def splice_embed(ids: torch.Tensor, text_lens: torch.Tensor, image_index, shared: torch.Tensor, feats: torch.Tensor, P: int,
                     rows_per_image: int, row_offset: int = 1, image_token: int = -200, out=None, seq_lens=None):
        """The multimodal splice: ids int32 [B, L], text_lens int32 [B], image_index int32 [B] or None, shared [vocab, D], feats [rows, >= D]
        (row stride feats.stride(0)), image i's P feature rows from row i * rows_per_image + row_offset. Returns (out [B, L - 1 + P, D],
        seq_lens int32 [B])."""
        B, L = ids.shape
        D = shared.shape[1]
        if out is None:
            out = torch.empty(B, L - 1 + P, D, dtype=torch.bfloat16, device=ids.device)
        if seq_lens is None:
            seq_lens = torch.empty(B, dtype=torch.int32, device=ids.device)
        _call("vqa_op_splice_embed", _ptr(ids), _ptr(text_lens), _ptr(image_index), _ptr(shared), _ptr(feats), feats.stride(0), row_offset,
              rows_per_image, _ptr(out), _ptr(seq_lens), B, L, P, D, image_token, _stream_ptr(ids.device))
        return out, seq_lens

    @staticmethod
    def decoder_embed(labels, shared: torch.Tensor, B: int, T: int, start_id: int = 0, pad_id: int = 0, out=None):
        """Decoder input embeddings of shift_right(labels int32 [B, T]) (labels None: T = 1, the start token). Returns [B * T, D]."""
        D = shared.shape[1]
        if out is None:
            out = torch.empty(B * T, D, dtype=torch.bfloat16, device=shared.device)
        _call("vqa_op_decoder_embed", _ptr(labels), _ptr(shared), _ptr(out), B, T, D, start_id, pad_id, _stream_ptr(shared.device))
        return out

    @staticmethod
    def t5_bias_table(rel_emb: torch.Tensor, bucket_lut: torch.Tensor, max_distance: int, S: int, out=None):
        """The encoder's relative-position bias table fp32 [H, 2S - 1] from rel_emb bf16 [buckets, H] and a device bucket LUT."""
        H = rel_emb.shape[1]
        if out is None:
            out = torch.empty(H, 2 * S - 1, dtype=torch.float32, device=rel_emb.device)
        _call("vqa_op_t5_bias_table", _ptr(rel_emb), _ptr(bucket_lut), max_distance, _ptr(out), H, S, _stream_ptr(rel_emb.device))
        return out

    @staticmethod
    def lmhead_score(h: torch.Tensor, w: torch.Tensor, labels: torch.Tensor, scores=None, logprobs=None):
        """The CLIP-FlanT5 score's lm_head and finalisation: h [B * T, K] against w [N, K], labels int32 [B, T]. Returns (scores fp32 [B],
        logprobs fp32 [B * T]); both are allocated NaN-filled when not given, and ignored positions of logprobs keep their value."""
        B, T = labels.shape
        N, K = w.shape[0], h.shape[1]
        if scores is None:
            scores = torch.full((B,), float("nan"), dtype=torch.float32, device=h.device)
        if logprobs is None:
            logprobs = torch.full((B * T,), float("nan"), dtype=torch.float32, device=h.device)
        st = _stream_ptr(h.device)
        args = (_ptr(h), h.stride(0), _ptr(w), w.stride(0), B, T, N, K, _ptr(labels), _ptr(scores), _ptr(logprobs))
        need = _size_query("vqa_op_lmhead_score", C.c_size_t, args, (st,))
        scratch = torch.empty((need + 3) // 4, dtype=torch.float32, device=h.device)
        _call("vqa_op_lmhead_score", *args, _ptr(scratch), scratch.numel() * 4, None, st)
        return scores, logprobs

    @staticmethod
    def row_ssq(x: torch.Tensor, ssq: torch.Tensor):
        """Sum of squares of the rows of x bf16 [rows, D] into column 0 of ssq fp32 [rows, stride] (in place)."""
        _call("vqa_op_row_ssq", _ptr(x), _ptr(ssq), x.shape[0], x.shape[1], ssq.stride(0), _stream_ptr(x.device))
        return ssq

    @staticmethod
    def gemm_f32acc(a: torch.Tensor, w: torch.Tensor, c: torch.Tensor, bias=None, variant=0):
        """The CLIP tower's residual GEMM: fp32 c[M, N] += bf16(a . w^T + bias), in place (row stride c.stride(0))."""
        M, K = a.shape
        N = w.shape[0]
        _call("vqa_op_gemm_bf16_f32acc", _ptr(a), a.stride(0), _ptr(w), w.stride(0), N, _ptr(c), c.stride(0), M, N, K, _ptr(bias), variant,
              _stream_ptr(a.device))
        return c

    @staticmethod
    def gemm_batched(a: torch.Tensor, w: torch.Tensor, c: torch.Tensor, M: int, N: int, K: int, nb: int, a_off=(0, 0), w_off=(0, 0),
                     c_stride: int = 0, a_extent=None, w_extent=None, variant: int = 0):
        """`nb` store-GEMMs in one launch (see vqa_op_gemm_bf16_batched): batch b reads a at (row, k) + b * a_off, w at (row, k) + b * w_off
        and writes c.flatten()[b * c_stride + m * c.stride(0) + n]. a_extent / w_extent (rows, cols) default to the tensors' shapes."""
        a_rows, a_cols = a_extent or a.shape
        w_rows, w_cols = w_extent or w.shape
        _call("vqa_op_gemm_bf16_batched", _ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(c), c.stride(0), M, N, K, nb, a_off[0], a_off[1],
              w_off[0], w_off[1], c_stride, a_rows, a_cols, w_rows, w_cols, variant, _stream_ptr(a.device))
        return c

    @staticmethod
    def t5_cross_attention(q: torch.Tensor, x: torch.Tensor, seq_lens: torch.Tensor, wkT, wkv: torch.Tensor, B: int, T: int, S: int, H: int,
                           mode: int = 0, round_scores: bool = False, out=None, workspace=None):
        """One CLIP-FlanT5 decoder cross-attention layer (see vqa_op_t5_cross_attention): mode 0 absorbed, mode 1 the reference association.
        Returns (out [B * T, H * 64], the uint8 workspace, whose mode-0 layout the header documents)."""
        Dm = x.shape[1]
        if out is None:
            out = torch.empty(B * T, H * 64, dtype=torch.bfloat16, device=q.device)
        st = _stream_ptr(q.device)
        args = (_ptr(q), _ptr(x), _ptr(seq_lens), _ptr(wkT), _ptr(wkv), _ptr(out), B, T, S, H, Dm, mode, 1 if round_scores else 0)
        if workspace is None:
            workspace = torch.empty(_size_query("vqa_op_t5_cross_attention", C.c_size_t, args, (st,)), dtype=torch.uint8, device=q.device)
        _call("vqa_op_t5_cross_attention", *args, _ptr(workspace), workspace.numel(), None, st)
        return out, workspace

    @staticmethod
    def layernorm_f32(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5, out=None):
        """LayerNorm of an fp32 [rows, D] stream into bf16 (the CLIP tower's ln1 / ln2)."""
        if out is None:
            out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
        _call("vqa_op_layernorm_f32", _ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), x.shape[0], x.shape[1], float(eps), _stream_ptr(x.device))
        return out

    @staticmethod
    def clip_embed_ln(patch: torch.Tensor, cls: torch.Tensor, pos: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, n_images: int,
                      eps: float = 1e-5, out=None):
        """CLIP embeddings + pre_layrnorm: patch rows [n_images * P, D] -> fp32 [n_images * (P + 1), D]."""
        P, D = patch.shape[0] // n_images, patch.shape[1]
        if out is None:
            out = torch.empty(n_images * (P + 1), D, dtype=torch.float32, device=patch.device)
        _call("vqa_op_clip_embed_ln", _ptr(patch), _ptr(cls), _ptr(pos), _ptr(gamma), _ptr(beta), _ptr(out), n_images, P, D, float(eps),
              _stream_ptr(patch.device))
        return out

    @staticmethod
    def attention_d128(qkv: torch.Tensor, out: torch.Tensor, q_col0: int, k_col0: int, v_col0: int, n_seq: int, max_len: int, q_heads: int,
                       kv_group: int, scale: float, causal: bool, S: int = 0, seq_lens=None, cu_seqlens=None, kv_prefix=None,
                       pair_sequences: bool = False, o_head_stride: int = 128, d_out: int = 128, rows: Optional[int] = None):
        """Head-dim-128 attention on packed rows qkv [rows, ld] into out (row stride out.stride(0)), in place: fixed stride S with seq_lens
        [n_seq] (cu_seqlens None, vqa_op_attention_d128), or variable-length cu_seqlens [n_seq + 1] with the extras of
        vqa_op_attention_d128_ex. rows defaults to qkv.shape[0]."""
        rows = qkv.shape[0] if rows is None else rows
        st = _stream_ptr(qkv.device)
        if cu_seqlens is None:
            _call("vqa_op_attention_d128", _ptr(qkv), qkv.stride(0), rows, q_col0, k_col0, v_col0, _ptr(out), out.stride(0), n_seq, max_len, S,
                  q_heads, kv_group, None, _ptr(seq_lens), float(scale), 1 if causal else 0, st)
        else:
            _call("vqa_op_attention_d128_ex", _ptr(qkv), qkv.stride(0), rows, q_col0, k_col0, v_col0, _ptr(out), out.stride(0), n_seq, max_len,
                  q_heads, kv_group, _ptr(cu_seqlens), _ptr(kv_prefix), float(scale), 1 if causal else 0, 1 if pair_sequences else 0,
                  o_head_stride, d_out, st)
        return out

    @staticmethod
    def qwen_rope(positions: torch.Tensor, axis_of_dim: torch.Tensor, inv_freq: torch.Tensor, x: torch.Tensor, col0: int, n_heads: int,
                  head_stride: int, head_dim: int, text_mode: bool, cos_t=None, sin_t=None):
        """M-RoPE as the scoring path applies it: tables from positions int32 [n_axes, rows], axis_of_dim int32 / inv_freq fp32 [head_dim / 2]
        into cos_t / sin_t fp32 [rows, head_dim] (allocated when None), then n_heads heads of x bf16 [rows, ld] rotated in place.
        Returns (cos_t, sin_t)."""
        rows = positions.shape[1]
        if cos_t is None:
            cos_t = torch.empty(rows, head_dim, dtype=torch.float32, device=x.device)
            sin_t = torch.empty(rows, head_dim, dtype=torch.float32, device=x.device)
        _call("vqa_op_qwen_rope", _ptr(positions), rows, _ptr(axis_of_dim), _ptr(inv_freq), head_dim // 2, _ptr(cos_t), _ptr(sin_t), _ptr(x),
              x.stride(0), col0, n_heads, head_stride, head_dim, 1 if text_mode else 0, _stream_ptr(x.device))
        return cos_t, sin_t

    @staticmethod
    def gather_rows(src: torch.Tensor, index: torch.Tensor, group: int, out=None):
        """out row r = src row index[r / group] * group + r % group, for every row of out (default: src's shape)."""
        if out is None:
            out = torch.empty_like(src)
        _call("vqa_op_gather_rows", _ptr(src), _ptr(out), _ptr(index), out.shape[0], group, out.shape[1], _stream_ptr(src.device))
        return out

    @staticmethod
    def qwen_embed(ids: torch.Tensor, feat_index: torch.Tensor, seq_lens: torch.Tensor, embed: torch.Tensor, feats: torch.Tensor, S: int, out=None):
        """The embedding splice over rows = ids.numel() rows of S (packed rows: seq_lens = cu_seqlens[n_seq:], S = rows). Returns out [rows, D]."""
        rows, D = ids.numel(), embed.shape[1]
        if out is None:
            out = torch.empty(rows, D, dtype=torch.bfloat16, device=embed.device)
        _call("vqa_op_qwen_embed", _ptr(ids), _ptr(feat_index), _ptr(seq_lens), _ptr(embed), _ptr(feats), _ptr(out), rows, S, D,
              _stream_ptr(embed.device))
        return out

    @staticmethod
    def token_bitmap(ids: torch.Tensor, vocab: int, B: int, seq_lens=None, S: int = 0, cu_seqlens=None, kv_prefix=None, pair_seq=None,
                     max_prompt_len: int = 0, bitmap=None):
        """The repetition-penalty bitmap int32 [B, ceil(vocab / 32)] (zeroed here when not given) of padded prompts (seq_lens, S) or packed
        rows (cu_seqlens, kv_prefix, pair_seq, max_prompt_len)."""
        if bitmap is None:
            bitmap = torch.zeros(B, (vocab + 31) // 32, dtype=torch.int32, device=ids.device)
        _call("vqa_op_token_bitmap", _ptr(ids), _ptr(seq_lens), B, S, _ptr(cu_seqlens), _ptr(kv_prefix), _ptr(pair_seq), max_prompt_len, vocab,
              _ptr(bitmap), _stream_ptr(ids.device))
        return bitmap

    @staticmethod
    def topk_softmax(logits: torch.Tensor, K: int, V: Optional[int] = None, temperature: float = 1.0, pen_bitmap=None,
                     repetition_penalty: float = 1.0):
        """The trace top-K of bf16 logits [B, >= V] (row stride logits.stride(0)): (ids int32 [B, K], probabilities fp32 [B, K])."""
        B = logits.shape[0]
        V = logits.shape[1] if V is None else V
        ids = torch.full((B, K), -2, dtype=torch.int32, device=logits.device)
        probs = torch.full((B, K), float("nan"), dtype=torch.float32, device=logits.device)
        _call("vqa_op_topk_softmax", _ptr(logits), logits.stride(0), B, V, float(temperature), _ptr(pen_bitmap), float(repetition_penalty), K,
              _ptr(ids), _ptr(probs), _stream_ptr(logits.device))
        return ids, probs


# ------------------------------------------------------------------------------------------------ image pre-processing
class _PinnedRing:
    """A few pinned host buffers handed to the library as `host_staging`, each guarded by a CUDA event recorded after the call that
    used it, so a buffer is never rewritten before the stream has consumed it (keeps the pre-processing call fully asynchronous)."""

    def __init__(self, slots: int = 4):
        self.bufs = [None] * slots
        self.events = [None] * slots
        self.i = 0

    def acquire(self, nbytes: int) -> torch.Tensor:
        self.i = (self.i + 1) % len(self.bufs)
        if self.events[self.i] is not None:
            self.events[self.i].synchronize()
        if self.bufs[self.i] is None or self.bufs[self.i].numel() < nbytes:
            self.bufs[self.i] = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, pin_memory=True)
        return self.bufs[self.i]

    def release(self, device):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        self.events[self.i] = ev


_staging_rings: Dict[int, _PinnedRing] = {}


def _staging(device: torch.device) -> _PinnedRing:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _staging_rings:
        _staging_rings[idx] = _PinnedRing()
    return _staging_rings[idx]


CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def _upload_u8(items, dev: torch.device):
    """The uint8 pixels of `items` (images [h, w, 3] or frame stacks [n, h, w, 3]) as one device byte buffer, item after item, and the
    byte offset of every frame in it. A packed [n, h, w, 3] tensor of equal-size images is used in place on the device or sent with one
    H2D copy; a list of device tensors is concatenated; a list with host tensors is staged once in pinned memory and copied once."""
    offs, total = [], 0
    for it in items:
        step = int(it.shape[-3]) * int(it.shape[-2]) * 3
        offs.extend(total + f * step for f in range(int(it.shape[0]) if it.dim() == 4 else 1))
        total += int(it.numel())
    if isinstance(items, torch.Tensor):
        src = items.contiguous().view(-1)
        src = src if src.is_cuda else src.to(dev, non_blocking=True)
    elif all(it.is_cuda for it in items):
        src = items[0].contiguous().view(-1) if len(items) == 1 else torch.cat([it.contiguous().view(-1) for it in items])
    else:
        stage = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        o = 0
        for it in items:
            stage[o:o + it.numel()] = it.contiguous().view(-1)
            o += it.numel()
        src = stage.to(dev, non_blocking=True)
    return src, offs


def clip_preprocess_u8(images: Sequence[torch.Tensor], out_size: int, device, pad: bool = True, mean=CLIP_MEAN, std=CLIP_STD,
                       background=None, out_dtype: torch.dtype = torch.float32, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Decoded images (uint8 HWC RGB tensors, each [h, w, 3], on the host or on `device`) -> CLIP input [n, 3, S, S] on the device,
    by ONE kernel launch of libvqa_b200.so: expand2square (reference mm_utils.py:128-139, background = int(mean * 255)) + PIL-exact
    bicubic resize + centre crop + /255 + normalise. Host images are packed into one pinned buffer and copied once (a 512x512 image
    is 0.79 MB as uint8 against 1.35 MB as the fp32 336x336 tensor the CPU path ships). Enqueued on the current stream."""
    lib = _lib.load()
    dev = torch.device(device)
    n = len(images)
    assert n > 0
    for im in images:
        assert im.dtype == torch.uint8 and im.dim() == 3 and im.shape[2] == 3, "images must be uint8 [h, w, 3]"
    src, offs = _upload_u8(images, dev)
    H = (C.c_int32 * n)(*[int(im.shape[0]) for im in images])
    W = (C.c_int32 * n)(*[int(im.shape[1]) for im in images])
    need = int(lib.vqa_clip_preprocess_workspace_bytes(H, W, n, out_size, 1 if pad else 0))
    if need == 0:
        raise RuntimeError(f"vqa_clip_preprocess_workspace_bytes: {_lib.last_error(None)}")
    wsb = torch.empty(need, dtype=torch.uint8, device=dev)
    if out is None:
        out = torch.empty(n, 3, out_size, out_size, dtype=out_dtype, device=dev)
    assert out.is_cuda and out.is_contiguous() and out.shape == (n, 3, out_size, out_size) and out.dtype in (torch.float32, torch.bfloat16)
    bg = background if background is not None else tuple(int(x * 255) for x in mean)
    ring = _staging(dev)
    hs = ring.acquire(need)
    with torch.cuda.device(dev):
        rc = lib.vqa_clip_preprocess(_ptr(src), (C.c_int64 * n)(*offs), H, W, n, out_size, 1 if pad else 0, (C.c_uint8 * 3)(*bg),
                                     (C.c_float * 3)(*mean), (C.c_float * 3)(*std), _ptr(out), _dtype_code(out.dtype), _ptr(wsb), need,
                                     hs.data_ptr(), _stream_ptr(dev))
    ring.release(dev)
    _check(rc, None, "vqa_clip_preprocess")
    # src / wsb stay referenced by the caching allocator's stream ordering: both were allocated on the current stream
    return out


# Decoded images of one CLIP call go to the device in slices of at most this many bytes of uint8 pixels (at least one image per slice):
# the concatenated frames of a video are one wide image (a 1080p 8-frame canvas is 50 MB), so a call of many videos is uploaded and
# resized piecewise into one output tensor instead of being staged whole in pinned memory.
CLIP_SLICE_BYTES = 64 << 20


def clip_preprocess_u8_sliced(images: Sequence[torch.Tensor], out_size: int, device, pad: bool = True,
                              out_dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """clip_preprocess_u8 over consecutive slices of `images` of at most CLIP_SLICE_BYTES each, one kernel launch per slice, written into
    the rows of one [n, 3, S, S] tensor. A call whose images fit one slice is exactly one clip_preprocess_u8 call."""
    n = len(images)
    assert n > 0
    out = torch.empty(n, 3, out_size, out_size, dtype=out_dtype, device=torch.device(device))
    lo = 0
    while lo < n:
        hi, nbytes = lo + 1, int(images[lo].numel())
        while hi < n and nbytes + int(images[hi].numel()) <= CLIP_SLICE_BYTES:
            nbytes += int(images[hi].numel())
            hi += 1
        clip_preprocess_u8(images[lo:hi], out_size, device, pad=pad, out=out[lo:hi])
        lo = hi
    return out


def _qwen_plan(n_frames, heights, widths, is_video, patch: int, temporal_patch: int, merge: int, min_pixels: int, max_pixels: int):
    """vqa_qwen_preprocess_video_plan (host only) -> ([(t, gh, gw), ...], total patch rows, workspace bytes)."""
    n = len(heights)
    i32 = lambda v: (C.c_int32 * n)(*v)
    grid = (C.c_int32 * (3 * n))()
    rows, need = C.c_int64(0), C.c_size_t(0)
    _call("vqa_qwen_preprocess_video_plan", i32(n_frames), i32(heights), i32(widths), i32(is_video), n, patch, temporal_patch, merge, min_pixels,
          max_pixels, grid, C.byref(rows), C.byref(need))
    return [tuple(int(grid[3 * i + k]) for k in range(3)) for i in range(n)], int(rows.value), int(need.value)


def qwen_preprocess_plan(sizes_hw: Sequence[Sequence[int]], patch: int = 14, merge: int = 2, min_pixels: int = 56 * 56,
                         max_pixels: int = 14 * 14 * 4 * 1280):
    """Host-only geometry of the Qwen pre-processing (smart_resize): -> ([(1, gh, gw), ...], total patch rows, workspace bytes)."""
    n = len(sizes_hw)
    # still images: the temporal patch size changes neither the rows nor the workspace
    return _qwen_plan([1] * n, [int(s[0]) for s in sizes_hw], [int(s[1]) for s in sizes_hw], [0] * n, patch, 1, merge, min_pixels, max_pixels)


def qwen_preprocess_u8(images: Sequence[torch.Tensor], device, patch: int = 14, temporal_patch: int = 2, merge: int = 2,
                       min_pixels: int = 56 * 56, max_pixels: int = 14 * 14 * 4 * 1280, mean=CLIP_MEAN, std=CLIP_STD,
                       out_dtype: torch.dtype = torch.float32):
    """Decoded still images (uint8 HWC RGB, host or device; a packed [n, h, w, 3] tensor is n stills) -> (pixel_patches
    [sum gh*gw, 3*temporal*patch^2] on the device, [(1, gh, gw), ...]) by ONE kernel launch: smart_resize + PIL-exact bicubic + /255 +
    normalise + frame duplication + merge-order patch rows -- bit-identical to models/vqascore_models/qwen_utils.qwen_image_to_patches
    (the CPU path). The still-image case of qwen_preprocess_video_u8."""
    for im in images:
        assert im.dtype == torch.uint8 and im.dim() == 3 and im.shape[2] == 3, "images must be uint8 [h, w, 3]"
    return qwen_preprocess_video_u8(images, device, patch, temporal_patch, merge, min_pixels, max_pixels, mean, std, out_dtype)


def qwen_preprocess_video_u8(items: Sequence[torch.Tensor], device, patch: int = 14, temporal_patch: int = 2, merge: int = 2,
                             min_pixels: int = 56 * 56, max_pixels: int = 14 * 14 * 4 * 1280, mean=CLIP_MEAN, std=CLIP_STD,
                             out_dtype: torch.dtype = torch.float32):
    """Decoded still images (uint8 [h, w, 3]) and video frame stacks (uint8 [n, h, w, 3]), host or device, in any mix -> (pixel_patches
    [sum t*gh*gw, 3*temporal*patch^2] on the device, [(t, gh, gw), ...]) by ONE kernel launch (vqa_qwen_preprocess_video): every frame
    gets the still-image pre-processing of qwen_preprocess_u8, and a stack's frames fill consecutive temporal slots of its patch rows, the
    last frame repeated into the slots a count that is not a multiple of temporal_patch leaves -- bit-identical to
    models/vqascore_models/qwen_utils.qwen_video_to_patches. A still keeps grid t = 1 and the rows of qwen_preprocess_u8. A packed
    [n, h, w, 3] tensor is n still images."""
    lib = _lib.load()
    dev = torch.device(device)
    n = len(items)
    assert n > 0
    for it in items:
        assert it.dtype == torch.uint8 and it.dim() in (3, 4) and it.shape[-1] == 3, "items must be uint8 [h, w, 3] or [n, h, w, 3]"
    nf = [int(it.shape[0]) if it.dim() == 4 else 1 for it in items]
    hs, ws = [int(it.shape[-3]) for it in items], [int(it.shape[-2]) for it in items]
    vid = [int(it.dim() == 4) for it in items]
    grids, rows, need = _qwen_plan(nf, hs, ws, vid, patch, temporal_patch, merge, min_pixels, max_pixels)
    src, offs = _upload_u8(items, dev)
    out = torch.empty(rows, 3 * temporal_patch * patch * patch, dtype=out_dtype, device=dev)
    wsb = torch.empty(max(need, 16), dtype=torch.uint8, device=dev)
    i32 = lambda v: (C.c_int32 * n)(*v)
    ring = _staging(dev)
    stage_buf = ring.acquire(wsb.numel())
    with torch.cuda.device(dev):
        rc = lib.vqa_qwen_preprocess_video(_ptr(src), (C.c_int64 * len(offs))(*offs), i32(nf), i32(hs), i32(ws), i32(vid), n, patch,
                                           temporal_patch, merge, min_pixels, max_pixels, (C.c_float * 3)(*mean), (C.c_float * 3)(*std),
                                           _ptr(out), _dtype_code(out_dtype), _ptr(wsb), wsb.numel(), stage_buf.data_ptr(), _stream_ptr(dev))
    ring.release(dev)
    _check(rc, None, "vqa_qwen_preprocess_video")
    return out, grids


# Frames of a video file go to the device in slices of at most this many bytes (at least one frame), so that host and device staging
# stay bounded for long or large clips.
VIDEO_SLICE_BYTES = 32 << 20


@functools.lru_cache(maxsize=64)
def _aa_bicubic_taps(in_size: int, out_size: int):
    """torch's fp32 weights of interpolate(mode="bicubic", antialias=True, align_corners=False) along one axis, in_size -> out_size, as
    (first input of each output's window int32 [out], weights fp32 [out, taps], taps). They are read off torch itself: channel j of the
    input holds an impulse at position j, so output i of channel j is weight (i, j) exactly, whatever order torch sums in (every other
    term is 0). An axis whose size does not change is copied, as torch does (weight 1)."""
    eye = torch.eye(in_size, dtype=torch.float32)[None, :, None, :]
    w = torch.nn.functional.interpolate(eye, size=(1, out_size), mode="bicubic", antialias=True, align_corners=False)[0, :, 0, :].t()
    nz = (w != 0).int()
    lo, hi = nz.argmax(1), in_size - 1 - nz.flip(1).argmax(1)
    # a window whose first tap has weight exactly 0 starts one later than its neighbour's: the suffix minimum keeps the starts
    # non-decreasing (the kernel's bands need it) and only adds zero-weight taps
    first = lo.flip(0).cummin(0).values.flip(0)
    taps = int((hi - first).max()) + 1
    first = torch.clamp(first, max=in_size - taps)
    return first.to(torch.int32).contiguous(), torch.gather(w, 1, first[:, None] + torch.arange(taps)).contiguous(), taps


def qwen_preprocess_video_file_u8(frames, size, device, n_frames: Optional[int] = None, patch: int = 14, temporal_patch: int = 2,
                                  merge: int = 2, mean=CLIP_MEAN, std=CLIP_STD, out_dtype: torch.dtype = torch.float32):
    """Frames sampled from one video file -> (pixel_patches [t*gh*gw, 3*temporal*patch^2] on the device, (t, gh, gw)), what qwen_vl_utils
    fetch_video + Qwen2VLVideoProcessor(do_resize=False) make of them: torchvision's antialiased bicubic resize to size = (rh, rw) in
    fp32 with torch's weights, round half to even, then the frame-stack patch rows of qwen_preprocess_video_u8. `frames` is uint8
    [n, h, w, 3] RGB (host or device), or an iterable of such slices of one video with n_frames their total; a host tensor goes to the
    device in slices of VIDEO_SLICE_BYTES. One kernel launch (vqa_qwen_preprocess_video_aa) per slice. The resized uint8 frames equal
    models/vqascore_models/qwen_utils.qwen_video_file_to_patches's except where torch's fp32 value is a rounding tie that a different
    summation order on the host's CPU puts on the other side (DESIGN §4)."""
    lib = _lib.load()
    dev = torch.device(device)
    if isinstance(frames, torch.Tensor) or hasattr(frames, "__array__"):
        frames = torch.as_tensor(frames)
        n_frames = int(frames.shape[0])
        per = max(1, VIDEO_SLICE_BYTES // max(1, frames[0].numel()))
        frames = [frames[i:i + per] for i in range(0, n_frames, per)]
    assert n_frames is not None and n_frames > 0, "n_frames must be given with an iterable of slices"
    rh, rw = (int(s) for s in size)
    i32p, f32p = C.POINTER(C.c_int32), C.POINTER(C.c_float)
    ip = lambda t: C.cast(t.data_ptr(), i32p)
    fp = lambda t: C.cast(t.data_ptr(), f32p)
    ring = _staging(dev)
    hw, out, done = None, None, 0
    for sl in frames:
        sl = torch.as_tensor(sl)
        assert sl.dtype == torch.uint8 and sl.dim() == 4 and sl.shape[-1] == 3, "frames must be uint8 [n, h, w, 3]"
        k = int(sl.shape[0])
        if hw is None:
            hw = (int(sl.shape[1]), int(sl.shape[2]))
            (fh, wh, th), (fv, wv, tv) = _aa_bicubic_taps(hw[1], rw), _aa_bicubic_taps(hw[0], rh)
            rows, need = C.c_int64(0), C.c_size_t(0)
            _check(lib.vqa_qwen_preprocess_video_aa_plan(hw[0], hw[1], rh, rw, ip(fh), th, ip(fv), tv, patch, temporal_patch, merge, n_frames,
                                                         C.byref(rows), C.byref(need)), None, "vqa_qwen_preprocess_video_aa_plan")
            out = torch.empty(int(rows.value), 3 * temporal_patch * patch * patch, dtype=out_dtype, device=dev)
            wsb = torch.empty(int(need.value), dtype=torch.uint8, device=dev)
        assert tuple(sl.shape[1:3]) == hw, "all frames of a video must have one size"
        assert done + k <= n_frames, "more frames than n_frames"
        if sl.is_cuda:
            src = sl.contiguous()
        else:
            stage = ring.acquire(sl.numel())
            stage[:sl.numel()].copy_(sl.reshape(-1))
            src = torch.empty(sl.numel(), dtype=torch.uint8, device=dev)
            src.copy_(stage[:sl.numel()], non_blocking=True)
            ring.release(dev)
        stage_buf = ring.acquire(wsb.numel())
        with torch.cuda.device(dev):
            rc = lib.vqa_qwen_preprocess_video_aa(_ptr(src), k, done, n_frames, hw[0], hw[1], rh, rw, ip(fh), fp(wh), th, ip(fv), fp(wv), tv,
                                                  patch, temporal_patch, merge, (C.c_float * 3)(*mean), (C.c_float * 3)(*std), _ptr(out),
                                                  _dtype_code(out_dtype), _ptr(wsb), wsb.numel(), stage_buf.data_ptr(), _stream_ptr(dev))
        ring.release(dev)
        _check(rc, None, "vqa_qwen_preprocess_video_aa")
        done += k
    assert done == n_frames, f"{done} frames given, n_frames = {n_frames}"
    return out, ((n_frames + temporal_patch - 1) // temporal_patch, rh // patch, rw // patch)


# ================================================================================================ Qwen2.5-VL
def convert_qwen_state_dict(sd: Dict[str, torch.Tensor], cfg, device) -> Dict[str, torch.Tensor]:
    """HF `Qwen2_5_VLForConditionalGeneration` names -> the engine's fused bf16 layout:
      * vision qkv / proj: the HF tensors as they are ([3*H*hd, Dv] rows ordered (q|k|v, head, dim); [Dv, H*hd]). The qkv GEMM's epilogue
        scatters each 80-wide head into the 128-wide slots of the packed activation [L, 3*H*128] the attention kernel reads (pad columns
        zeroed once per forward), the attention kernel writes compact heads [L, H*hd];
      * vision gate|up rows concatenated with the MLP width zero-padded to a multiple of 128; down-projection columns padded;
      * language-model q|k|v rows concatenated (+ biases), gate|up rows concatenated;
      * with cfg.tie_word_embeddings, `llm.lm_head` is the same device tensor as `llm.embed`."""
    out: Dict[str, torch.Tensor] = {}

    def put(name, t):
        out[name] = t.detach().to(device=device, dtype=torch.bfloat16).contiguous()

    v = "model.visual."
    Dv, H, hd = cfg.vit_hidden, cfg.vit_heads, cfg.vit_head_dim
    mp = cfg.vit_mlp_padded
    put("vis.patch_embed", sd[v + "patch_embed.proj.weight"].reshape(Dv, -1))
    for l in range(cfg.vit_depth):
        p, q = v + f"blocks.{l}.", f"vis.{l}."
        put(q + "norm1", sd[p + "norm1.weight"]); put(q + "norm2", sd[p + "norm2.weight"])
        # HF's fused qkv rows are already ordered (q|k|v, head, dim) and proj's columns (head, dim): bound as they are, at the native head width
        put(q + "qkv.weight", sd[p + "attn.qkv.weight"]); put(q + "qkv.bias", sd[p + "attn.qkv.bias"])
        put(q + "proj.weight", sd[p + "attn.proj.weight"]); put(q + "proj.bias", sd[p + "attn.proj.bias"])
        gu = torch.zeros(2 * mp, Dv); gb = torch.zeros(2 * mp)
        gu[: cfg.vit_mlp] = sd[p + "mlp.gate_proj.weight"].float(); gu[mp: mp + cfg.vit_mlp] = sd[p + "mlp.up_proj.weight"].float()
        gb[: cfg.vit_mlp] = sd[p + "mlp.gate_proj.bias"].float(); gb[mp: mp + cfg.vit_mlp] = sd[p + "mlp.up_proj.bias"].float()
        put(q + "gate_up.weight", gu); put(q + "gate_up.bias", gb)
        dw = torch.zeros(Dv, mp); dw[:, : cfg.vit_mlp] = sd[p + "mlp.down_proj.weight"].float()
        put(q + "down.weight", dw); put(q + "down.bias", sd[p + "mlp.down_proj.bias"])
    put("vis.merger.ln_q", sd[v + "merger.ln_q.weight"])
    put("vis.merger.fc1.weight", sd[v + "merger.mlp.0.weight"]); put("vis.merger.fc1.bias", sd[v + "merger.mlp.0.bias"])
    put("vis.merger.fc2.weight", sd[v + "merger.mlp.2.weight"]); put("vis.merger.fc2.bias", sd[v + "merger.mlp.2.bias"])
    t = "model.language_model."
    put("llm.embed", sd[t + "embed_tokens.weight"])
    put("llm.norm", sd[t + "norm.weight"])
    if getattr(cfg, "tie_word_embeddings", False):
        # one device tensor for both bindings; a tied checkpoint that also stores lm_head.weight loses it to the embedding, as HF's
        # tie_weights() does
        out["llm.lm_head"] = out["llm.embed"]
    elif "lm_head.weight" in sd:
        put("llm.lm_head", sd["lm_head.weight"])
    else:
        raise KeyError("the checkpoint has no lm_head.weight and its config does not tie the embeddings (tie_word_embeddings false): "
                       "an untied Qwen2.5-VL checkpoint must carry its lm_head")
    for l in range(cfg.layers):
        p, q = t + f"layers.{l}.", f"llm.{l}."
        put(q + "ln1", sd[p + "input_layernorm.weight"]); put(q + "ln2", sd[p + "post_attention_layernorm.weight"])
        put(q + "qkv.weight", torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], dim=0))
        put(q + "qkv.bias", torch.cat([sd[p + f"self_attn.{n}_proj.bias"] for n in "qkv"], dim=0))
        put(q + "o.weight", sd[p + "self_attn.o_proj.weight"])
        put(q + "gate_up.weight", torch.cat([sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]], dim=0))
        put(q + "down.weight", sd[p + "mlp.down_proj.weight"])
    return out


class QwenVLEngine(_Engine):
    """Qwen2.5-VL VQAScore engine: P(answer token | image, prompt) for a whole batch of prompts in one prefill."""

    def __init__(self, cfg, device="cuda:0", emulate_bf16_rounding: bool = True):
        from . import qwen_host
        if cfg.head_dim != 128:
            raise ValueError("the language-model attention kernel is specialised for head_dim == 128")
        mask = 0
        for l in cfg.fullatt_block_indexes:
            mask |= 1 << l
        c = _lib.VqaQwen25VLConfig(vit_depth=cfg.vit_depth, vit_hidden=cfg.vit_hidden, vit_heads=cfg.vit_heads,
                                   vit_head_dim=cfg.vit_head_dim, vit_mlp=cfg.vit_mlp, patch_dim=cfg.patch_dim,
                                   spatial_merge=cfg.spatial_merge_size, out_hidden=cfg.out_hidden, fullatt_mask=mask,
                                   hidden=cfg.hidden, layers=cfg.layers, heads=cfg.heads, kv_heads=cfg.kv_heads, mlp=cfg.mlp,
                                   vocab=cfg.vocab, rms_eps=cfg.rms_eps, emulate_bf16_rounding=1 if emulate_bf16_rounding else 0)
        super().__init__(cfg, device, "vqa_create_qwen25vl", c)
        t_inv, t_axis, v_inv, v_axis = qwen_host.rope_tables(cfg.head_dim, cfg.rope_theta, cfg.mrope_section, cfg.vit_head_dim)
        fp = lambda t: t.numpy().ctypes.data_as(C.POINTER(C.c_float))
        ip = lambda t: t.numpy().ctypes.data_as(C.POINTER(C.c_int32))
        self._run("vqa_qwen25vl_set_rope", fp(t_inv), ip(t_axis), t_inv.numel(), fp(v_inv), ip(v_axis), v_inv.numel())
        self._vision_cache: "collections.OrderedDict[tuple, dict]" = collections.OrderedDict()   # per-batch index sets, LRU-bounded

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        self.bind_engine_tensors(convert_qwen_state_dict(sd, self.cfg, self.device))

    def vision_indices(self, grid_thw):
        """Window order, rotary positions and cumulative lengths for a list of (t, h, w) grids, keyed by their vqa_qwen25vl_prompts field
        names; cached per grid tuple."""
        from . import qwen_host
        key = tuple(tuple(int(x) for x in g) for g in grid_thw)
        hit = self._vision_cache.get(key)
        if hit is not None:
            self._vision_cache.move_to_end(key)
            return hit
        cfg, dev = self.cfg, self.device
        merge, unit = cfg.spatial_merge_size, cfg.spatial_merge_size ** 2
        widx, cu_win, cu_frames = qwen_host.vision_window_index(key, merge, cfg.window_size, cfg.patch_size)
        pos = qwen_host.vision_rot_pos_ids(key, merge)                                   # [L, 2] processor order
        L = pos.shape[0]
        pos_win = pos.reshape(L // unit, unit, 2)[widx].reshape(L, 2)                    # window order (:478-484)
        i32 = lambda t: t.to(torch.int32).contiguous().to(dev)
        out = dict(window_index=i32(widx), reverse_index=i32(torch.argsort(widx)), vis_pos_hw=i32(pos_win.t()),
                   cu_window=i32(cu_win), cu_frames=i32(cu_frames), n_windows=cu_win.numel() - 1, n_frames=cu_frames.numel() - 1,
                   max_window_len=int((cu_win[1:] - cu_win[:-1]).max()), max_frame_len=int((cu_frames[1:] - cu_frames[:-1]).max()),
                   n_patches=L)
        self._vision_cache[key] = out
        while len(self._vision_cache) > 64:          # a dataset with varied image sizes makes a new key per batch: keep the device memory bounded
            self._vision_cache.popitem(last=False)
        return out

    def _prompts(self, pixel_patches, vi, input_ids, seq_lens, feat_index, position_ids, batch: int, seq_len: int = 0):
        """The vqa_qwen25vl_prompts of one prefill (packed rows: no seq_lens, seq_len 0). It holds raw device addresses: the caller keeps
        the tensors alive until the call that reads it has returned."""
        vision = {k: (_ptr(v) if torch.is_tensor(v) else v) for k, v in vi.items()}
        return _lib.VqaQwen25VLPrompts(pixel_patches=_ptr(pixel_patches), pixel_dtype=_dtype_code(pixel_patches.dtype), input_ids=_ptr(input_ids),
                                       seq_lens=_ptr(seq_lens), feat_index=_ptr(feat_index), position_ids=_ptr(position_ids), batch=batch,
                                       seq_len=seq_len, **vision)

    def _check_inputs(self, pixel_patches: torch.Tensor, vi: dict, *int32_tensors):
        assert pixel_patches.is_cuda and pixel_patches.is_contiguous() and pixel_patches.shape == (vi["n_patches"], self.cfg.patch_dim)
        assert pixel_patches.dtype in (torch.float32, torch.bfloat16)
        for t in int32_tensors:
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()

    def _indices(self, build, prompts, grid_thw, image_of_sample, second_per_grid_ts, **kw) -> dict:
        """qwen_host.build_batch_indices or build_packed_indices (`build`) of id-list prompts over grid_thw; image_of_sample None: prompt b
        shows item b."""
        cfg = self.cfg
        img = list(image_of_sample) if image_of_sample is not None else list(range(len(prompts)))
        return build([list(map(int, p)) for p in prompts], [tuple(map(int, g)) for g in grid_thw], img, cfg.image_token_id,
                     cfg.spatial_merge_size, cfg.tokens_per_second, video_token_id=cfg.video_token_id, second_per_grid_ts=second_per_grid_ts,
                     **kw)

    def _score(self, prompts, packed, rows: int, answer_ids, temperature, repetition_penalty, out, logp):
        """One vqa_qwen25vl_score call over `rows` language-model rows: padded rows (packed None) or packed rows."""
        ws = self._grow("_workspace", int(self.lib.vqa_qwen25vl_workspace_bytes(self._h, prompts.batch, rows, prompts.n_patches)), self._graphs)
        self._run("vqa_qwen25vl_score", C.byref(prompts), None if packed is None else C.byref(packed), _ptr(answer_ids), float(temperature),
                  float(repetition_penalty), _ptr(out), _ptr(logp), _ptr(ws), ws.numel(), _stream_ptr(self.device))
        self._last_call = (prompts.batch, rows, prompts.n_patches)     # what topk_last() needs to find the final hidden states again

    def score_tensors(self, pixel_patches: torch.Tensor, grid_thw, input_ids: torch.Tensor, seq_lens: torch.Tensor,
                      feat_index: torch.Tensor, position_ids: torch.Tensor, answer_ids: torch.Tensor, temperature: float = 1.0,
                      out: Optional[torch.Tensor] = None, return_logprobs: bool = False, repetition_penalty: float = 1.0):
        """pixel_patches [sum P, patch_dim] fp32/bf16 cuda; grid_thw list of (t,h,w); the int32 cuda tensors come from
        qwen_host.build_batch_indices. repetition_penalty != 1 applies HF's RepetitionPenaltyLogitsProcessor over each sample's
        prompt ids before the softmax (what `generate(..., output_scores=True)` returns when the checkpoint's
        generation_config.json carries one, SURVEY F8). Returns probabilities [B] fp32 on the device."""
        dev = self.device
        vi = self.vision_indices(grid_thw)
        self._check_inputs(pixel_patches, vi, input_ids, seq_lens, feat_index, position_ids, answer_ids)
        B, S = input_ids.shape
        if out is None:
            out = torch.empty(B, dtype=torch.float32, device=dev)
        logp = torch.empty(B, dtype=torch.float32, device=dev) if return_logprobs else None
        prompts = self._prompts(pixel_patches, vi, input_ids, seq_lens, feat_index, position_ids, B, S)
        self._score(prompts, None, B * S, answer_ids, temperature, repetition_penalty, out, logp)
        return (out, logp) if return_logprobs else out

    def topk_last(self, k: int = 5, temperature: float = 1.0, repetition_penalty: float = 1.0):
        """Top-k next tokens (ids [B, k] int32, probabilities [B, k] fp32, most probable first) of the prompts of the LAST score_tensors /
        score_prompts call, under the same logit processing as the scores -- the reference's forward_with_trace output
        (qwen2vl_model.py:439-447). Trace mode only: materialises the last position's [B, vocab] logits in the workspace."""
        if getattr(self, "_last_call", None) is None:
            raise RuntimeError("topk_last() follows a scoring call")
        B, rows, n_patches = self._last_call
        dev = self.device
        ids = torch.empty(B, k, dtype=torch.int32, device=dev)
        probs = torch.empty(B, k, dtype=torch.float32, device=dev)
        self._run("vqa_qwen25vl_topk", B, rows, n_patches, k, float(temperature), float(repetition_penalty), _ptr(ids), _ptr(probs),
                  _ptr(self._workspace), self._workspace.numel(), _stream_ptr(dev))
        return ids, probs

    def debug_tensors(self, batch: int, seq_len: int, n_patches: int) -> Dict[str, torch.Tensor]:
        """Views into the workspace of the LAST call with these sizes (synchronise first). Parity investigations only."""
        off = (C.c_size_t * 4)()
        self._run("vqa_qwen25vl_debug_layout", batch, batch * seq_len, n_patches, off, 4)
        cfg, ws = self.cfg, self._workspace
        unit = cfg.spatial_merge_size ** 2

        def view(o, rows, cols):
            return ws[o:o + rows * cols * 2].view(torch.bfloat16).view(rows, cols)
        return dict(last_hidden=view(off[0], batch, cfg.hidden), vision_feats=view(off[1], n_patches // unit, cfg.out_hidden))

    def score_packed(self, pixel_patches: torch.Tensor, grid_thw, packed: Dict[str, torch.Tensor], answer_ids: torch.Tensor,
                     temperature: float = 1.0, repetition_penalty: float = 1.0, out: Optional[torch.Tensor] = None):
        """One prefill over PACKED rows (qwen_host.build_packed_indices, tensors already on the device): prompts over the same image share
        the K/V of their [chat prefix + vision tokens]."""
        dev = self.device
        vi = self.vision_indices(grid_thw)
        self._check_inputs(pixel_patches, vi)
        B, R = int(answer_ids.numel()), int(packed["total_rows"])
        if out is None:
            out = torch.empty(B, dtype=torch.float32, device=dev)
        prompts = self._prompts(pixel_patches, vi, packed["input_ids"], None, packed["feat_index"], packed["position_ids"], B)
        pk = _lib.VqaQwen25VLPacked(total_rows=R, n_seq=int(packed["n_seq"]), max_seq_len=int(packed["max_seq_len"]),
                                    max_prompt_len=int(packed["max_prompt_len"]),
                                    **{k: _ptr(packed[k]) for k in ("cu_seqlens", "kv_prefix", "pair_row", "pair_seq")})
        self._score(prompts, pk, R, answer_ids, temperature, repetition_penalty, out, None)
        return out

    def score_prompts(self, pixel_patches, grid_thw, prompts, answer_ids, image_of_sample=None, temperature: float = 1.0,
                      repetition_penalty: float = 1.0, second_per_grid_ts=None, share_prefix: Optional[bool] = None):
        """Convenience: prompts = list of 1-D id lists (each with one image- or video-token run). Host index logic + one engine
        call. Videos are grids with t > 1 whose prompt run uses cfg.video_token_id (second_per_grid_ts = temporal_patch / fps).
        share_prefix: None = automatically when at least two prompts start with the same [chat prefix + vision run] over the same image
        (the M x N scoring API repeats every image N times, reference score.py:104-106); their prefix then runs through the language
        model once (KV-prefix sharing, exact under causal attention). The shared part is cut to whole key tiles of the attention kernel
        (ATTN_KEY_TILE rows), so a shared prefill is bit-identical to the unshared one; a prefix shorter than one tile is not shared."""
        from . import qwen_host
        dev = self.device
        ans = torch.as_tensor(list(map(int, answer_ids)), dtype=torch.int32).to(dev)
        if share_prefix is None or share_prefix:
            pk = self._indices(qwen_host.build_packed_indices, prompts, grid_thw, image_of_sample, second_per_grid_ts, align=ATTN_KEY_TILE)
            if pk["n_shared"] > 0 or share_prefix:
                d = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in pk.items()}
                return self.score_packed(pixel_patches.to(dev), grid_thw, d, ans, temperature, repetition_penalty)
        idx = self._indices(qwen_host.build_batch_indices, prompts, grid_thw, image_of_sample, second_per_grid_ts)
        d = {k: v.to(dev) for k, v in idx.items()}
        return self.score_tensors(pixel_patches.to(dev), grid_thw, d["input_ids"], d["seq_lens"], d["feat_index"], d["position_ids"],
                                  ans, temperature, repetition_penalty=repetition_penalty)

    # ------------------------------------------------------------------------------------------ greedy generation
    def score_workspace_bytes(self, batch: int, seq_len: int, n_patches: int) -> int:
        """Device bytes of one padded scoring prefill (vqa_qwen25vl_workspace_bytes), the most score_prompts needs; 0 for invalid sizes."""
        return int(self.lib.vqa_qwen25vl_workspace_bytes(self._h, batch, batch * seq_len, n_patches))

    def generate_workspace_bytes(self, batch: int, seq_len: int, n_patches: int, max_new_tokens: int) -> int:
        """Device bytes of one generation or scored rollout (vqa_qwen25vl_generate_workspace_bytes); 0 for invalid sizes."""
        return int(self.lib.vqa_qwen25vl_generate_workspace_bytes(self._h, batch, seq_len, n_patches, max_new_tokens))

    def generate_begin(self, pixel_patches, grid_thw, prompts, max_new_tokens: int, eos_ids: Sequence[int], image_of_sample=None,
                       repetition_penalty: float = 1.0, second_per_grid_ts=None, score: Optional[dict] = None,
                       sample: Optional[dict] = None) -> dict:
        """The prefill of a greedy generation (vqa_qwen25vl_generate_prefill): vision tower, padded prompt prefill into the K/V cache, first
        token. Returns the generation state that generate_step() advances: device tensors `tokens` [B, max_new_tokens] (-1 after a prompt's
        last token), `lengths` [B] and `all_done` [1], all owned by the state of this call shape.
        score = dict(answer_ids=[ids per prompt], temperature=T, top_k=k) makes it a scored rollout (an answer score in the generation): the
        state also holds `logp` [B, max_new_tokens, n_max] (NaN where nothing was written) and, with k > 0, `topk_ids` / `topk_probs`
        [B, max_new_tokens, k].
        sample = dict(seeds=[one int per prompt], temperature=T, top_k=k, top_p=p) makes it a sampled generation
        (vqa_qwen25vl_generate_*_sampled). The seeds go to a device buffer of the state before each prefill, so one captured step graph
        serves every seed."""
        from . import qwen_host
        cfg, dev = self.cfg, self.device
        B = len(prompts)
        idx = self._indices(qwen_host.build_batch_indices, prompts, grid_thw, image_of_sample, second_per_grid_ts)
        first = qwen_host.first_generated_positions(idx)
        vi = self.vision_indices(grid_thw)
        pixel_patches = pixel_patches.to(dev).contiguous()
        self._check_inputs(pixel_patches, vi)
        S, max_new = int(idx["input_ids"].shape[1]), int(max_new_tokens)
        eos = [int(e) for e in eos_ids]
        need = int(self.lib.vqa_qwen25vl_generate_workspace_bytes(self._h, B, S, vi["n_patches"], max_new))
        if need == 0:
            raise ValueError(f"bad generation size: batch {B}, prompt length {S}, max_new_tokens {max_new}")
        key = (B, S, vi["n_patches"], max_new, float(repetition_penalty), len(eos))
        if score is not None:
            answers = [[int(t) for t in a] for a in score["answer_ids"]]
            if len(answers) != B or not all(answers):
                raise ValueError("rollout scoring needs one non-empty answer id list per prompt")
            n_max, temp, top_k = max(len(a) for a in answers), float(score.get("temperature", 1.0)), int(score.get("top_k", 0))
            key += ("rollout", n_max, temp, top_k)
        if sample is not None:
            seeds = [int(x) for x in sample["seeds"]]
            if len(seeds) != B or not all(0 <= x < 1 << 64 for x in seeds):
                raise ValueError("sampling needs one seed in [0, 2^64) per prompt")
            smp_t, smp_k, smp_p = float(sample["temperature"]), int(sample["top_k"]), float(sample["top_p"])
            key += ("sample", smp_t, smp_k, smp_p)

        def make() -> dict:
            i32 = lambda *shape: torch.empty(*shape, dtype=torch.int32, device=dev)
            st = dict(B=B, S=S, n_patches=vi["n_patches"], max_new=max_new, seq_lens=i32(B), first=i32(B), eos=i32(max(len(eos), 1)),
                      tokens=i32(B, max_new), lengths=i32(B), all_done=i32(1), graph=None, score=None, sample=None)
            # the vqa_qwen25vl_generation every call of this state passes, built once: its pointers are the state's own tensors
            st["gen"] = _lib.VqaQwen25VLGeneration(
                seq_lens=_ptr(st["seq_lens"]), first_position=_ptr(st["first"]), eos_ids=_ptr(st["eos"]), n_eos=len(eos), max_new_tokens=max_new,
                repetition_penalty=float(repetition_penalty), out_tokens=_ptr(st["tokens"]), out_lengths=_ptr(st["lengths"]),
                all_done=_ptr(st["all_done"]))
            if score is not None:
                sc = st["score"] = dict(n_max=n_max, temperature=temp, top_k=top_k, answer_ids=i32(B, n_max), counts=i32(B),
                                        logp=torch.empty(B, max_new, n_max, dtype=torch.float32, device=dev),
                                        topk_ids=i32(B, max_new, top_k) if top_k > 0 else None,
                                        topk_probs=torch.empty(B, max_new, top_k, dtype=torch.float32, device=dev) if top_k > 0 else None)
                sc["struct"] = _lib.VqaQwen25VLAnswerScore(answer_ids=_ptr(sc["answer_ids"]), answer_counts=_ptr(sc["counts"]), n_max=n_max,
                                                           temperature=temp, top_k=top_k, out_logp=_ptr(sc["logp"]),
                                                           out_topk_ids=_ptr(sc["topk_ids"]), out_topk_probs=_ptr(sc["topk_probs"]))
                st["gen"].score = C.pointer(sc["struct"])
            if sample is not None:
                sm = st["sample"] = dict(seeds=torch.empty(B, dtype=torch.int64, device=dev))
                sm["struct"] = _lib.VqaQwen25VLSampling(seeds=_ptr(sm["seeds"]), temperature=smp_t, top_k=smp_k, top_p=smp_p)
            return st
        st = self._gen_state(key, need, make)
        st["seq_lens"].copy_(idx["seq_lens"], non_blocking=True)
        st["first"].copy_(first, non_blocking=True)
        if eos:
            st["eos"].copy_(torch.as_tensor(eos, dtype=torch.int32), non_blocking=True)
        sc = st["score"]
        if sc is not None:
            ans = torch.full((B, sc["n_max"]), -1, dtype=torch.int32)
            for b, a in enumerate(answers):
                ans[b, :len(a)] = torch.as_tensor(a, dtype=torch.int32)
            sc["answer_ids"].copy_(ans, non_blocking=True)
            sc["counts"].copy_(torch.as_tensor([len(a) for a in answers], dtype=torch.int32), non_blocking=True)
            sc["logp"].fill_(float("nan"))
            if sc["top_k"] > 0:
                sc["topk_ids"].fill_(-1)
                sc["topk_probs"].fill_(float("nan"))
        if st["sample"] is not None:
            # uint64 seeds in an int64 buffer: the same 8 bytes
            st["sample"]["seeds"].copy_(torch.tensor([x - (1 << 64) if x >= 1 << 63 else x for x in seeds], dtype=torch.int64), non_blocking=True)
        d = {k: v.to(dev) for k, v in idx.items()}

        def prefill():
            prompts = self._prompts(pixel_patches, vi, d["input_ids"], st["seq_lens"], d["feat_index"], d["position_ids"], B, S)
            ws = self._gen_workspace
            if st["sample"] is None:
                self._run("vqa_qwen25vl_generate_prefill", C.byref(prompts), C.byref(st["gen"]), _ptr(ws), ws.numel(), _stream_ptr(dev))
            else:
                self._run("vqa_qwen25vl_generate_prefill_sampled", C.byref(prompts), C.byref(st["gen"]), C.byref(st["sample"]["struct"]),
                          _ptr(ws), ws.numel(), _stream_ptr(dev))
        st["prefill"] = prefill          # relaunches this prefill on the same device inputs (no host work)
        prefill()
        return st

    def generate_step(self, st: dict):
        """One decode step of the generation `st` (vqa_qwen25vl_generate_step, or _step_sampled), launched directly."""
        ws = self._gen_workspace
        if st["sample"] is None:
            self._run("vqa_qwen25vl_generate_step", C.byref(st["gen"]), st["B"], st["S"], st["n_patches"], _ptr(ws), ws.numel(),
                      _stream_ptr(self.device))
        else:
            self._run("vqa_qwen25vl_generate_step_sampled", C.byref(st["gen"]), C.byref(st["sample"]["struct"]), st["B"], st["S"],
                      st["n_patches"], _ptr(ws), ws.numel(), _stream_ptr(self.device))

    def generate_prompts(self, pixel_patches, grid_thw, prompts, max_new_tokens: int, eos_ids: Sequence[int], image_of_sample=None,
                         repetition_penalty: float = 1.0, second_per_grid_ts=None, use_graph: bool = True, check_every: int = 16):
        """Greedy generation (HF generate(do_sample=False)) for a batch of prompts (1-D id lists, one image- or video-token run each, as in
        score_prompts): one prefill, then decode steps replayed from a CUDA graph captured once per (batch, prompt length, max_new_tokens).
        The host reads the all-finished flag through pinned memory every `check_every` steps and never synchronises in between.
        Returns each prompt's generated ids, the EOS id included when one ended it."""
        st = self.generate_begin(pixel_patches, grid_thw, prompts, max_new_tokens, eos_ids, image_of_sample, repetition_penalty,
                                 second_per_grid_ts)
        return self._decode_loop(st, use_graph, check_every)[0]

    def rollout_scores(self, pixel_patches, grid_thw, prompts, answer_ids, max_new_tokens: int, eos_ids: Sequence[int],
                       temperature: float = 1.0, repetition_penalty: float = 1.0, top_k: int = 0, image_of_sample=None,
                       second_per_grid_ts=None, use_graph: bool = True, check_every: int = 16) -> dict:
        """A greedy rollout scored at every step: generate_prompts' decode loop (same tokens, bit for bit) plus, at each step s of each
        prompt b, log softmax(processed scores / temperature) at each of the prompt's answer ids (answer_ids: one id list per prompt) -- the
        per-step probabilities the reference's forward / forward_with_trace read from generate(output_scores=True) (qwen2vl_model.py:160-167).
        With top_k > 0 (<= 8) also the step's top_k ids and probabilities. The temperature never changes a token.
        Returns CPU tensors: dict(tokens=[ids per prompt], lengths [B], logp [B, max_new_tokens, n_max] (NaN beyond a prompt's length or its
        answer), topk_ids / topk_probs [B, max_new_tokens, top_k] or None)."""
        st = self.generate_begin(pixel_patches, grid_thw, prompts, max_new_tokens, eos_ids, image_of_sample, repetition_penalty,
                                 second_per_grid_ts, score=dict(answer_ids=answer_ids, temperature=temperature, top_k=top_k))
        tokens, lengths = self._decode_loop(st, use_graph, check_every)
        sc = st["score"]
        cpu = lambda t: None if t is None else t.cpu()
        return dict(tokens=tokens, lengths=lengths, logp=cpu(sc["logp"]), topk_ids=cpu(sc["topk_ids"]), topk_probs=cpu(sc["topk_probs"]))

    def sample_prompts(self, pixel_patches, grid_thw, prompts, max_new_tokens: int, eos_ids: Sequence[int], seeds: Sequence[int],
                       temperature: float, top_k: int, top_p: float, image_of_sample=None, repetition_penalty: float = 1.0,
                       second_per_grid_ts=None, use_graph: bool = True, check_every: int = 16):
        """Sampled generation (HF generate(do_sample=True) with the repetition penalty, temperature, top_k and top_p warpers) for a batch
        of prompts, as generate_prompts runs greedy generation: one prefill, then decode steps replayed from a CUDA graph captured once per
        (call shape, temperature, top_k, top_p). Prompt b's tokens depend on seeds[b] (an integer in [0, 2^64)), its prompt and the sizes,
        not on its batch position. Returns each prompt's generated ids, the EOS id included when one ended it."""
        st = self.generate_begin(pixel_patches, grid_thw, prompts, max_new_tokens, eos_ids, image_of_sample, repetition_penalty,
                                 second_per_grid_ts, sample=dict(seeds=seeds, temperature=temperature, top_k=top_k, top_p=top_p))
        return self._decode_loop(st, use_graph, check_every)[0]

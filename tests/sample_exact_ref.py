"""Exact host restatement of sample_select_kernel's decision for the tests, from the per-id terms vqa_debug_sample_terms reads back.

The kernel's arithmetic is deterministic by design: scores are compared through order-preserving integer keys, the top-p cut sums
integer masses of 2^-40 units, and the Gumbel uniforms are Philox4x32-10 keyed by (seed, step, id). Only expf, logf and log1pf cannot
be restated on the host, so the restatement takes the fp32 scores, the uint64 masses and the fp32 perturbed values from the device and
recomputes everything else in integers: top-k as every id whose score is >= the k-th largest, top-p as the first key at which the
ascending running sum of masses exceeds tg = floor(fp32(1 - top_p) * total) (clamped to total - 1), with the lowest rest // q ids of
that key's group going, and the token as the arg-max of the perturbed values over the kept ids, ties to the lowest id. Sorting and
cumulative sums stand in for the kernel's histogram passes. The bookkeeping after the draw is SelectState's (test_gpu_decode_kernels)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import torch

import sample_ref as sr
from test_gpu_decode_kernels import SelectState

TWO40 = np.float32(2.0 ** 40)
SELECT_THREADS = 1024             # qwen_decode.cuh: threads of sample_select_kernel; its tie-group pass gives each a contiguous id range
RADIX_SHIFTS = (21, 10, 0)        # the three radix digits (11, 11, 10 bits) of a 32-bit key, highest first

# the deliberate errors the GPU test's fixtures must each expose (see select_row / perturbed_f64)
MUTATIONS = ("float_top_p", "topk_no_ties", "drop_plus_one", "split_from_top", "philox_id_step_swapped", "lanes_reversed",
             "argmax_ties_high")


def order_key(x) -> np.ndarray:
    """fp32 -> uint32 whose unsigned order is the float order (qwen_decode.cuh order_key; -0 must have been merged into +0)."""
    u = np.asarray(x, np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def mass_of_exp(ex) -> np.ndarray:
    """The kernel's quantisation of an fp32 ex = expf(x - max) to 2^-40 units: (uint64)(fp32(ex * 2^40 + 0.5)). The product is exact
    (a power-of-two scale of a value <= 1), so a fused multiply-add and a multiply then add round alike."""
    ex = np.asarray(ex, np.float32)
    return (ex * TWO40 + np.float32(0.5)).astype(np.float32).astype(np.uint64)


def threshold(top_p: float, mutation: Optional[str] = None) -> np.float32:
    """HF's top-p threshold: fp32(1 - top_p) of the caller's double. The float_top_p mutation rounds top_p to fp32 first."""
    if mutation == "float_top_p":
        return np.float32(1.0 - float(np.float32(top_p)))
    return np.float32(1.0 - float(top_p))


def cut_target(thr: np.float32, total: int) -> int:
    """tg = floor(double(thr) * double(total)) as the device forms it (cvt.rn.f64.u64, one double product, truncation), clamped to
    total - 1 so the last unit is always past it."""
    return min(int(float(thr) * float(total)), total - 1)


def resolved_pass(keys: np.ndarray, key: int) -> int:
    """The radix pass (0, 1, 2) after which `key` is the only key left among `keys` sharing its digits so far: the pass that decides."""
    for p, s in enumerate(RADIX_SHIFTS):
        same = keys[(keys >> np.uint32(s)) == np.uint32(key >> s)]
        if np.all(same == np.uint32(key)):
            return p
    raise AssertionError("unreachable: pass 2 compares whole keys")


@dataclass
class Selection:
    kept: np.ndarray                  # bool [V]
    token: int
    key_k: int = 0                    # top-k threshold key (0 = off)
    k_pass: Optional[int] = None      # radix pass that decided key_k
    total: int = 0                    # integer mass of the ids top-k kept
    tg: int = 0
    clamped: bool = False             # tg was clamped to total - 1
    key_p: int = 0                    # top-p cut key (0 = off)
    p_pass: Optional[int] = None
    drop: int = 0                     # ids of the cut group that go (lowest ids first)
    group: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))      # ids of the cut group, ascending
    tg_equals_cumsum: bool = False    # tg is exactly one of the member-level ascending running sums
    zero_mass_kept: int = 0           # ids with mass 0 that top-k passed (they add nothing to the running sum)


def select_row(x: np.ndarray, mass: np.ndarray, v: np.ndarray, top_k: int, top_p: float, mutation: Optional[str] = None) -> Selection:
    """The kernel's kept set and token for one row from its fp32 scores x, uint64 masses and fp32 perturbed values v (all [V]; v may
    be fp64 values for a mutated Philox stream)."""
    V = x.shape[0]
    keys = order_key(x).astype(np.int64)
    ids = np.arange(V)
    sel = Selection(kept=np.ones(V, bool), token=-1)
    if 0 < top_k < V:
        sel.key_k = int(np.sort(keys)[::-1][top_k - 1])
        sel.k_pass = resolved_pass(keys.astype(np.uint32), sel.key_k)
        if mutation == "topk_no_ties":          # exactly k ids: the k largest, lower ids first among equals
            order = np.lexsort((ids, -keys))
            sel.kept[:] = False
            sel.kept[order[:top_k]] = True
        else:
            sel.kept = keys >= sel.key_k
    m = np.asarray(mass, np.uint64)         # V < 2^23 masses of <= 2^40: every sum is exact in uint64
    if top_p < 1.0:
        cand = np.nonzero(sel.kept)[0]
        total = int(m[cand].sum())
        sel.total = total
        thr = threshold(top_p, mutation)
        sel.clamped = int(float(thr) * float(total)) >= total
        sel.tg = tg = cut_target(thr, total)
        sel.zero_mass_kept = int(np.count_nonzero(m[cand] == 0))
        # ascending (key, id) order of the candidates; running sums of whole key groups find the cut key
        order = cand[np.lexsort((cand, keys[cand]))]
        ok = keys[order]
        ends = np.nonzero(np.r_[ok[1:] != ok[:-1], True])[0]            # last position of each key group
        csum = np.cumsum(m[order])
        gsum = csum[ends]
        g = int(np.argmax(gsum > np.uint64(tg)))                          # exists: gsum[-1] = total > tg
        below = int(gsum[g - 1]) if g else 0
        sel.key_p = int(ok[ends[g]])
        sel.p_pass = resolved_pass(keys[cand].astype(np.uint32), sel.key_p)
        sel.tg_equals_cumsum = bool(np.any(csum == np.uint64(tg)))
        group = order[ok == sel.key_p]                                   # ascending ids
        q = int(m[group[0]])
        drop = (tg - below) // q
        if mutation == "drop_plus_one":
            drop = min(drop + 1, len(group))
        sel.drop, sel.group = drop, group
        sel.kept[order[ok < sel.key_p]] = False
        if drop:
            gone = group[-drop:] if mutation == "split_from_top" else group[:drop]
            sel.kept[gone] = False
    kept_ids = np.nonzero(sel.kept)[0]
    if not len(kept_ids):                   # only a mutation can empty the kept set
        return sel
    vk = np.asarray(v)[kept_ids]
    assert not np.isnan(vk).any()
    best = np.nonzero(vk == vk.max())[0]
    sel.token = int(kept_ids[best[-1] if mutation == "argmax_ties_high" else best[0]])
    return sel


def pack_bits(kept: np.ndarray) -> np.ndarray:
    """bool [B, V] -> the kernel's bitmap words uint32 [B, ceil(V / 32)], bits past V zero."""
    B, V = kept.shape
    words = -(-V // 32)
    pad = np.zeros((B, words * 32), bool)
    pad[:, :V] = kept
    return (pad.reshape(B, words, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)


def philox_bits(seed: int, step: int, V: int, mutation: Optional[str] = None) -> np.ndarray:
    """uint32 [V]: lane n & 3 of Philox4x32-10 under key seed (low word first) at counter (n >> 2, step, 0, 0), via sample_ref's
    Philox. The philox_id_step_swapped mutation uses counter (step, n >> 2, 0, 0); lanes_reversed takes lane 3 - (n & 3)."""
    G = (V + 3) // 4
    ctr = np.zeros((G, 4), dtype=np.uint32)
    ctr[:, 0] = np.arange(G, dtype=np.uint32)
    ctr[:, 1] = step
    if mutation == "philox_id_step_swapped":
        ctr[:, [0, 1]] = ctr[:, [1, 0]]
    r = sr.philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    if mutation == "lanes_reversed":
        r = r[:, ::-1]
    return r.reshape(-1)[:V].copy()


def gumbel_e_f64(bits: np.ndarray) -> np.ndarray:
    """-log(u) in fp64 of u = ((bits >> 8) + 0.5) 2^-24 (exact in fp64); through log1p for u >= 1/2, as the kernel does."""
    m = (np.asarray(bits, np.uint32) >> np.uint32(8)).astype(np.float64)
    lo = m < 2.0 ** 23
    return np.where(lo, -np.log(np.where(lo, m + 0.5, 1.0) * 2.0 ** -24), -np.log1p(-(2.0 ** 24 - m - 0.5) * 2.0 ** -24))


def perturbed_f64(x: np.ndarray, mx: np.float32, bits: np.ndarray) -> np.ndarray:
    """fp64 value of the kernel's perturbed score from lane bits: fp32(x - max) - log(-log u)."""
    d = (np.asarray(x, np.float32) - np.float32(mx)).astype(np.float64)
    return d - np.log(gumbel_e_f64(bits))


def device_terms(logits: torch.Tensor, bitmap, penalty: float, seeds, temperature: float, lengths, top_k: int = 0, top_p: float = 1.0):
    """vqa_debug_sample_terms on bf16 logits [B, V] (any device; bitmap int32 [B, ceil(V / 32)] or None, seeds ints, lengths int32 [B])
    -> dict of numpy arrays: score, row_max, ex, mass, bits, e, v."""
    from t2v_metrics_b200 import _lib
    B, V = logits.shape
    dev = torch.device("cuda")
    lg = logits.to(dev).contiguous()
    bm = bitmap.to(dev).contiguous() if bitmap is not None else None
    sd = torch.tensor([int(s) - (1 << 64) if int(s) >= 1 << 63 else int(s) for s in seeds], dtype=torch.int64, device=dev)
    ln = torch.as_tensor(lengths, dtype=torch.int32).to(dev)
    out = dict(score=torch.empty(B, V, dtype=torch.float32, device=dev), row_max=torch.empty(B, dtype=torch.float32, device=dev),
               ex=torch.empty(B, V, dtype=torch.float32, device=dev), mass=torch.empty(B, V, dtype=torch.int64, device=dev),
               bits=torch.empty(B, V, dtype=torch.int32, device=dev), e=torch.empty(B, V, dtype=torch.float32, device=dev),
               v=torch.empty(B, V, dtype=torch.float32, device=dev))
    smp = _lib.VqaQwen25VLSampling(seeds=sd.data_ptr(), temperature=float(temperature), top_k=int(top_k), top_p=float(top_p))
    p = lambda t: None if t is None else t.data_ptr()
    rc = _lib.load().vqa_debug_sample_terms(p(lg), B, V, p(bm), float(penalty), p(ln), C.byref(smp), p(out["score"]), p(out["row_max"]),
                                            p(out["ex"]), p(out["mass"]), p(out["bits"]), p(out["e"]), p(out["v"]),
                                            torch.cuda.current_stream(dev).cuda_stream)
    if rc:
        raise RuntimeError(f"vqa_debug_sample_terms: status {rc}: {_lib.last_error(None)}")
    torch.cuda.synchronize()
    res = {k: t.cpu().numpy() for k, t in out.items()}
    res["mass"] = res["mass"].view(np.uint64)
    res["bits"] = res["bits"].view(np.uint32)
    return res


def expected_state(state: SelectState, tokens, eos_ids) -> SelectState:
    """SelectState's step with each unfinished row's token given (a one-hot row at it, no penalty), in place; returns state."""
    B, V = state.B, state.V
    onehot = torch.full((B, V), -1.0)
    onehot[torch.arange(B), torch.as_tensor([max(int(t), 0) for t in tokens])] = 1.0
    state.step_ref(onehot.bfloat16(), list(eos_ids), 1.0)
    return state

// Kernels of the CLIP-FlanT5 greedy decode loop: the decoder self-attention K/V cache append and the self-attention of one new row per
// sequence over that cache. Token selection and the per-step bookkeeping are qwen_decode.cuh's generate_init_kernel / greedy_select_kernel.
// Every step-dependent value (tokens generated so far, finished flags, next input ids) lives in device memory, so the launches of one
// decode step take the same arguments at every step and replay from one CUDA graph.
#pragma once
#include "ptx.cuh"
#include "elementwise.cuh"

namespace vqa {

// Decoder position of the step's input row: the start token sits at 0 and generated token t at t + 1, so the input of a sequence that
// has generated n tokens is at n. A sequence that finished by length (n == cap) is recomputed but never selected from again; the clamp
// keeps its rows inside the cache.
__device__ __forceinline__ int t5_decode_pos(const int* lengths, int b, int cap) { return min(lengths[b], cap - 1); }

// K/V cache of one decoder layer: K and V each [B, H, cap, 64] bf16. Source: the step's packed qkv [B, 3 * H * 64] (q | k | v); the row of
// sequence b goes to slot t5_decode_pos(b). One thread per (sequence, head, 16-byte chunk).
__global__ void t5_kv_cache_append_kernel(const __nv_bfloat16* __restrict__ qkv, int B, int H, const int* __restrict__ lengths,
                                          __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc, int cap) {
    pdl_launch_dependents();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * H * 8) return;
    const int c = idx & 7, h = (idx >> 3) % H, b = idx / (8 * H);
    const int slot = t5_decode_pos(lengths, b, cap);
    const size_t dst = (((size_t)b * H + h) * cap + slot) * 64 + c * 8;
    const __nv_bfloat16* src = qkv + (size_t)b * 3 * H * 64 + h * 64 + c * 8;
    *reinterpret_cast<uint4*>(kc + dst) = *reinterpret_cast<const uint4*>(src + H * 64);
    *reinterpret_cast<uint4*>(vc + dst) = *reinterpret_cast<const uint4*>(src + 2 * H * 64);
}

// Decoder self-attention of the one new row of each sequence over its cache: query at position t = t5_decode_pos(b), keys in slots 0..t,
// unidirectional relative buckets of (key - query), no scale. Row for row the arithmetic of t5_decoder_self_attn_kernel (attention.cuh):
// lanes hold pairs of dims, warp-sum dot products, optional bf16 rounding of the score before and after the bias, fp32 softmax, P rounded
// to bf16 before P.V, keys summed in order. q: the step's packed qkv [B, 3 * H * 64]; out [B, H * 64]. One warp per (sequence, head);
// the scores of the row live in shared memory (dynamic: warps per block * cap floats).
__global__ void t5_decode_self_attn_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ kc,
                                           const __nv_bfloat16* __restrict__ vc, int cap, const int* __restrict__ lengths,
                                           __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ rel_emb,
                                           const int* __restrict__ bucket_lut, int max_dist, int B, int H, int round_scores) {
    pdl_launch_dependents();
    extern __shared__ float t5_dec_sc[];
    const int widx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (widx >= B * H) return;
    const int lane = threadIdx.x & 31;
    float* sc = t5_dec_sc + (size_t)(threadIdx.x >> 5) * cap;
    const int h = widx % H, b = widx / H;
    const int tq = t5_decode_pos(lengths, b, cap);
    const float2 qv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(qkv + (size_t)b * 3 * H * 64 + h * 64 + 2 * lane));
    const size_t base = ((size_t)b * H + h) * cap * 64 + 2 * lane;
    float mx = -INFINITY;
    for (int tk = 0; tk <= tq; ++tk) {
        const float2 kv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kc + base + (size_t)tk * 64));
        float v = warp_sum(qv.x * kv.x + qv.y * kv.y);
        if (round_scores) v = bf16_round(v);
        int rel = tk - tq;
        rel = min(max(rel, -max_dist), max_dist);
        v += __bfloat162float(rel_emb[bucket_lut[rel + max_dist] * H + h]);
        if (round_scores) v = bf16_round(v);
        if (lane == 0) sc[tk] = v;
        mx = fmaxf(mx, v);
    }
    __syncwarp();
    float denom = 0.f;
    for (int tk = 0; tk <= tq; ++tk) denom += __expf(sc[tk] - mx);
    float ox = 0.f, oy = 0.f;
    for (int tk = 0; tk <= tq; ++tk) {
        const float2 vv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vc + base + (size_t)tk * 64));
        const float pw = bf16_round(__expf(sc[tk] - mx) / denom);   // attn_weights are cast back to bf16 before the PV matmul
        ox += pw * vv.x;
        oy += pw * vv.y;
    }
    *reinterpret_cast<uint32_t*>(out + (size_t)b * H * 64 + h * 64 + 2 * lane) = pack_bf16x2(ox, oy);
}

}  // namespace vqa

// Bandwidth-bound glue kernels of the CLIP-FlanT5 scoring path: norms, patch gather, embedding splice,
// relative-position bias table, log-sum-exp finalisation. All 16-byte vectorised, one row per block/warp.
#pragma once
#include "ptx.cuh"

namespace vqa {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// Block-wide sum for blockDim.x <= 1024; `red` is >= 32 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    float r = (l < nw) ? red[l] : 0.f;
    r = warp_sum(r);
    return r;
}

// T5LayerNorm (transformers/models/t5/modeling_t5.py:55-68): y = w * bf16(x * rsqrt(mean(x^2) + eps)); fp32 variance.
// One WARP per row (8 rows per 256-thread block): the lane keeps its NV 16-byte vectors of the row in registers, the sum of squares
// is a shuffle reduction (no shared memory, no block barrier), all NV loads of a lane are independent and in flight together.
// D == 256 * NV (each lane owns vectors lane, lane + 32, ... so every load/store instruction of the warp is a contiguous 512 bytes).
// Used for rows narrower than 4096 columns (the Qwen widths 1280 / 3584); 4096-wide T5 rows keep the block-per-row kernel below.
template <int NV>
__global__ void __launch_bounds__(256) t5_rmsnorm_warp_kernel(const __nv_bfloat16* __restrict__ x,
                                                             const __nv_bfloat16* __restrict__ w,
                                                             __nv_bfloat16* __restrict__ y, int rows, float eps) {
    pdl_launch_dependents();
    constexpr int D = 256 * NV;
    const int lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= (size_t)rows) return;
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * D);
    const uint4* wr = reinterpret_cast<const uint4*>(w);
    uint4* yr = reinterpret_cast<uint4*>(y + row * D);
    uint4 v[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = xr[lane + 32 * i];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const uint32_t* u = reinterpret_cast<const uint32_t*>(&v[i]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = unpack_bf16x2(u[e]);
            ss = fmaf(f.x, f.x, ss);
            ss = fmaf(f.y, f.y, ss);
        }
    }
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / (float)D + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const uint4 wv = __ldg(&wr[lane + 32 * i]);
        const uint32_t* u = reinterpret_cast<const uint32_t*>(&v[i]);
        const uint32_t* wu = reinterpret_cast<const uint32_t*>(&wv);
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = unpack_bf16x2(u[e]);
            const float2 g = unpack_bf16x2(wu[e]);
            o[e] = pack_bf16x2(g.x * bf16_round(f.x * rstd), g.y * bf16_round(f.y * rstd));
        }
        yr[lane + 32 * i] = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// Same norm for any D % 8 == 0 up to 8 * 256 * VPT: one block per row, block-wide reduction (T5-XXL's 4096 columns, and the odd widths of
// test configs).
template <int VPT>
__global__ void __launch_bounds__(256) t5_rmsnorm_kernel(const __nv_bfloat16* __restrict__ x,
                                                        const __nv_bfloat16* __restrict__ w,
                                                        __nv_bfloat16* __restrict__ y, int D, float eps) {
    pdl_launch_dependents();
    __shared__ float red[32];
    const size_t row = blockIdx.x;
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * D);
    const uint4* wr = reinterpret_cast<const uint4*>(w);
    uint4* yr = reinterpret_cast<uint4*>(y + row * D);
    const int nvec = D >> 3;
    uint4 v[VPT];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * blockDim.x;
        if (idx < nvec) {
            v[i] = xr[idx];
            const uint32_t* u = reinterpret_cast<const uint32_t*>(&v[i]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 f = unpack_bf16x2(u[e]);
                ss += f.x * f.x + f.y * f.y;
            }
        }
    }
    ss = block_sum(ss, red);
    const float rstd = rsqrtf(ss / (float)D + eps);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * blockDim.x;
        if (idx < nvec) {
            const uint4 wv = __ldg(&wr[idx]);
            const uint32_t* u = reinterpret_cast<const uint32_t*>(&v[i]);
            const uint32_t* wu = reinterpret_cast<const uint32_t*>(&wv);
            uint32_t o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 f = unpack_bf16x2(u[e]);
                float2 g = unpack_bf16x2(wu[e]);
                o[e] = pack_bf16x2(g.x * bf16_round(f.x * rstd), g.y * bf16_round(f.y * rstd));
            }
            yr[idx] = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

// nn.LayerNorm with affine, fp32 statistics (autocast runs layer_norm in fp32), bf16 out.
// One warp per row, D == 1024 (CLIP ViT-L hidden) or any D % 256 == 0 up to 2048.
// TIn = __nv_bfloat16 or float (the CLIP tower's fp32 residual stream); the output is always the bf16 tensor the next Linear consumes.
template <int D, typename TIn = __nv_bfloat16>
__global__ void __launch_bounds__(256) layernorm_kernel(const TIn* __restrict__ x,
                                                       const __nv_bfloat16* __restrict__ gamma,
                                                       const __nv_bfloat16* __restrict__ beta,
                                                       __nv_bfloat16* __restrict__ y, int rows, float eps) {
    pdl_launch_dependents();
    constexpr int VPL = D / 256;  // groups of 8 elements per lane
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    float f[VPL * 8];
    float s = 0.f;
    if constexpr (sizeof(TIn) == 4) {
        const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * D);
#pragma unroll
        for (int i = 0; i < VPL; ++i) {
            const float4 a = xr[(lane + i * 32) * 2], b = xr[(lane + i * 32) * 2 + 1];
            f[i * 8] = a.x; f[i * 8 + 1] = a.y; f[i * 8 + 2] = a.z; f[i * 8 + 3] = a.w;
            f[i * 8 + 4] = b.x; f[i * 8 + 5] = b.y; f[i * 8 + 6] = b.z; f[i * 8 + 7] = b.w;
            s += (a.x + a.y) + (a.z + a.w) + (b.x + b.y) + (b.z + b.w);
        }
    } else {
        const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * D);
#pragma unroll
        for (int i = 0; i < VPL; ++i) {
            uint4 v = xr[lane + i * 32];
            const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 t = unpack_bf16x2(u[e]);
                f[i * 8 + 2 * e] = t.x;
                f[i * 8 + 2 * e + 1] = t.y;
                s += t.x + t.y;
            }
        }
    }
    s = warp_sum(s);
    const float mean = s / (float)D;
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < VPL * 8; ++i) {
        const float d = f[i] - mean;
        var += d * d;
    }
    var = warp_sum(var) / (float)D;
    const float rstd = rsqrtf(var + eps);
    uint4* yr = reinterpret_cast<uint4*>(y + (size_t)row * D);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const uint4 g = __ldg(reinterpret_cast<const uint4*>(gamma) + lane + i * 32);
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(beta) + lane + i * 32);
        const uint32_t* gu = reinterpret_cast<const uint32_t*>(&g);
        const uint32_t* bu = reinterpret_cast<const uint32_t*>(&b);
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float2 gg = unpack_bf16x2(gu[e]);
            float2 bb = unpack_bf16x2(bu[e]);
            o[e] = pack_bf16x2((f[i * 8 + 2 * e] - mean) * rstd * gg.x + bb.x,
                               (f[i * 8 + 2 * e + 1] - mean) * rstd * gg.y + bb.y);
        }
        yr[lane + i * 32] = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// Non-overlapping 14x14 patches of [B,3,H,W] pixels -> rows of a [B*P, KPAD] bf16 matrix, k = c*ps*ps + ky*ps + kx
// (the flattening of the Conv2d weight [D,3,ps,ps], transformers/models/clip/modeling_clip.py:148-154,209-210).
// Pixels are rounded to bf16 first, as `pixel_values.to(dtype=target_dtype)` does. Columns >= 3*ps*ps are zero.
template <typename PixelT>
__global__ void patchify_kernel(const PixelT* __restrict__ pix, __nv_bfloat16* __restrict__ out, int B, int H, int W,
                                int ps, int kpad) {
    pdl_launch_dependents();
    const int gw = W / ps, gh = H / ps;
    const int P = gw * gh;
    const size_t row = blockIdx.x;  // b * P + p
    const int b = (int)(row / P), pidx = (int)(row % P);
    const int py = pidx / gw, px = pidx % gw;
    const int kreal = 3 * ps * ps;
    for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
        float v = 0.f;
        if (k < kreal) {
            const int c = k / (ps * ps), r = k % (ps * ps);
            const int ky = r / ps, kx = r % ps;
            v = (float)pix[(((size_t)b * 3 + c) * H + (py * ps + ky)) * W + (px * ps + kx)];
        }
        out[row * kpad + k] = __float2bfloat16_rn(v);
    }
}

// CLIP embeddings (+ class token, + position embedding) followed by pre_layrnorm, fused:
//   e[b,0] = cls + pos[0]; e[b,1+p] = patch[b,p] + pos[1+p]; h = LN(e)   (modeling_clip.py:212-217, 680)
// One warp per output row. D = 1024.
template <int D>
__global__ void __launch_bounds__(256) clip_embed_ln_kernel(const __nv_bfloat16* __restrict__ patch,  // [B*P, D]
                                                           const __nv_bfloat16* __restrict__ cls,    // [D]
                                                           const __nv_bfloat16* __restrict__ pos,    // [P+1, D]
                                                           const __nv_bfloat16* __restrict__ gamma,
                                                           const __nv_bfloat16* __restrict__ beta,
                                                           float* __restrict__ y,  // [B*(P+1), D] fp32: pre_layrnorm's output under autocast
                                                           int B, int P, float eps) {
    pdl_launch_dependents();
    constexpr int VPL = D / 256;
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= B * (P + 1)) return;
    const int lane = threadIdx.x & 31;
    const int b = row / (P + 1), t = row % (P + 1);
    const uint4* src = (t == 0) ? reinterpret_cast<const uint4*>(cls)
                                : reinterpret_cast<const uint4*>(patch + ((size_t)b * P + (t - 1)) * D);
    const uint4* pr = reinterpret_cast<const uint4*>(pos + (size_t)t * D);
    float f[VPL * 8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        uint4 v = src[lane + i * 32];
        uint4 pv = __ldg(&pr[lane + i * 32]);
        const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
        const uint32_t* pu = reinterpret_cast<const uint32_t*>(&pv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float2 a = unpack_bf16x2(u[e]);
            float2 c = unpack_bf16x2(pu[e]);
            const float x0 = bf16_round(a.x + c.x), x1 = bf16_round(a.y + c.y);  // bf16 add in the reference
            f[i * 8 + 2 * e] = x0;
            f[i * 8 + 2 * e + 1] = x1;
            s += x0 + x1;
        }
    }
    s = warp_sum(s);
    const float mean = s / (float)D;
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < VPL * 8; ++i) {
        const float d = f[i] - mean;
        var += d * d;
    }
    var = warp_sum(var) / (float)D;
    const float rstd = rsqrtf(var + eps);
    float4* yr = reinterpret_cast<float4*>(y + (size_t)row * D);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const uint4 g = __ldg(reinterpret_cast<const uint4*>(gamma) + lane + i * 32);
        const uint4 bb4 = __ldg(reinterpret_cast<const uint4*>(beta) + lane + i * 32);
        const uint32_t* gu = reinterpret_cast<const uint32_t*>(&g);
        const uint32_t* bu = reinterpret_cast<const uint32_t*>(&bb4);
        float o[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float2 gg = unpack_bf16x2(gu[e]);
            float2 bb = unpack_bf16x2(bu[e]);
            o[2 * e] = (f[i * 8 + 2 * e] - mean) * rstd * gg.x + bb.x;
            o[2 * e + 1] = (f[i * 8 + 2 * e + 1] - mean) * rstd * gg.y + bb.y;
        }
        yr[(lane + i * 32) * 2] = make_float4(o[0], o[1], o[2], o[3]);
        yr[(lane + i * 32) * 2 + 1] = make_float4(o[4], o[5], o[6], o[7]);
    }
}

// Multimodal splice (v3.0 prepare_inputs_labels_for_multimodal, SURVEY App. A): per sample the text ids before the
// image slot (-200) are embedded with `shared`, then the P projected patch features of image image_index[b], then
// the remaining ids; rows beyond the sample's length are zero. Output [B, S, D];
// seq_len[b] = text_len[b] - 1 + P. One block per output row.
__global__ void splice_embed_kernel(const int* __restrict__ ids,          // [B, L]  (image_token = image slot)
                                    const int* __restrict__ text_lens,    // [B]
                                    const int* __restrict__ image_index,  // [B] or nullptr (identity)
                                    const __nv_bfloat16* __restrict__ shared_emb,  // [V, D]
                                    const __nv_bfloat16* __restrict__ img_feat,    // [n_images * rows_per_image, ldf]
                                    int ldf, int feat_row_offset,  // first patch row inside each image's block (1: skip CLS)
                                    int feat_rows_per_image,
                                    __nv_bfloat16* __restrict__ out,  // [B, S, D]
                                    int* __restrict__ seq_lens,       // [B]
                                    int B, int L, int S, int P, int D, int image_token) {
    pdl_launch_dependents();
    const int b = blockIdx.x / S, s = blockIdx.x % S;
    const int tl = text_lens[b];
    __shared__ int slot_sh;
    if (threadIdx.x == 0) {
        int slot = -1;
        for (int i = 0; i < tl; ++i)
            if (ids[b * L + i] == image_token) { slot = i; break; }
        slot_sh = slot;
        if (s == 0) seq_lens[b] = (slot >= 0) ? tl - 1 + P : tl;
    }
    __syncthreads();
    const int slot = slot_sh;
    const int total = (slot >= 0) ? tl - 1 + P : tl;
    const int img = image_index ? image_index[b] : b;
    const uint4* src = nullptr;
    if (s < total) {
        if (slot < 0 || s < slot)
            src = reinterpret_cast<const uint4*>(shared_emb + (size_t)ids[b * L + s] * D);
        else if (s < slot + P)
            src = reinterpret_cast<const uint4*>(img_feat +
                                                 ((size_t)img * feat_rows_per_image + feat_row_offset + (s - slot)) * ldf);
        else
            src = reinterpret_cast<const uint4*>(shared_emb + (size_t)ids[b * L + (s - P + 1)] * D);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + ((size_t)b * S + s) * D);
    for (int i = threadIdx.x; i < (D >> 3); i += blockDim.x) dst[i] = src ? src[i] : make_uint4(0, 0, 0, 0);
}

// Decoder input embedding: decoder_input_ids = shift_right(labels) (modeling_t5.py:595-614): [start, l0, l1, ...],
// -100 -> pad. Every negative label becomes pad, not only -100: lse_finalize_kernel ignores all of them, and no negative id may index
// shared_emb. One block per (b, t).
__global__ void decoder_embed_kernel(const int* __restrict__ labels,  // [B, T]
                                     const __nv_bfloat16* __restrict__ shared_emb, __nv_bfloat16* __restrict__ out,
                                     int T, int D, int start_id, int pad_id) {
    pdl_launch_dependents();
    const int b = blockIdx.x / T, t = blockIdx.x % T;
    int id = (t == 0) ? start_id : labels[b * T + t - 1];
    if (id < 0) id = pad_id;
    const uint4* src = reinterpret_cast<const uint4*>(shared_emb + (size_t)id * D);
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)blockIdx.x * D);
    for (int i = threadIdx.x; i < (D >> 3); i += blockDim.x) dst[i] = src[i];
}

// bias_table[h, r] = rel_emb[lut[clamp(r - (S-1), +-max_dist) + max_dist], h] for r = key - query + (S-1).
// The bucket LUT is computed on the host (vqa_b200.cu host_rel_bucket, mirror of modeling_t5.py:189-234).
__global__ void bias_table_from_lut_kernel(const __nv_bfloat16* __restrict__ rel_emb, const int* __restrict__ lut,
                                           int max_dist, float* __restrict__ table, int H, int S) {
    pdl_launch_dependents();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int width = 2 * S - 1;
    if (idx >= H * width) return;
    const int hh = idx / width, r = idx % width;
    int rel = r - (S - 1);
    rel = min(max(rel, -max_dist), max_dist);
    table[idx] = __bfloat162float(rel_emb[lut[rel + max_dist] * H + hh]);
}

// Combine per-tile (max, sumexp) partials and the gathered label logits into the score:
//   logp[b,t] = logit[label] - logsumexp ; score[b] = exp(mean_t logp[b,t]) over labels >= 0
// (v3.0 CLIPT5Model.forward: (-CrossEntropyLoss(reduction='mean')(logits[k], labels[k])).exp()). A sample without a label scores NaN, the
// 0 / 0 of that mean. logprobs of ignored labels are not written. One warp per sample.
__global__ void lse_finalize_kernel(const float* __restrict__ lse_max, const float* __restrict__ lse_sum,
                                    const float* __restrict__ label_logit, const int* __restrict__ labels,
                                    float* __restrict__ scores, float* __restrict__ logprobs, int B, int T,
                                    int num_tiles) {
    pdl_launch_dependents();
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= B) return;
    const int lane = threadIdx.x & 31;
    float acc = 0.f;
    int cnt = 0;
    for (int t = 0; t < T; ++t) {
        const int row = b * T + t;
        if (labels[row] < 0) continue;
        float m = -INFINITY;
        for (int i = lane; i < num_tiles; i += 32) m = fmaxf(m, lse_max[(size_t)row * num_tiles + i]);
        m = warp_max(m);
        float s = 0.f;
        for (int i = lane; i < num_tiles; i += 32) {
            const float pm = lse_max[(size_t)row * num_tiles + i];
            if (pm > -INFINITY) s += lse_sum[(size_t)row * num_tiles + i] * expf(pm - m);
        }
        s = warp_sum(s);
        const float lp = label_logit[row] - (m + logf(s));
        if (logprobs && lane == 0) logprobs[row] = lp;
        acc += lp;
        ++cnt;
    }
    if (lane == 0) scores[b] = cnt > 0 ? expf(acc / (float)cnt) : __int_as_float(0x7fc00000);
}

}  // namespace vqa

// Glue kernels of the Qwen2.5-VL scoring path (rotary embeddings, window re-ordering, feature splice, last-token gather).
// All index arrays (positions, window order, feature rows) come from the host, which mirrors the reference's Python index
// logic bit for bit (t2v_metrics_b200/qwen_host.py <-> transformers/models/qwen2_5_vl/modeling_qwen2_5_vl.py:382-451,
// 1024-1133).
#pragma once
#include "ptx.cuh"
#include "elementwise.cuh"

namespace vqa {

// Block sizes of the glue kernels below (their launches: qwen25vl.cuh).
constexpr int GLUE_THREADS = 256;        // rope, bitmaps, top-k
constexpr int ROW_COPY_THREADS = 128;    // one block per row: gathers, embedding splice
inline int token_bitmap_words(int vocab) { return (vocab + 31) / 32; }

// cos/sin table for rotary embeddings: for i < half: angle = pos[axis_of_dim[i]][row] * inv_freq[i];
// table[row, i] = table[row, i + half] = cos/sin(angle)   (emb = cat(freqs, freqs), modeling_qwen2_5_vl.py:487, :611)
// pos: [n_axes, rows] int32. round_bf16: the text model casts cos/sin to the activation dtype (:614).
__global__ void rope_table_kernel(const int* __restrict__ pos, int rows, const int* __restrict__ axis_of_dim,
                                  const float* __restrict__ inv_freq, int half, float* __restrict__ cos_t,
                                  float* __restrict__ sin_t, int round_bf16) {
    pdl_launch_dependents();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * half) return;
    const int row = idx / half, i = idx % half;
    const float ang = (float)pos[(size_t)axis_of_dim[i] * rows + row] * inv_freq[i];
    float c = cosf(ang), s = sinf(ang);
    if (round_bf16) { c = bf16_round(c); s = bf16_round(s); }
    const size_t o = (size_t)row * (2 * half);
    cos_t[o + i] = c; cos_t[o + i + half] = c;
    sin_t[o + i] = s; sin_t[o + i + half] = s;
}

// In-place rotary embedding on `n_heads` consecutive heads of a packed row-major buffer (head h at column col0 + h*head_stride,
// `head_dim` <= head_stride real dims, head_dim % 16 == 0): x' = x*cos + rotate_half(x)*sin  (modeling_qwen2_5_vl.py:156-167,
// :650-669). bf16_products: the text path multiplies in bf16 (each product and the sum are rounded); the vision path works in
// fp32. One thread per (row, head, 8-dim chunk of the first half): 16-byte loads/stores of both halves.
__global__ void rope_inplace_kernel(__nv_bfloat16* __restrict__ x, int ld, int col0, int n_heads, int head_stride,
                                    int head_dim, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                    long long rows, int bf16_products) {
    pdl_launch_dependents();
    const int half = head_dim >> 1;
    const int chunks = half >> 3;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * n_heads * chunks) return;
    const int c = (int)(idx % chunks);
    const int h = (int)((idx / chunks) % n_heads);
    const long long row = idx / ((long long)chunks * n_heads);
    __nv_bfloat16* px = x + (size_t)row * ld + col0 + h * head_stride + c * 8;
    const float* pc = cos_t + (size_t)row * head_dim + c * 8;
    const float* ps = sin_t + (size_t)row * head_dim + c * 8;
    const uint4 v1 = *reinterpret_cast<const uint4*>(px);
    const uint4 v2 = *reinterpret_cast<const uint4*>(px + half);
    const uint32_t* u1 = reinterpret_cast<const uint32_t*>(&v1);
    const uint32_t* u2 = reinterpret_cast<const uint32_t*>(&v2);
    float c1[8], s1[8], c2[8], s2[8];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        *reinterpret_cast<float4*>(&c1[4 * i]) = *reinterpret_cast<const float4*>(pc + 4 * i);
        *reinterpret_cast<float4*>(&s1[4 * i]) = *reinterpret_cast<const float4*>(ps + 4 * i);
        *reinterpret_cast<float4*>(&c2[4 * i]) = *reinterpret_cast<const float4*>(pc + half + 4 * i);
        *reinterpret_cast<float4*>(&s2[4 * i]) = *reinterpret_cast<const float4*>(ps + half + 4 * i);
    }
    uint32_t o1[4], o2[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 a = unpack_bf16x2(u1[e]), b2 = unpack_bf16x2(u2[e]);
        float r1x, r1y, r2x, r2y;
        if (bf16_products) {
            r1x = bf16_round(a.x * c1[2 * e]) + bf16_round(-b2.x * s1[2 * e]);
            r1y = bf16_round(a.y * c1[2 * e + 1]) + bf16_round(-b2.y * s1[2 * e + 1]);
            r2x = bf16_round(b2.x * c2[2 * e]) + bf16_round(a.x * s2[2 * e]);
            r2y = bf16_round(b2.y * c2[2 * e + 1]) + bf16_round(a.y * s2[2 * e + 1]);
        } else {
            r1x = a.x * c1[2 * e] - b2.x * s1[2 * e];
            r1y = a.y * c1[2 * e + 1] - b2.y * s1[2 * e + 1];
            r2x = b2.x * c2[2 * e] + a.x * s2[2 * e];
            r2y = b2.y * c2[2 * e + 1] + a.y * s2[2 * e + 1];
        }
        o1[e] = pack_bf16x2(r1x, r1y);
        o2[e] = pack_bf16x2(r2x, r2y);
    }
    *reinterpret_cast<uint4*>(px) = make_uint4(o1[0], o1[1], o1[2], o1[3]);
    *reinterpret_cast<uint4*>(px + half) = make_uint4(o2[0], o2[1], o2[2], o2[3]);
}

// dst row r = src row index[r / group] * group + r % group (window re-ordering of 2x2 patch groups, and its inverse on the
// merged tokens with group = 1). D % 8 == 0. One block per destination row.
__global__ void gather_rows_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                   const int* __restrict__ index, int group, int D) {
    pdl_launch_dependents();
    const size_t r = blockIdx.x;
    const size_t s = (size_t)index[r / group] * group + r % group;
    const uint4* sp = reinterpret_cast<const uint4*>(src + s * D);
    uint4* dp = reinterpret_cast<uint4*>(dst + r * D);
    for (int i = threadIdx.x; i < (D >> 3); i += blockDim.x) dp[i] = sp[i];
}

// fp32 (or bf16) pixel patches -> bf16 (the Conv3d input cast, modeling_qwen2_5_vl.py:112-113)
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, size_t n) {
    pdl_launch_dependents();
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        const float4 v = *reinterpret_cast<const float4*>(src + i);
        *reinterpret_cast<uint2*>(dst + i) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    } else {
        for (size_t k = i; k < n; ++k) dst[k] = __float2bfloat16_rn(src[k]);
    }
}

// inputs_embeds = embed_tokens(ids); image-token positions are overwritten with the merged vision features
// (masked_scatter, modeling_qwen2_5_vl.py:1298-1307). feat_index[b*S+s] = row of `feats` or -1. Rows >= seq_len stay zero.
__global__ void qwen_embed_kernel(const int* __restrict__ ids, const int* __restrict__ feat_index, const int* __restrict__ seq_lens,
                                  const __nv_bfloat16* __restrict__ embed, const __nv_bfloat16* __restrict__ feats,
                                  __nv_bfloat16* __restrict__ out, int S, int D) {
    pdl_launch_dependents();
    const int b = blockIdx.x / S, s = blockIdx.x % S;
    const uint4* src = nullptr;
    if (s < seq_lens[b]) {
        const int f = feat_index[blockIdx.x];
        src = (f >= 0) ? reinterpret_cast<const uint4*>(feats + (size_t)f * D)
                       : reinterpret_cast<const uint4*>(embed + (size_t)ids[blockIdx.x] * D);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)blockIdx.x * D);
    for (int i = threadIdx.x; i < (D >> 3); i += blockDim.x) dst[i] = src ? src[i] : make_uint4(0, 0, 0, 0);
}

// out[b] = x[b*S + seq_len[b] - 1]: the last prompt position, the only one lm_head is applied to (logits_to_keep = 1).
__global__ void gather_last_rows_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ seq_lens,
                                        __nv_bfloat16* __restrict__ out, int S, int D) {
    pdl_launch_dependents();
    const int b = blockIdx.x;
    const int last = max(seq_lens[b], 1) - 1;
    const uint4* src = reinterpret_cast<const uint4*>(x + ((size_t)b * S + last) * D);
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)b * D);
    for (int i = threadIdx.x; i < (D >> 3); i += blockDim.x) dst[i] = src[i];
}

// bitmap[b, id / 32] |= 1 << (id % 32) for every prompt id of sample b (the set RepetitionPenaltyLogitsProcessor gathers over).
__global__ void token_bitmap_kernel(const int* __restrict__ ids, const int* __restrict__ seq_lens, int B, int S, int vocab,
                                    uint32_t* __restrict__ bitmap, int words) {
    pdl_launch_dependents();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * S) return;
    const int b = idx / S, s = idx % S;
    if (s >= seq_lens[b]) return;
    const int id = ids[idx];
    if (id < 0 || id >= vocab) return;
    atomicOr(&bitmap[(size_t)b * words + (id >> 5)], 1u << (id & 31));
}

// Packed-rows mode (shared vision prefixes): out[b] = x[row[b]], the last prompt position of pair b.
__global__ void gather_rows_by_index_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ row, __nv_bfloat16* __restrict__ out, int D) {
    pdl_launch_dependents();
    const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)row[blockIdx.x] * D);
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)blockIdx.x * D);
    for (int i = threadIdx.x; i < (D >> 3); i += blockDim.x) dst[i] = src[i];
}

// Packed-rows mode: the prompt of pair b = rows of its prefix sequence (kv_prefix[pair_seq[b]], if any) + rows of its own sequence.
// grid (ceil(max_prompt_len / 256), B).
__global__ void token_bitmap_packed_kernel(const int* __restrict__ ids, const int* __restrict__ cu, const int* __restrict__ kv_prefix,
                                           const int* __restrict__ pair_seq, int vocab, uint32_t* __restrict__ bitmap, int words) {
    pdl_launch_dependents();
    const int b = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
    const int sq = pair_seq[b], pre = kv_prefix ? kv_prefix[sq] : -1;
    const int pre_len = pre >= 0 ? cu[pre + 1] - cu[pre] : 0;
    const int own_len = cu[sq + 1] - cu[sq];
    if (t >= pre_len + own_len) return;
    const int id = t < pre_len ? ids[cu[pre] + t] : ids[cu[sq] + (t - pre_len)];
    if (id < 0 || id >= vocab) return;
    atomicOr(&bitmap[(size_t)b * words + (id >> 5)], 1u << (id & 31));
}

// prob[b] = exp(logprob[b])
__global__ void exp_kernel(const float* __restrict__ lp, float* __restrict__ out, int n) {
    pdl_launch_dependents();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = expf(lp[i]);
}

// Trace output (reference forward_with_trace, qwen2vl_model.py:439-447: torch.topk(softmax(scores / T), 5)): the k most probable tokens of
// one row of materialised last-position logits, with their probabilities under the same processing as the scoring path (bf16 logits ->
// fp32 -> repetition penalty -> 1/T -> full-vocabulary softmax). One block per row; a debugging aid, not on the scoring path.
constexpr int TOPK_MAX = 8;
__global__ void __launch_bounds__(256) topk_softmax_kernel(const __nv_bfloat16* __restrict__ logits, long long ldl, int V, float inv_temp,
                                                           const uint32_t* __restrict__ pen_bitmap, int pen_words, float penalty, int K,
                                                           int* __restrict__ out_ids, float* __restrict__ out_probs) {
    pdl_launch_dependents();
    __shared__ float s_val[256 * TOPK_MAX];
    __shared__ int s_idx[256 * TOPK_MAX];
    __shared__ float s_red[2][8];
    const int row = blockIdx.x, tid = threadIdx.x;
    const __nv_bfloat16* lr = logits + (size_t)row * ldl;
    const uint32_t* pb = pen_bitmap ? pen_bitmap + (size_t)row * pen_words : nullptr;
    float tv[TOPK_MAX];
    int ti[TOPK_MAX];
#pragma unroll
    for (int i = 0; i < TOPK_MAX; ++i) { tv[i] = -INFINITY; ti[i] = -1; }
    float mx = -INFINITY, sm = 0.f;
    for (int n = tid; n < V; n += 256) {
        float x = __bfloat162float(lr[n]);
        if (pb && ((pb[n >> 5] >> (n & 31)) & 1u)) x = x < 0.f ? x * penalty : __fdiv_rn(x, penalty);
        x *= inv_temp;
        if (x > mx) { sm = sm * __expf(mx - x) + 1.f; mx = x; } else { sm += __expf(x - mx); }
        if (x > tv[TOPK_MAX - 1]) {          // insert into the sorted local list (ties keep the lower id first, like torch.topk on a scan)
            int pos = TOPK_MAX - 1;
#pragma unroll
            for (int i = TOPK_MAX - 2; i >= 0; --i)
                if (x > tv[i]) { tv[i + 1] = tv[i]; ti[i + 1] = ti[i]; pos = i; }
            tv[pos] = x; ti[pos] = n;
        }
    }
    // block-wide log-sum-exp
    float bm = mx;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, o));
    if ((tid & 31) == 0) s_red[0][tid >> 5] = bm;
    __syncthreads();
    bm = s_red[0][0];
#pragma unroll
    for (int i = 1; i < 8; ++i) bm = fmaxf(bm, s_red[0][i]);
    float bs = (mx == -INFINITY) ? 0.f : sm * __expf(mx - bm);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bs += __shfl_xor_sync(0xffffffffu, bs, o);
    if ((tid & 31) == 0) s_red[1][tid >> 5] = bs;
#pragma unroll
    for (int i = 0; i < TOPK_MAX; ++i) { s_val[tid * TOPK_MAX + i] = tv[i]; s_idx[tid * TOPK_MAX + i] = ti[i]; }
    __syncthreads();
    if (tid < 32) {
        float total = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) total += s_red[1][i];
        for (int k = 0; k < K; ++k) {
            float best = -INFINITY; int bpos = -1, bid = 0x7fffffff;
            for (int j = tid; j < 256 * TOPK_MAX; j += 32) {
                const float v = s_val[j]; const int id = s_idx[j];
                if (id >= 0 && (v > best || (v == best && id < bid))) { best = v; bpos = j; bid = id; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, best, o);
                const int op = __shfl_xor_sync(0xffffffffu, bpos, o), oid = __shfl_xor_sync(0xffffffffu, bid, o);
                if (ov > best || (ov == best && oid < bid)) { best = ov; bpos = op; bid = oid; }
            }
            if (tid == 0) {
                out_ids[row * K + k] = bpos >= 0 ? bid : -1;
                out_probs[row * K + k] = bpos >= 0 ? __expf(best - bm) / total : 0.f;
                if (bpos >= 0) s_idx[bpos] = -1;      // remove the winner
            }
            __syncwarp();
        }
    }
}

}  // namespace vqa

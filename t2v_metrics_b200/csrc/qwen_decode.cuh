// Kernels of the Qwen2.5-VL decode loop and their launches: the K/V cache write, flash-decoding attention over the cache, and greedy or
// sampled token selection with the per-step bookkeeping. Every step-dependent value (generated lengths, finished flags, next input ids and
// positions) lives in device memory, so the launches of one decode step take the same arguments at every step and replay from one CUDA graph.
#pragma once
#include <cfloat>
#include "host.cuh"

namespace vqa {

// K/V cache of one layer: K and V each [B, Hkv, cap, 128] bf16 (post-rope K, as HF's DynamicCache stores it).
// Source: the packed qkv activation [rows, ld] of the layer, K heads at k_col0, V heads at v_col0, row r = b * S + s.
//   prefill (gen_len == nullptr): rows s < seq_lens[b] go to slot s;
//   decode  (S == 1):             the one row of sequence b goes to slot seq_lens[b] + gen_len[b] - 1 (the position of the input token).
// One thread per (row, kv head, 16-byte chunk).
__global__ void kv_cache_write_kernel(const __nv_bfloat16* __restrict__ qkv, int ld, int k_col0, int v_col0, int Hkv, int S, long long rows,
                                      const int* __restrict__ seq_lens, const int* __restrict__ gen_len, __nv_bfloat16* __restrict__ kc,
                                      __nv_bfloat16* __restrict__ vc, int cap) {
    pdl_launch_dependents();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * Hkv * 16) return;
    const int c = (int)(idx & 15), h = (int)((idx >> 4) % Hkv);
    const long long r = idx / (16LL * Hkv);
    const int b = (int)(r / S), s = (int)(r % S);
    int slot;
    if (gen_len) {
        slot = seq_lens[b] + gen_len[b] - 1 + s;
    } else {
        if (s >= seq_lens[b]) return;
        slot = s;
    }
    const size_t dst = (((size_t)b * Hkv + h) * cap + slot) * 128 + c * 8;
    const __nv_bfloat16* src = qkv + (size_t)r * ld + h * 128 + c * 8;
    *reinterpret_cast<uint4*>(kc + dst) = *reinterpret_cast<const uint4*>(src + k_col0);
    *reinterpret_cast<uint4*>(vc + dst) = *reinterpret_cast<const uint4*>(src + v_col0);
}

// Decode attention, head_dim 128, causal GQA over the cache (flash-decoding). One query row per q head; sequence b attends to cache
// slots [0, seq_lens[b] + gen_len[b]) -- the prompt, every generated token before this step's input, and the input itself.
// grid (splits, Hkv, B), 128 threads: the CTA holds the G q heads of one KV head, so each K/V byte is read once per group, and covers
// keys [split * chunk, (split + 1) * chunk). Each warp runs an online softmax over every 4th key of the range (lane = 4 dims), the four
// warps are merged in shared memory, and the CTA writes its unnormalised partial (max, sum, output) for decode_attn_merge_kernel.
constexpr int DEC_ATTN_WARPS = 4;
template <int G>
__global__ void __launch_bounds__(32 * DEC_ATTN_WARPS) decode_attn_partial_kernel(
        const __nv_bfloat16* __restrict__ q, int ldq, const __nv_bfloat16* __restrict__ kc, const __nv_bfloat16* __restrict__ vc, int cap,
        const int* __restrict__ seq_lens, const int* __restrict__ gen_len, int Hkv, int chunk, float scale, float* __restrict__ part_o,
        float* __restrict__ part_ml) {
    pdl_launch_dependents();
    __shared__ float s_m[DEC_ATTN_WARPS][G], s_l[DEC_ATTN_WARPS][G];
    __shared__ float s_o[DEC_ATTN_WARPS][G][128];
    const int sp = blockIdx.x, kh = blockIdx.y, b = blockIdx.z, splits = gridDim.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int len = seq_lens[b] + gen_len[b];
    const int k0 = sp * chunk, k1 = min(len, k0 + chunk);
    const int Hq = Hkv * G;
    float qv[G][4], acc[G][4], m[G], l[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
        const uint2 u = *reinterpret_cast<const uint2*>(q + (size_t)b * ldq + (kh * G + g) * 128 + lane * 4);
        const float2 a = unpack_bf16x2(u.x), c = unpack_bf16x2(u.y);
        qv[g][0] = a.x * scale; qv[g][1] = a.y * scale; qv[g][2] = c.x * scale; qv[g][3] = c.y * scale;
        acc[g][0] = acc[g][1] = acc[g][2] = acc[g][3] = 0.f;
        m[g] = -INFINITY; l[g] = 0.f;
    }
    const size_t base = ((size_t)b * Hkv + kh) * cap * 128 + lane * 4;
    for (int j = k0 + warp; j < k1; j += DEC_ATTN_WARPS) {
        const uint2 ku = *reinterpret_cast<const uint2*>(kc + base + (size_t)j * 128);
        const uint2 vu = *reinterpret_cast<const uint2*>(vc + base + (size_t)j * 128);
        const float2 k01 = unpack_bf16x2(ku.x), k23 = unpack_bf16x2(ku.y), v01 = unpack_bf16x2(vu.x), v23 = unpack_bf16x2(vu.y);
#pragma unroll
        for (int g = 0; g < G; ++g) {
            float s = qv[g][0] * k01.x + qv[g][1] * k01.y + qv[g][2] * k23.x + qv[g][3] * k23.y;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            const float mn = fmaxf(m[g], s);
            const float c = __expf(m[g] - mn), p = __expf(s - mn);
            l[g] = l[g] * c + p;
            acc[g][0] = acc[g][0] * c + p * v01.x; acc[g][1] = acc[g][1] * c + p * v01.y;
            acc[g][2] = acc[g][2] * c + p * v23.x; acc[g][3] = acc[g][3] * c + p * v23.y;
            m[g] = mn;
        }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
        if (lane == 0) { s_m[warp][g] = m[g]; s_l[warp][g] = l[g]; }
        *reinterpret_cast<float4*>(&s_o[warp][g][lane * 4]) = make_float4(acc[g][0], acc[g][1], acc[g][2], acc[g][3]);
    }
    __syncthreads();
    const int d = threadIdx.x;     // 128 threads = 128 output dims
#pragma unroll
    for (int g = 0; g < G; ++g) {
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < DEC_ATTN_WARPS; ++w) M = fmaxf(M, s_m[w][g]);
        float L = 0.f, O = 0.f;
#pragma unroll
        for (int w = 0; w < DEC_ATTN_WARPS; ++w) {
            const float e = s_m[w][g] == -INFINITY ? 0.f : __expf(s_m[w][g] - M);
            L += s_l[w][g] * e;
            O += s_o[w][g][d] * e;
        }
        const size_t row = ((size_t)b * Hq + kh * G + g) * splits + sp;
        part_o[row * 128 + d] = O;
        if (d == 0) { part_ml[row * 2] = M; part_ml[row * 2 + 1] = L; }
    }
}

// out[b, h * 128 + d] = bf16(sum_s o_s[d] e^(m_s - M) / sum_s l_s e^(m_s - M)) over the splits of (b, h). grid B * Hq, 128 threads.
__global__ void decode_attn_merge_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml, int splits,
                                         __nv_bfloat16* __restrict__ out, int ldo, int Hq) {
    pdl_launch_dependents();
    const int bh = blockIdx.x, b = bh / Hq, h = bh % Hq, d = threadIdx.x;
    const float* ml = part_ml + (size_t)bh * splits * 2;
    float M = -INFINITY;
    for (int s = 0; s < splits; ++s) M = fmaxf(M, ml[2 * s]);
    float L = 0.f, O = 0.f;
    for (int s = 0; s < splits; ++s) {
        const float ms = ml[2 * s];
        if (ms == -INFINITY) continue;
        const float e = __expf(ms - M);
        L += ml[2 * s + 1] * e;
        O += part_o[((size_t)bh * splits + s) * 128 + d] * e;
    }
    out[(size_t)b * ldo + h * 128 + d] = __float2bfloat16_rn(O / L);
}

// Generation state at the start of a prefill: nothing generated, nothing finished, output ids -1.
__global__ void generate_init_kernel(int B, int max_new, int* __restrict__ tokens, int* __restrict__ lengths, int* __restrict__ done,
                                     int* __restrict__ n_done, int* __restrict__ all_done) {
    pdl_launch_dependents();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    for (int k = i; k < B * max_new; k += gridDim.x * blockDim.x) tokens[k] = -1;
    if (i < B) { lengths[i] = 0; done[i] = 0; }
    if (i == 0) { *n_done = 0; *all_done = 0; }
}

// Greedy token selection and the per-token bookkeeping, one block per sequence. The processed logit of id n is HF's: the bf16 lm_head
// output cast to fp32, then RepetitionPenaltyLogitsProcessor when a penalty bitmap is given (every prompt id and every generated id);
// the token is the arg-max, ties to the lowest id (torch.argmax). A sequence that is not finished appends the token to tokens[b],
// sets its penalty bit, advances lengths[b], and stores the next step's input id and, when pos3 is given, its (t, h, w) position (all
// three axes advance together after the prompt: first_pos[b] + index of the token; the T5 decoder passes nullptr for both and has no
// positions to keep). It finishes on an EOS id or at max_new tokens; the block that finishes the last sequence raises *all_done. A finished
// sequence is left untouched.
constexpr int SELECT_THREADS = 1024;

// The per-token bookkeeping of both selection kernels, run by one thread of sequence b's block once its token `tok` is chosen.
__device__ __forceinline__ void select_commit(int b, int tok, uint32_t* pen_bitmap, int pen_words, const int* eos_ids, int n_eos, int max_new,
                                              const int* first_pos, int B, int* tokens, int* lengths, int* done, int* n_done, int* all_done,
                                              int* next_ids, int* pos3) {
    const int t = lengths[b];
    tokens[(size_t)b * max_new + t] = tok;
    lengths[b] = t + 1;
    if (pen_bitmap) pen_bitmap[(size_t)b * pen_words + (tok >> 5)] |= 1u << (tok & 31);
    next_ids[b] = tok;
    if (pos3) {
        const int p = first_pos[b] + t;
        pos3[b] = p; pos3[B + b] = p; pos3[2 * B + b] = p;
    }
    bool fin = t + 1 >= max_new;
    for (int e = 0; e < n_eos; ++e) fin |= tok == eos_ids[e];
    if (fin) {
        done[b] = 1;
        if (atomicAdd(n_done, 1) + 1 == B) *all_done = 1;
    }
}

// bf16 logit -> fp32 -> HF's RepetitionPenaltyLogitsProcessor when id n's bit is set in the row's bitmap pb (NULL = no penalty)
__device__ __forceinline__ float penalised_logit(const __nv_bfloat16* lr, const uint32_t* pb, float penalty, int n) {
    float x = __bfloat162float(lr[n]);
    if (pb && ((pb[n >> 5] >> (n & 31)) & 1u)) x = x < 0.f ? x * penalty : __fdiv_rn(x, penalty);
    return x;
}

// Block-wide arg-max of (best, bid) over SELECT_THREADS threads, ties to the lowest id; every thread gets the result. s_v / s_i hold
// SELECT_THREADS / 32 entries.
__device__ __forceinline__ int block_argmax(float best, int bid, float* s_v, int* s_i) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bid, o);
        if (ov > best || (ov == best && oi < bid)) { best = ov; bid = oi; }
    }
    if ((tid & 31) == 0) { s_v[tid >> 5] = best; s_i[tid >> 5] = bid; }
    __syncthreads();
    best = s_v[0]; bid = s_i[0];
    for (int w = 1; w < SELECT_THREADS / 32; ++w)
        if (s_v[w] > best || (s_v[w] == best && s_i[w] < bid)) { best = s_v[w]; bid = s_i[w]; }
    return bid;
}

__global__ void __launch_bounds__(SELECT_THREADS) greedy_select_kernel(
        const __nv_bfloat16* __restrict__ logits, int V, uint32_t* __restrict__ pen_bitmap, int pen_words, float penalty,
        const int* __restrict__ eos_ids, int n_eos, int max_new, const int* __restrict__ first_pos, int B, int* __restrict__ tokens,
        int* __restrict__ lengths, int* __restrict__ done, int* __restrict__ n_done, int* __restrict__ all_done, int* __restrict__ next_ids,
        int* __restrict__ pos3) {
    pdl_launch_dependents();
    __shared__ float s_v[SELECT_THREADS / 32];
    __shared__ int s_i[SELECT_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    if (done[b]) return;
    const __nv_bfloat16* lr = logits + (size_t)b * V;
    const uint32_t* pb = pen_bitmap ? pen_bitmap + (size_t)b * pen_words : nullptr;
    float best = -INFINITY;
    int bid = 0x7fffffff;
    for (int n = tid; n < V; n += SELECT_THREADS) {
        const float x = penalised_logit(lr, pb, penalty, n);
        if (x > best || bid == 0x7fffffff) { best = x; bid = n; }      // ids rise along the scan: strict > keeps the lowest of equals
    }
    const int tok = block_argmax(best, bid, s_v, s_i);
    if (tid == 0)
        select_commit(b, tok, pen_bitmap, pen_words, eos_ids, n_eos, max_new, first_pos, B, tokens, lengths, done, n_done, all_done, next_ids,
                      pos3);
}

// ------------------------------------------------------------------------------------------------ sampled selection
// Philox4x32-10 (Salmon, Moraes, Dror & Shaw, SC'11; the philox4x32 of Random123 with 10 rounds): counter c, key (k0, k1).
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// fp32 -> uint32 whose unsigned order is the float order (+0 and -0 must have been merged before)
__device__ __forceinline__ uint32_t order_key(float x) {
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// The processed score of id n for sampling (see sample_select_kernel): the penalised logit, / temperature (none at 1), -0 as +0,
// saturated to [-FLT_MAX, FLT_MAX] (fmaxf(NaN, -FLT_MAX) is -FLT_MAX)
__device__ __forceinline__ float sample_score(const __nv_bfloat16* lr, const uint32_t* pb, float penalty, float temperature, int n) {
    float x = penalised_logit(lr, pb, penalty, n);
    if (temperature != 1.0f) x = __fdiv_rn(x, temperature);
    return x == 0.f ? 0.f : fminf(fmaxf(x, -FLT_MAX), FLT_MAX);
}

// Mass exp(x - max) of one token as an integer of 2^-40 units: sums of them are exact and independent of the summation order, so the
// top-p cut is deterministic. A vocabulary of < 2^23 tokens, each <= 2^40, cannot overflow 64 bits; dropping terms below 2^-41 moves a
// cumulative probability by < V * 2^-41 (7e-8 at V = 152,064). mass_of_exp is the quantisation of the fp32 ex = expf(x - max).
__device__ __forceinline__ unsigned long long mass_of_exp(float ex) {
    return (unsigned long long)(ex * 1099511627776.0f + 0.5f);
}
__device__ __forceinline__ unsigned long long mass_fx(float x, float mx) { return mass_of_exp(expf(x - mx)); }

// The Philox block of ids 4g .. 4g + 3 at step t under seed (lo, hi), and lane l of it (id 4g + l)
__device__ __forceinline__ uint4 sample_philox(int g, int step, uint32_t seed_lo, uint32_t seed_hi) {
    return philox4x32_10(make_uint4((uint32_t)g, (uint32_t)step, 0u, 0u), seed_lo, seed_hi);
}
__device__ __forceinline__ uint32_t philox_lane(uint4 r, int l) { return l == 0 ? r.x : l == 1 ? r.y : l == 2 ? r.z : r.w; }

// The Gumbel term of one id from its Philox lane bits: e = -log(u), u = (m + 0.5) 2^-24 with m = bits >> 8, taken without rounding u:
// for m >= 2^23, 1 - u = (2^24 - m - 0.5) 2^-24 is exact instead. The perturbed score is (x - max) - log(e).
__device__ __forceinline__ float gumbel_e(uint32_t bits) {
    const uint32_t m = bits >> 8;
    return m < (1u << 23) ? -logf(((float)m + 0.5f) * 5.9604644775390625e-8f) : -log1pf(-((float)((1u << 24) - m) - 0.5f) * 5.9604644775390625e-8f);
}
__device__ __forceinline__ float gumbel_perturbed(float x, float mx, float e) { return (x - mx) - logf(e); }

constexpr int SAMPLE_BINS = 2048;       // 11-bit radix digits: three passes (11, 11, 10 bits) select one 32-bit key
constexpr int SAMPLE_UNROLL = 8;

// Of the bins h[0, nb) taken from the highest when from_top (else from the lowest), the first whose inclusive running sum exceeds
// *target; on return every thread sees that bin in *bin and *target reduced by the sum of the bins before it. With frac >= 0 the target is
// first set to floor(frac * sum of all bins). A target at or past the sum of all bins (frac rounded to 1, e.g. fp32(1 - 1e-8)) is taken
// as that sum - 1: the last unit then sits past it, so the last bin is found, as HF keeps its last id when every cumulative probability
// is at or below the threshold. The callers' bins never sum to 0. Each thread owns two consecutive positions of the order; s_w holds 32
// partial sums.
__device__ void radix_find(const unsigned long long* h, int nb, bool from_top, float frac, unsigned long long* target, int* bin,
                           unsigned long long* s_w) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    auto at = [&](int o) -> unsigned long long { return o < nb ? h[from_top ? nb - 1 - o : o] : 0ull; };
    const unsigned long long a = at(2 * tid), c = at(2 * tid + 1);
    unsigned long long incl = a + c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    unsigned long long before = 0, total = 0;
    for (int w = 0; w < SELECT_THREADS / 32; ++w) {
        if (w < warp) before += s_w[w];
        total += s_w[w];
    }
    const unsigned long long excl = before + incl - a - c;
    unsigned long long tg = frac >= 0.f ? (unsigned long long)((double)frac * (double)total) : *target;
    if (tg >= total) tg = total - 1;
    __syncthreads();      // every thread has read *target and s_w
    if (excl <= tg && tg < excl + a + c) {
        const bool first = tg < excl + a;
        const int o = 2 * tid + (first ? 0 : 1);
        *bin = from_top ? nb - 1 - o : o;
        *target = tg - (first ? excl : excl + a);
    }
    __syncthreads();
}

// Sampled token selection, a drop-in for greedy_select_kernel (same bookkeeping through select_commit), one block per sequence. The
// processed score of id n is HF's for generate(do_sample=True): the penalised fp32 logit, then TemperatureLogitsWarper (an IEEE fp32
// division by `temperature`, skipped at 1), with -0 taken as +0 and saturated to [-FLT_MAX, FLT_MAX] (a score that overflows, or a NaN
// logit, makes HF's softmax NaN and torch.multinomial raise; here +inf ties at FLT_MAX and -inf or NaN take -FLT_MAX, so the maximum is
// finite, the mass of the maximum is 2^40 and a kept id always exists). Then, as HF's warpers in order:
//   top-k (0 < top_k < V): the k-th largest score v_k, found by radix select; every id with score >= v_k stays, ties included;
//   top-p (top_p < 1): in ascending (score, id) order, the ids whose cumulative probability among the kept ones is <= fp32(1 - top_p)
//     go; the most probable id always stays. Within the group of equal scores at the cut, lower ids go first (what a stable ascending
//     sort gives). The cut's score is found by radix select over the cumulative mass; the group's split by one pass in id order.
// The token is the Gumbel-max over the kept ids: argmax((score_n - max) - log(-log u_n)) (ties to the lowest id), which draws id n with
// probability softmax(kept scores)[n]. u_n is lane n & 3 of Philox4x32-10 with key seeds[b] (low word first) and counter
// (n >> 2, t, 0, 0), t = lengths[b], as ((bits >> 8) + 0.5) * 2^-24 (-log u is taken without rounding u; both logs are the accurate
// logf / log1pf): the draw depends on (seed, step, id) only, not on the batch position, the launch or the thread layout.
// kept (debugging, NULL = none): the kept set as a bitmap [B, ceil(V / 32)], fully rewritten.
__global__ void __launch_bounds__(SELECT_THREADS) sample_select_kernel(
        const __nv_bfloat16* __restrict__ logits, int V, uint32_t* __restrict__ pen_bitmap, int pen_words, float penalty,
        const unsigned long long* __restrict__ seeds, float temperature, int top_k, double top_p, const int* __restrict__ eos_ids, int n_eos,
        int max_new, const int* __restrict__ first_pos, int B, int* __restrict__ tokens, int* __restrict__ lengths, int* __restrict__ done,
        int* __restrict__ n_done, int* __restrict__ all_done, int* __restrict__ next_ids, int* __restrict__ pos3, uint32_t* __restrict__ kept) {
    pdl_launch_dependents();
    __shared__ unsigned long long s_h[SAMPLE_BINS];
    __shared__ unsigned long long s_w[SELECT_THREADS / 32];
    __shared__ float s_v[SELECT_THREADS / 32];
    __shared__ int s_i[SELECT_THREADS / 32];
    __shared__ unsigned long long s_target;
    __shared__ int s_bin;
    const int b = blockIdx.x, tid = threadIdx.x;
    if (done[b]) return;
    const __nv_bfloat16* lr = logits + (size_t)b * V;
    const uint32_t* pb = pen_bitmap ? pen_bitmap + (size_t)b * pen_words : nullptr;
    const int step = lengths[b];
    auto score = [&](int n) { return sample_score(lr, pb, penalty, temperature, n); };
    // fn(n, score(n)) for every id; a thread reads SAMPLE_UNROLL ids before it consumes them, so it has that many loads in flight
    auto scan_row = [&](auto&& fn) {
        for (int base = 0; base < V; base += SELECT_THREADS * SAMPLE_UNROLL) {
            float x[SAMPLE_UNROLL];
#pragma unroll
            for (int u = 0; u < SAMPLE_UNROLL; ++u) {
                const int n = base + u * SELECT_THREADS + tid;
                x[u] = n < V ? score(n) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < SAMPLE_UNROLL; ++u) {
                const int n = base + u * SELECT_THREADS + tid;
                if (n < V) fn(n, x[u]);
            }
        }
    };
    // the maximum (the reference point of the masses)
    float mx = -INFINITY;
    scan_row([&](int, float x) { mx = fmaxf(mx, x); });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) s_v[tid >> 5] = mx;
    __syncthreads();
    for (int w = 0; w < SELECT_THREADS / 32; ++w) mx = fmaxf(mx, s_v[w]);
    __syncthreads();

    // Three radix passes over the keys of the ids `in` admits: the key at which the running sum of add(n) -- taken from the highest key
    // when from_top -- first exceeds the target; returns it, the target reduced by the sum of all keys before it.
    auto radix_select = [&](auto&& in, auto&& add, bool from_top, float frac, unsigned long long target, uint32_t* key_out) {
        uint32_t prefix = 0, mask = 0;
        if (tid == 0) s_target = target;
        for (int pass = 0; pass < 3; ++pass) {
            const int shift = pass == 0 ? 21 : pass == 1 ? 10 : 0, nb = pass == 2 ? 1024 : 2048;
            for (int i = tid; i < SAMPLE_BINS; i += SELECT_THREADS) s_h[i] = 0ull;
            __syncthreads();
            scan_row([&](int, float x) {
                const uint32_t k = order_key(x);
                if ((k & mask) == prefix && in(k)) atomicAdd(&s_h[(k >> shift) & (nb - 1)], add(x));
            });
            __syncthreads();
            radix_find(s_h, nb, from_top, pass == 0 ? frac : -1.f, &s_target, &s_bin, s_w);
            prefix |= (uint32_t)s_bin << shift;
            mask |= (uint32_t)(nb - 1) << shift;
        }
        *key_out = prefix;
        return s_target;
    };
    // top-k: the k-th largest key (k - 1 keys above it); ids below it are out
    uint32_t key_k = 0;
    if (top_k > 0 && top_k < V)
        radix_select([](uint32_t) { return true; }, [](float) { return 1ull; }, true, -1.f, (unsigned long long)(top_k - 1), &key_k);
    // top-p: the key whose group holds the cut, and how many of the group (lowest ids first) go
    uint32_t key_p = 0;
    int id_p = 0;
    if (top_p < 1.0) {
        const float thr = (float)(1.0 - top_p);      // HF's threshold: the caller's 1 - top_p in double, compared in fp32
        unsigned long long rest = radix_select([&](uint32_t k) { return k >= key_k; }, [&](float x) { return mass_fx(x, mx); }, false, thr,
                                               0ull, &key_p);
        // ids of the group at the cut with cumulative mass below + (j + 1) q <= limit go: the first floor(rest / q)
        const float xv = __uint_as_float((key_p & 0x80000000u) ? (key_p & 0x7fffffffu) : ~key_p);
        const unsigned long long q = mass_fx(xv, mx);
        const int drop = (int)(rest / q);
        if (drop > 0) {
            // the id of group member `drop` in id order: each thread counts the members in its own contiguous id range
            const int per = (V + SELECT_THREADS - 1) / SELECT_THREADS, n0 = min(V, tid * per), n1 = min(V, n0 + per);
            int cnt = 0;
            for (int n = n0; n < n1; ++n) cnt += order_key(score(n)) == key_p;
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, o);
                if ((tid & 31) >= o) incl += v;
            }
            if ((tid & 31) == 31) s_i[tid >> 5] = incl;
            __syncthreads();
            int before = incl - cnt;
            for (int w = 0; w < (tid >> 5); ++w) before += s_i[w];
            if (before <= drop && drop < before + cnt) {
                int j = before;
                for (int n = n0; n < n1; ++n)
                    if (order_key(score(n)) == key_p && j++ == drop) { s_bin = n; break; }
            }
            __syncthreads();
            id_p = s_bin;
            __syncthreads();
        }
    }
    // Gumbel-max over the kept ids; each thread takes four consecutive ids, the four lanes of one Philox block
    const uint32_t seed_lo = (uint32_t)seeds[b], seed_hi = (uint32_t)(seeds[b] >> 32);
    uint32_t* kb = kept ? kept + (size_t)b * pen_words : nullptr;
    if (kb) {
        for (int w = tid; w < pen_words; w += SELECT_THREADS) kb[w] = 0u;
        __syncthreads();
    }
    float best = -INFINITY;
    int bid = 0x7fffffff;
    for (int g0 = 0; g0 * 4 < V; g0 += SELECT_THREADS * 2) {
        float x[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int n = (g0 + (i >> 2) * SELECT_THREADS + tid) * 4 + (i & 3);
            x[i] = n < V ? score(n) : 0.f;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int g = g0 + h * SELECT_THREADS + tid;
            uint4 r = make_uint4(0u, 0u, 0u, 0u);
            bool drawn = false;
#pragma unroll
            for (int l = 0; l < 4; ++l) {
                const int n = g * 4 + l;
                const uint32_t k = order_key(x[h * 4 + l]);
                if (n >= V || k < key_k || k < key_p || (k == key_p && n < id_p)) continue;
                if (!drawn) { r = sample_philox(g, step, seed_lo, seed_hi); drawn = true; }
                const float v = gumbel_perturbed(x[h * 4 + l], mx, gumbel_e(philox_lane(r, l)));
                if (v > best || bid == 0x7fffffff) { best = v; bid = n; }
                if (kb) atomicOr(&kb[n >> 5], 1u << (n & 31));
            }
        }
    }
    const int tok = block_argmax(best, bid, s_v, s_i);
    if (tid == 0)
        select_commit(b, tok, pen_bitmap, pen_words, eos_ids, n_eos, max_new, first_pos, B, tokens, lengths, done, n_done, all_done, next_ids,
                      pos3);
}

// The per-id terms sample_select_kernel decides on, through the same helpers, for tests: for row b and id n (t = lengths[b])
//   score[b, n] = sample_score, row_max[b] = the row's maximum score, ex[b, n] = expf(score - max), mass[b, n] = mass_of_exp(ex),
//   bits[b, n] = lane n & 3 of the Philox block (seeds[b], n >> 2, t), e[b, n] = gumbel_e(bits), v[b, n] = gumbel_perturbed(score, max, e).
// Every row is written, finished or not (the maximum is exact in any order). One block per row.
constexpr int SAMPLE_TERMS_THREADS = 256;
__global__ void __launch_bounds__(SAMPLE_TERMS_THREADS) sample_terms_kernel(
        const __nv_bfloat16* __restrict__ logits, int V, const uint32_t* __restrict__ pen_bitmap, int pen_words, float penalty,
        const unsigned long long* __restrict__ seeds, float temperature, const int* __restrict__ lengths, float* __restrict__ score,
        float* __restrict__ row_max, float* __restrict__ ex, unsigned long long* __restrict__ mass, uint32_t* __restrict__ bits,
        float* __restrict__ e_out, float* __restrict__ v_out) {
    pdl_launch_dependents();
    __shared__ float s_m[SAMPLE_TERMS_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const __nv_bfloat16* lr = logits + (size_t)b * V;
    const uint32_t* pb = pen_bitmap ? pen_bitmap + (size_t)b * pen_words : nullptr;
    float mx = -INFINITY;
    for (int n = tid; n < V; n += SAMPLE_TERMS_THREADS) mx = fmaxf(mx, sample_score(lr, pb, penalty, temperature, n));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) s_m[tid >> 5] = mx;
    __syncthreads();
    for (int w = 0; w < SAMPLE_TERMS_THREADS / 32; ++w) mx = fmaxf(mx, s_m[w]);
    if (tid == 0) row_max[b] = mx;
    const uint32_t seed_lo = (uint32_t)seeds[b], seed_hi = (uint32_t)(seeds[b] >> 32);
    const int step = lengths[b];
    for (int n = tid; n < V; n += SAMPLE_TERMS_THREADS) {
        const size_t i = (size_t)b * V + n;
        const float x = sample_score(lr, pb, penalty, temperature, n), xe = expf(x - mx);
        const uint32_t u = philox_lane(sample_philox(n >> 2, step, seed_lo, seed_hi), n & 3);
        const float e = gumbel_e(u);
        score[i] = x; ex[i] = xe; mass[i] = mass_of_exp(xe); bits[i] = u; e_out[i] = e; v_out[i] = gumbel_perturbed(x, mx, e);
    }
}

// Answer log-probabilities of one generation step (the scores a rollout is scored on), one block per sequence, launched between the
// lm_head and greedy_select_kernel so the penalty bitmap is still the one this step's token was chosen under. The processed score of id n
// is that of the scoring path and topk_softmax_kernel: bf16 logit -> fp32 -> repetition penalty (bitmap) -> * inv_temp; over the full
// vocabulary, logp(n) = score(n) - max - log(sum exp(score - max)). With t = lengths[b] (the step's index), writes
// out_logp[b, t, j] = logp(answer_ids[b, j]) for j < answer_counts[b] (other entries untouched), and with top_k > 0 the top_k most probable
// ids and their probabilities to out_topk_ids / out_topk_probs[b, t, :] (ties to the lower id). A finished sequence returns at once.
// Each thread reads 8 logits (and their penalty words) before it consumes them, so a thread has 8 loads in flight.
constexpr int ANSWER_THREADS = 256, ANSWER_UNROLL = 8, ANSWER_TOPK_MAX = 8;
__global__ void __launch_bounds__(ANSWER_THREADS) answer_logprob_kernel(
        const __nv_bfloat16* __restrict__ logits, int V, const uint32_t* __restrict__ pen_bitmap, int pen_words, float penalty, float inv_temp,
        const int* __restrict__ answer_ids, const int* __restrict__ answer_counts, int n_max, int max_new, const int* __restrict__ lengths,
        const int* __restrict__ done, int top_k, float* __restrict__ out_logp, int* __restrict__ out_topk_ids, float* __restrict__ out_topk_probs) {
    pdl_launch_dependents();
    __shared__ float s_val[ANSWER_THREADS * ANSWER_TOPK_MAX];
    __shared__ int s_idx[ANSWER_THREADS * ANSWER_TOPK_MAX];
    __shared__ float s_red[2][ANSWER_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    if (done[b]) return;
    const __nv_bfloat16* lr = logits + (size_t)b * V;
    const uint32_t* pb = pen_bitmap ? pen_bitmap + (size_t)b * pen_words : nullptr;
    auto processed = [&](float x, uint32_t word, int n) {
        if ((word >> (n & 31)) & 1u) x = x < 0.f ? x * penalty : __fdiv_rn(x, penalty);
        return x * inv_temp;
    };
    float tv[ANSWER_TOPK_MAX];
    int ti[ANSWER_TOPK_MAX];
#pragma unroll
    for (int i = 0; i < ANSWER_TOPK_MAX; ++i) { tv[i] = -INFINITY; ti[i] = -1; }
    float mx = -INFINITY, sm = 0.f;
    for (int base = 0; base < V; base += ANSWER_THREADS * ANSWER_UNROLL) {
        float x[ANSWER_UNROLL];
        uint32_t w[ANSWER_UNROLL];
#pragma unroll
        for (int u = 0; u < ANSWER_UNROLL; ++u) {
            const int n = base + u * ANSWER_THREADS + tid;
            x[u] = n < V ? __bfloat162float(lr[n]) : 0.f;
            w[u] = (pb && n < V) ? pb[n >> 5] : 0u;
        }
#pragma unroll
        for (int u = 0; u < ANSWER_UNROLL; ++u) {
            const int n = base + u * ANSWER_THREADS + tid;      // ids rise along a thread's scan
            if (n >= V) break;
            const float v = processed(x[u], w[u], n);
            if (v > mx) { sm = sm * __expf(mx - v) + 1.f; mx = v; } else { sm += __expf(v - mx); }
            if (top_k > 0 && v > tv[ANSWER_TOPK_MAX - 1]) {     // sorted insert; strict > keeps the lower id first among equals
                int pos = ANSWER_TOPK_MAX - 1;
#pragma unroll
                for (int i = ANSWER_TOPK_MAX - 2; i >= 0; --i)
                    if (v > tv[i]) { tv[i + 1] = tv[i]; ti[i + 1] = ti[i]; pos = i; }
                tv[pos] = v; ti[pos] = n;
            }
        }
    }
    // block-wide max and sum of exps
    float bm = mx;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, o));
    if ((tid & 31) == 0) s_red[0][tid >> 5] = bm;
    __syncthreads();
    bm = s_red[0][0];
#pragma unroll
    for (int i = 1; i < ANSWER_THREADS / 32; ++i) bm = fmaxf(bm, s_red[0][i]);
    float bs = (mx == -INFINITY) ? 0.f : sm * __expf(mx - bm);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bs += __shfl_xor_sync(0xffffffffu, bs, o);
    if ((tid & 31) == 0) s_red[1][tid >> 5] = bs;
    if (top_k > 0) {
#pragma unroll
        for (int i = 0; i < ANSWER_TOPK_MAX; ++i) { s_val[tid * ANSWER_TOPK_MAX + i] = tv[i]; s_idx[tid * ANSWER_TOPK_MAX + i] = ti[i]; }
    }
    __syncthreads();
    float total = 0.f;
#pragma unroll
    for (int i = 0; i < ANSWER_THREADS / 32; ++i) total += s_red[1][i];
    const float lse = bm + logf(total);
    const int t = lengths[b];
    const size_t row = (size_t)b * max_new + t;
    const int cnt = min(answer_counts[b], n_max);
    for (int j = tid; j < cnt; j += ANSWER_THREADS) {
        const int id = answer_ids[(size_t)b * n_max + j];
        out_logp[row * n_max + j] = (id >= 0 && id < V) ? processed(__bfloat162float(lr[id]), pb ? pb[id >> 5] : 0u, id) - lse : -INFINITY;
    }
    if (top_k <= 0 || tid >= 32) return;
    // warp 0 picks the top_k of the 256 sorted lists: highest score, lower id on equal scores
    for (int k = 0; k < top_k; ++k) {
        float best = -INFINITY;
        int bpos = -1, bid = 0x7fffffff;
        for (int j = tid; j < ANSWER_THREADS * ANSWER_TOPK_MAX; j += 32) {
            const float v = s_val[j];
            const int id = s_idx[j];
            if (id >= 0 && (v > best || (v == best && id < bid))) { best = v; bpos = j; bid = id; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int op = __shfl_xor_sync(0xffffffffu, bpos, o), oid = __shfl_xor_sync(0xffffffffu, bid, o);
            if (ov > best || (ov == best && oid < bid)) { best = ov; bpos = op; bid = oid; }
        }
        if (tid == 0) {
            out_topk_ids[row * top_k + k] = bpos >= 0 ? bid : -1;
            out_topk_probs[row * top_k + k] = bpos >= 0 ? __expf(best - bm) / total : 0.f;
            if (bpos >= 0) s_idx[bpos] = -1;      // remove the winner
        }
        __syncwarp();
    }
}

}  // namespace vqa

// ------------------------------------------------------------------------------------------------ decode-loop launches (see clipt5.cuh)

// Generation state at the start of a prefill for B sequences of up to max_new tokens.
static int generate_init(Forward& f, int B, int max_new, int* tokens, int* lengths, int* done, int* n_done, int* all_done) {
    return f.launch(CAT_OTHER, 0, "generate init", generate_init_kernel, (B * max_new + 255) / 256, 256, 0, B, max_new, tokens, lengths, done,
                    n_done, all_done);
}

// The K and V heads of the packed rows qkv [rows = B * S, ld] into the cache (prefill: gen_len NULL; decode: S == 1).
static int kv_cache_write(Forward& f, const bf16* qkv, int ld, int k_col0, int v_col0, int Hkv, int S, long long rows, const int* seq_lens,
                          const int* gen_len, bf16* kc, bf16* vc, int cap) {
    return f.launch(CAT_OTHER, 0, "kv cache write", kv_cache_write_kernel, (unsigned)((rows * Hkv * 16 + 255) / 256), 256, 0, qkv, ld, k_col0,
                    v_col0, Hkv, S, rows, seq_lens, gen_len, kc, vc, cap);
}

// Key splits of decode_attn_partial_kernel over a cache of `cap` slots: enough for two CTAs per SM (at B = 1 the 4 KV heads alone would
// occupy 4 of 132 SMs), at least 16 keys each. Fixed by the capacity, not the live lengths, so a step's launch shapes never change.
static int decode_attn_splits(int B, int kv_heads, int cap, int num_sms) {
    return std::max(1, std::min((2 * num_sms + B * kv_heads - 1) / (B * kv_heads), (cap + 15) / 16));
}

// the group sizes (q heads per KV head) launch_decode_attn instantiates
static bool decode_attn_group_supported(int G) { return G == 1 || G == 2 || G == 4 || G == 5 || G == 7 || G == 8; }

// decode_attn_partial_kernel for G q heads per KV head (the group sizes of the Qwen2.5-VL family: 7B 7, 3B 8, 32B 5, 72B 8)
template <typename... Args>
static cudaError_t launch_decode_attn(int G, dim3 grid, cudaStream_t st, Args... args) {
    switch (G) {
        case 1: decode_attn_partial_kernel<1><<<grid, 32 * DEC_ATTN_WARPS, 0, st>>>(args...); break;
        case 2: decode_attn_partial_kernel<2><<<grid, 32 * DEC_ATTN_WARPS, 0, st>>>(args...); break;
        case 4: decode_attn_partial_kernel<4><<<grid, 32 * DEC_ATTN_WARPS, 0, st>>>(args...); break;
        case 5: decode_attn_partial_kernel<5><<<grid, 32 * DEC_ATTN_WARPS, 0, st>>>(args...); break;
        case 7: decode_attn_partial_kernel<7><<<grid, 32 * DEC_ATTN_WARPS, 0, st>>>(args...); break;
        case 8: decode_attn_partial_kernel<8><<<grid, 32 * DEC_ATTN_WARPS, 0, st>>>(args...); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// Flash-decoding attention of the query rows q [B, ldq] over the cache: `splits` key ranges of ceil(cap / splits) slots into the fp32 partials
// part_o [B * Hq * splits, 128] and part_ml [B * Hq * splits, 2], then their merge into out [B, ldo].
static int decode_attention(Forward& f, const bf16* q, int ldq, const bf16* kc, const bf16* vc, int cap, const int* seq_lens, const int* gen_len,
                            int B, int Hq, int Hkv, float scale, int splits, float* part_o, float* part_ml, bf16* out, int ldo) {
    const double kv_bytes = 2.0 * B * Hkv * (double)cap * 128 * 2;      // upper bound: the full capacity
    return f.op(CAT_ATTENTION, 4.0 * B * Hq * (double)cap * 128, kv_bytes, 2, "decode attention", [&] {
        cudaError_t e = launch_decode_attn(Hq / Hkv, dim3(splits, Hkv, B), f.st, q, ldq, kc, vc, cap, seq_lens, gen_len, Hkv,
                                           (cap + splits - 1) / splits, scale, part_o, part_ml);
        if (e != cudaSuccess) return e;
        decode_attn_merge_kernel<<<B * Hq, 128, 0, f.st>>>(part_o, part_ml, splits, out, ldo, Hq);
        return cudaGetLastError();
    });
}

// The answer log-probabilities of one step of a scored rollout from the step's bf16 logits [B, V] (penalty bitmap NULL = none).
static int answer_logprob(Forward& f, const bf16* logits, int B, int V, const uint32_t* pen_bitmap, float penalty, const vqa_qwen25vl_answer_score& s,
                          int max_new, const int* lengths, const int* done) {
    return f.launch(CAT_OTHER, 0, "answer logprob", answer_logprob_kernel, B, ANSWER_THREADS, 0, logits, V, pen_bitmap, (V + 31) / 32, penalty,
                    1.0f / s.temperature, s.answer_ids, s.answer_counts, s.n_max, max_new, lengths, done, s.top_k, s.out_logp, s.out_topk_ids,
                    s.out_topk_probs);
}

// The greedy token of every unfinished sequence and its bookkeeping (penalty bitmap NULL = none; first_pos / pos3 NULL = no positions).
static int greedy_select(Forward& f, const bf16* logits, int B, int V, uint32_t* pen_bitmap, float penalty, const int* eos_ids, int n_eos,
                         int max_new, const int* first_pos, int* tokens, int* lengths, int* done, int* n_done, int* all_done, int* next_ids,
                         int* pos3) {
    return f.launch(CAT_OTHER, 0, "greedy select", greedy_select_kernel, B, SELECT_THREADS, 0, logits, V, pen_bitmap, (V + 31) / 32, penalty,
                    eos_ids, n_eos, max_new, first_pos, B, tokens, lengths, done, n_done, all_done, next_ids, pos3);
}

// The sampled token of every unfinished sequence under `s` and the same bookkeeping as greedy_select (kept: see sample_select_kernel).
static int sample_select(Forward& f, const bf16* logits, int B, int V, uint32_t* pen_bitmap, float penalty, const vqa_qwen25vl_sampling& s,
                         const int* eos_ids, int n_eos, int max_new, const int* first_pos, int* tokens, int* lengths, int* done, int* n_done,
                         int* all_done, int* next_ids, int* pos3, uint32_t* kept = nullptr) {
    return f.launch(CAT_OTHER, 0, "sample select", sample_select_kernel, B, SELECT_THREADS, 0, logits, V, pen_bitmap, (V + 31) / 32, penalty,
                    (const unsigned long long*)s.seeds, s.temperature, s.top_k, s.top_p, eos_ids, n_eos, max_new, first_pos, B, tokens,
                    lengths, done, n_done, all_done, next_ids, pos3, kept);
}

// The per-id terms of sample_select's draw for rows [0, B) at steps lengths[b] (tests; see sample_terms_kernel), each output [B, V]
// except row_max [B].
static int sample_terms(Forward& f, const bf16* logits, int B, int V, const uint32_t* pen_bitmap, float penalty, const vqa_qwen25vl_sampling& s,
                        const int* lengths, float* score, float* row_max, float* ex, unsigned long long* mass, uint32_t* bits, float* e,
                        float* v) {
    return f.launch(CAT_OTHER, 0, "sample terms", sample_terms_kernel, B, SAMPLE_TERMS_THREADS, 0, logits, V, pen_bitmap, (V + 31) / 32,
                    penalty, (const unsigned long long*)s.seeds, s.temperature, lengths, score, row_max, ex, mass, bits, e, v);
}

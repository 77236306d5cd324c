// wgmma flash attention for sm_90a. head_dim 64 runs the persistent warp-specialised attn64_ws_kernel (described at its definition).
// head_dim 128 runs attn_wgmma_kernel: one CTA = one 128-query tile of one (sequence, head); two warpgroups own 64 query rows each, and
// the score tile never leaves the registers:
//
//   thread 0       TMA : Q once, then K/V tiles (128 keys x head_dim) through a 2-stage shared-memory ring
//   warpgroup w    S = Q K^T    wgmma m64n128k16, both operands K-major in 128B-swizzled shared memory
//                  softmax      online (running row maximum, rescale of O and l per key tile), exp2 on the MUFU
//                  O += P V     wgmma m64n{64,128}k16, P from registers (bf16, the accumulator layout of S), V MN-major from shared memory
//                  O / l -> HBM
//
// head_dim 64: T5 encoder self-attention with relative-position bias + key padding mask, CLIP ViT self-attention with 1/sqrt(d) scale.
// Replaces the eager attention of transformers/models/t5/modeling_t5.py:308-334 (which materialises [B,H,S,S] scores in HBM) and
// transformers/models/clip/modeling_clip.py:261-336.
// head_dim 128: Qwen2.5-VL language model (causal GQA) and vision tower (windows / whole frames, 80-wide heads zero-padded to 128),
// variable-length sequences (cu_seqlens) or fixed stride S.
#pragma once
#include "ptx.cuh"
#include "gemm_sm90.cuh"   // tmap_bf16_2d_cached, PerDeviceOnce

namespace vqa {

// launch with the programmatic-stream-serialisation attribute (the kernel calls pdl_wait() before its first global access)
template <typename Kernel, typename... Args>
inline cudaError_t launch_pdl(Kernel kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, args...);
}

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct AttnParams {
    __nv_bfloat16* o;          // [rows, ldo], column h * o_head_stride + d
    int ldo;
    const int* cu_seqlens;     // [n_seq + 1] row offsets (varlen) or nullptr
    const int* seq_lens;       // [n_seq] valid rows (fixed-stride mode) or nullptr
    int S;                     // fixed-stride mode: rows per sequence
    int q_col0, k_col0, v_col0;
    int kv_group;              // query heads per key/value head (GQA); 1 for MHA
    float scale_log2e;
    int o_head_stride, d_out;  // only the first d_out (multiple of 8) head dims are written
                               // (heads stored zero-padded to 128 in qkv produce d_out real output columns: the projection then contracts over them only)
    int pair, n_seq;           // varlen mode, pair != 0: CTA z covers the two consecutive sequences 2z and 2z+1 (each <= 64 rows) as ONE 128-row
                               // tile with a block-diagonal mask -- the 64-token windows of the Qwen2.5-VL vision tower (modeling_qwen2_5_vl.py
                               // get_window_index: 112-px windows = 8x8 patches) otherwise fill half of a tile and double the CTA count
    const int* kv_prefix;      // varlen mode, [n_seq] or nullptr: sequence b additionally attends to ALL rows of sequence kv_prefix[b] (>= 0),
                               // placed in front of its own keys -- the shared [system + vision] prefix of several prompts over one image:
                               // its K/V rows are computed once and read by every prompt's suffix
};

constexpr int AT_THREADS = 256;

template <int D>
struct AttnSmem {
    static constexpr int TILE = 128 * D * 2;   // Q, K or V tile: 128 rows x D bf16 as D/64 column blocks of 128 x 64
    static constexpr int BLOCK = 128 * 64 * 2;
    static size_t bytes() { return 1024 + 5 * (size_t)TILE + 64; }
};

template <int D, bool CAUSAL>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnParams p) {
    pdl_launch_dependents();
    pdl_wait();      // cu_seqlens / seq_lens / qkv are outputs of earlier kernels
    using Sm = AttnSmem<D>;
    constexpr int NB = D / 64;                  // 64-column blocks of a head
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int kvh = h / p.kv_group;
    int row_base, len, write_rows, mid = 0;
    if (p.cu_seqlens && p.pair) {
        row_base = p.cu_seqlens[2 * b];
        mid = p.cu_seqlens[2 * b + 1] - row_base;                       // rows [0, mid): first sequence, [mid, len): second (absent for an odd tail)
        len = p.cu_seqlens[min(2 * b + 2, p.n_seq)] - row_base;
        write_rows = len;
    } else if (p.cu_seqlens) {
        row_base = p.cu_seqlens[b];
        len = p.cu_seqlens[b + 1] - row_base;
        write_rows = len;                       // rows past the sequence belong to the next one
    } else {
        row_base = b * p.S;
        len = p.seq_lens ? min(p.seq_lens[b], p.S) : p.S;
        write_rows = p.S;                       // padded rows of this sequence get zeros
    }
    const int q0 = qt * 128;
    if (q0 >= write_rows) return;
    if (q0 >= len) {
        for (int i = threadIdx.x; i < 128 * (D / 8); i += blockDim.x) {
            const int r = i / (D / 8), c = i % (D / 8);
            if (q0 + r < write_rows && c * 8 < p.d_out)
                *reinterpret_cast<uint4*>(p.o + (size_t)(row_base + q0 + r) * p.ldo + h * p.o_head_stride + c * 8) = make_uint4(0, 0, 0, 0);
        }
        return;
    }
    extern __shared__ uint8_t at_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = smem + Sm::TILE;        // [2]
    uint8_t* sV = smem + 3 * Sm::TILE;    // [2]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * Sm::TILE);
    uint64_t* q_full = bars;
    uint64_t* kv_full = bars + 1;         // [2]

    // key tiles: first the nA tiles of the shared prefix sequence (all of it visible), then this sequence's own tiles (causal)
    int pre_base = 0, pre_len = 0;
    if (p.kv_prefix && p.cu_seqlens) {
        const int ps = p.kv_prefix[b];
        if (ps >= 0) { pre_base = p.cu_seqlens[ps]; pre_len = p.cu_seqlens[ps + 1] - pre_base; }
    }
    const int nA = (pre_len + 127) / 128;
    int nkt_own = (len + 127) / 128;
    if (CAUSAL) nkt_own = min(nkt_own, qt + 1);
    const int nkt = nA + nkt_own;

    auto load_kv = [&](int j) {
        const int st = j & 1;
        mbar_arrive_expect_tx(&kv_full[st], 2 * Sm::TILE);
        const int r = j < nA ? pre_base + j * 128 : row_base + (j - nA) * 128;
#pragma unroll
        for (int c = 0; c < NB; ++c) {
            tma_load_2d(sK + st * Sm::TILE + c * Sm::BLOCK, &tmap_qkv, &kv_full[st], p.k_col0 + kvh * D + c * 64, r);
            tma_load_2d(sV + st * Sm::TILE + c * Sm::BLOCK, &tmap_qkv, &kv_full[st], p.v_col0 + kvh * D + c * 64, r);
        }
    };
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_qkv);
        mbar_init(q_full, 1);
        mbar_init(&kv_full[0], 1);
        mbar_init(&kv_full[1], 1);
        fence_barrier_init();
        mbar_arrive_expect_tx(q_full, Sm::TILE);
#pragma unroll
        for (int c = 0; c < NB; ++c) tma_load_2d(sQ + c * Sm::BLOCK, &tmap_qkv, q_full, p.q_col0 + h * D + c * 64, row_base + q0);
        load_kv(0);
    }
    __syncthreads();

    const int wg = threadIdx.x >> 7;
    const int tid = threadIdx.x & 127;
    const int lane = tid & 31;
    // this thread's rows of the tile (accumulator layout): r0 and r0 + 8; columns 8j + c0 + {0, 1}
    const int r0 = wg * 64 + (tid >> 5) * 16 + (lane >> 2);
    const int c0 = (lane & 3) * 2;
    const int qrow[2] = {q0 + r0, q0 + r0 + 8};

    float o_acc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o_acc[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    mbar_wait(q_full, 0);
    for (int j = 0; j < nkt; ++j) {
        // every thread is done with tile j - 1: its K/V slot takes tile j + 1
        if (j > 0) __syncthreads();
        if (threadIdx.x == 0 && j + 1 < nkt) load_kv(j + 1);
        const int st = j & 1;
        mbar_wait(&kv_full[st], ((uint32_t)j >> 1) & 1u);

        float s[64];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; ++k) {
            const uint64_t qd = make_sw128_desc(smem_u32(sQ + (k >> 2) * Sm::BLOCK + wg * 64 * 128)) + 2 * (k & 3);
            const uint64_t kd = make_sw128_desc(smem_u32(sK + st * Sm::TILE + (k >> 2) * Sm::BLOCK)) + 2 * (k & 3);
            wgmma_ss<128>(s, qd, kd, k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);

        const bool in_prefix = j < nA;
        const int k0 = in_prefix ? j * 128 : (j - nA) * 128;
        const int klen = in_prefix ? pre_len : len;
        const bool diag = CAUSAL && !in_prefix && (j - nA) == qt;
        const bool edge = (k0 + 128 > klen) || diag || p.pair;
        float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            const int hr = (i >> 1) & 1;                         // row r0 (0) or r0 + 8 (1)
            const int kcol = k0 + (i >> 2) * 8 + c0 + (i & 1);
            float x = s[i] * p.scale_log2e;
            if (edge) {
                const int qr = qrow[hr] - q0;
                if (kcol >= klen || (diag && kcol > qrow[hr]) || (p.pair && ((kcol < mid) != (qr < mid)))) x = -INFINITY;
            }
            s[i] = x;
            tmax[hr] = fmaxf(tmax[hr], x);
        }
        // Exponent reference of a row: the maximum of its first key tile, raised only when a later tile exceeds it by more than 2^8 (P may
        // then exceed 1 -- harmless in bf16 / fp32, l carries the same factor). A fixed reference makes P independent of where the key
        // tiles are cut (a shared key prefix gives the same bf16 P as the unshared sequence) and skips most rescales of O.
        float corr[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            tmax[hr] = fmaxf(tmax[hr], __shfl_xor_sync(0xffffffffu, tmax[hr], 1));
            tmax[hr] = fmaxf(tmax[hr], __shfl_xor_sync(0xffffffffu, tmax[hr], 2));
            const float m_new = (m_run[hr] == -INFINITY || tmax[hr] > m_run[hr] + 8.f) ? tmax[hr] : m_run[hr];
            // a row that has seen no key yet keeps reference 0: its exponentials are exp2(-inf) = 0
            const float m_use = m_new == -INFINITY ? 0.f : m_new;
            corr[hr] = m_run[hr] == -INFINITY ? 0.f : fast_exp2(m_run[hr] - m_use);
            m_run[hr] = m_new;
            tmax[hr] = m_use;
            l_run[hr] *= corr[hr];
        }
#pragma unroll
        for (int i = 0; i < D / 2; ++i) o_acc[i] *= corr[(i >> 1) & 1];
        // P = exp2(x - m) as bf16 pairs in the A-operand layout of the P.V wgmma; l sums the unrounded exponentials
        uint32_t pk[32];
        float lsum[2] = {0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int hr = (i >> 1) & 1;
            const float e0 = fast_exp2(s[i] - tmax[hr]), e1 = fast_exp2(s[i + 1] - tmax[hr]);
            lsum[hr] += e0 + e1;
            pk[i >> 1] = pack_bf16x2(e0, e1);
        }
        l_run[0] += lsum[0];
        l_run[1] += lsum[1];

        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            // keys [16 kk, 16 kk + 16): V rows 16 kk.. = two 8-row groups of 1 KB; head-dim blocks of 64 are Sm::BLOCK apart (LBO)
            const uint64_t vd = make_sw128_desc(smem_u32(sV + st * Sm::TILE + kk * 2048), Sm::BLOCK);
            const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
            wgmma_rs_tb<D>(o_acc, a, vd, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o_acc);
    }

    // ---- epilogue: O / l (row sums reduced over the four threads of a row)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 1);
        l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 2);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int qr = qrow[hr];
        const float inv = (qr < len && l_run[hr] > 0.f) ? 1.f / l_run[hr] : 0.f;
        if (qr < write_rows) {
            __nv_bfloat16* orow = p.o + (size_t)(row_base + qr) * p.ldo + h * p.o_head_stride;
#pragma unroll
            for (int jb = 0; jb < D / 8; ++jb) {
                const int col = jb * 8 + c0;
                if (jb * 8 < p.d_out)      // rows at or past len: +0 (O * 0 would be -0 where O < 0)
                    *reinterpret_cast<uint32_t*>(orow + col) =
                        qr < len ? pack_bf16x2(o_acc[jb * 4 + 2 * hr] * inv, o_acc[jb * 4 + 2 * hr + 1] * inv) : 0u;
            }
        }
    }
}

// Raises KERNEL's dynamic shared-memory limit to smem once per device.
template <auto KERNEL>
inline cudaError_t allow_smem(size_t smem) {
    static std::atomic<size_t> max_set[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (smem > max_set[dev & 63].load(std::memory_order_acquire)) {
        e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        max_set[dev & 63].store(smem, std::memory_order_release);
    }
    return cudaSuccess;
}

template <int D, bool CAUSAL>
inline cudaError_t launch_attn_t(const CUtensorMap& tm, const AttnParams& p, dim3 grid, size_t smem, cudaStream_t stream) {
    constexpr auto kernel = attn_wgmma_kernel<D, CAUSAL>;
    const cudaError_t e = allow_smem<kernel>(smem);
    if (e != cudaSuccess) return e;
    return launch_pdl(kernel, grid, dim3(AT_THREADS), smem, stream, tm, p);
}

// ================================================================ head_dim 64: persistent, warp-specialised
// T5 encoder self-attention (relative-position bias, key padding mask) and CLIP ViT self-attention (1/sqrt(d) scale), fixed stride S.
// A work item is one 128-query tile of one (sample, head); items are numbered head-major (head, sample, query tile) and each CTA (about one
// per SM) takes a contiguous run of them, so consecutive items share K/V in L2 and the head's bias row in shared memory.
//
//   warp 0 of warpgroup 0   TMA producer: Q of the next item (2 slots), then K/V tiles of 128 keys through a ring of up to
//                           A64_MAX_STAGES stages (fewer when a long bias row needs the space) with full / empty mbarriers. Gives up its registers (setmaxnreg) to the consumers.
//   warpgroups 1, 2         consumers, 64 query rows of the item each. Per key tile j: S_j = Q K_j^T is issued before O += P_{j-1} V_{j-1},
//                           and the softmax of S_j runs while that P.V wgmma is in flight (FlashAttention-3's intra-warpgroup overlap). The
//                           two consumer warpgroups are not synchronised with each other, so one's softmax also runs under the other's wgmma.
//
// Arithmetic per score and per row is the one of attn_wgmma_kernel before the split (bit-identical output): 128-wide key tiles from key 0,
// exponent reference = first tile's row maximum (raised only past 2^8), score x = fmaf(s, scale log2e, bias log2e) or, with ROUND,
// bf16(bf16(s) + bf16(bias)) * scale log2e, P = ex2(x - m) packed to bf16, l summed pairwise from the unrounded exponentials, O * (1/l).
// Only work whose result is exactly known is skipped:
//   - the softmax of the last key tile covers its valid width rounded up to 32 keys and writes P = 0 for the rest. Its wgmmas keep the full
//     width: a wgmma chosen at run time makes ptxas serialise every wgmma of the kernel (C7520), which costs far more than the dead columns;
//   - a consumer whose 64 rows all lie at or past the sequence length only writes zero rows;
//   - with bias_const_from = C > 0 the caller promises that the table is constant for key - query >= C and for key - query <= -C: a
//     (64-row, key tile) block wholly on one side uses that single value instead of a per-score lookup.
//
// ROUND: the reference's eager attention produces bf16 tensors before its fp32 softmax (modeling_t5.py:308-331: `scores = matmul(q, k^T)` is a
// bf16 tensor, `scores += position_bias` a bf16 add; modeling_clip.py: bf16 matmul * 2^-3). With |score| ~ 10 that rounding moves the exponent's
// argument by up to 0.04, far more than any other rounding on the path, so parity needs the same values: x = bf16(s), x = bf16(x + bf16(bias)),
// exponent x * scale * log2(e). Without ROUND: s * scale * log2(e) + bias * log2(e).
struct Attn64Params {
    __nv_bfloat16* o;          // [B*S, ldo], column h * 64 + d
    int ldo;
    const int* seq_lens;       // [B] valid rows or nullptr (all S)
    int B, S, H, n_qt;         // n_qt = ceil(S / 128) query tiles per (sample, head)
    int q_col0, k_col0, v_col0;
    float scale_log2e;
    const float* bias_table;   // [H, 2S-1] fp32 relative-position bias (natural-log domain, index key - query + S - 1) or nullptr
    int bias_const_from;       // see above; 0: every tile reads the table
    int stages;                // K/V ring depth (2..A64_MAX_STAGES)
};

constexpr int A64_THREADS = 384;
constexpr int A64_MAX_STAGES = 4;
constexpr int A64_TILE = 128 * 64 * 2;   // Q, K or V tile: 128 rows x 64 bf16, 128B-swizzled
// The head's bias row is staged with A64_BIAS_PAD copies of its first / last entry on either side: every (query row, key column) of a tile,
// padding included, lies within [-127, 2S + 125] of index key - query + S - 1, so a score reads its bias without clamping the index.
constexpr int A64_BIAS_PAD = 128;

constexpr size_t A64_SMEM_MAX = 227 * 1024;   // dynamic shared memory of one CTA on sm_90

constexpr size_t attn64_smem_bytes(int stages, int bias_entries) {
    return 1024 + (2 + 2 * (size_t)stages) * A64_TILE + 128 + (size_t)bias_entries * 4;
}

// The longest S whose padded bias row (2S - 1 + 2 A64_BIAS_PAD floats) fits next to a K/V ring of `stages` stages. A bias table longer than
// the 2-stage limit does not fit at all.
constexpr int attn64_max_bias_len(int stages) {
    return (int)(((A64_SMEM_MAX - attn64_smem_bytes(stages, 0)) / 4 + 1 - 2 * A64_BIAS_PAD) / 2);
}

// S = Q K^T for a 128-key tile
__device__ __forceinline__ void attn64_qk(float (&s)[64], uint32_t q_addr, uint32_t k_addr) {
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<128>(s, make_sw128_desc(q_addr) + 2 * k, make_sw128_desc(k_addr) + 2 * k, k > 0 ? 1u : 0u);
}

// O += P V for a 128-key tile
__device__ __forceinline__ void attn64_pv(float (&o)[32], const uint32_t (&pk)[32], uint32_t v_addr) {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
        const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
        wgmma_rs_tb<64>(o, a, make_sw128_desc(v_addr + kk * 2048, A64_TILE), 1u);
    }
}

// Scores of one key tile -> exponentials in s, updates the row state (m, l) and returns the factor O must be rescaled by. Only the first NW
// keys of the tile can be valid: the other exponentials are exactly 0 and are written as such. CB: the whole block uses the single bias value cb.
// EDGE: the tile reaches past len, keys at or past it are masked. sBias: the padded row (A64_BIAS_PAD).
template <bool HAS_BIAS, bool ROUND, int NW, bool CB, bool EDGE>
__device__ __forceinline__ void attn64_softmax(float (&s)[64], int k0, int len, const int (&qrow)[2], int c0, const float* sBias, int S,
                                               float cb, float scale_log2e, float (&m_run)[2], float (&l_run)[2], float (&corr)[2]) {
    // bias of (row hr, column 8 (i / 4) + c0 + (i & 1)) = brow[hr][8 (i / 4) + (i & 1)]: a compile-time offset from a per-row base
    const float* brow[2] = {sBias + (k0 + c0 - qrow[0] + S - 1 + A64_BIAS_PAD), sBias + (k0 + c0 - qrow[1] + S - 1 + A64_BIAS_PAD)};
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) {
        const int hr = (i >> 1) & 1;
        const int kcol = k0 + (i >> 2) * 8 + c0 + (i & 1);
        float x = s[i];
        if constexpr (HAS_BIAS) {
            const float bv = CB ? cb : brow[hr][(i >> 2) * 8 + (i & 1)];
            if constexpr (ROUND) x = __bfloat162float(__hadd(__float2bfloat16_rn(x), __float2bfloat16_rn(bv)));
            else                 x = fmaf(x, scale_log2e, bv);
        } else if constexpr (ROUND) {
            x = bf16_round(x);
        }
        if constexpr (ROUND) x *= scale_log2e;
        else if (!HAS_BIAS) x *= scale_log2e;
        if (EDGE && kcol >= len) x = -INFINITY;
        s[i] = x;
        tmax[hr] = fmaxf(tmax[hr], x);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        tmax[hr] = fmaxf(tmax[hr], __shfl_xor_sync(0xffffffffu, tmax[hr], 1));
        tmax[hr] = fmaxf(tmax[hr], __shfl_xor_sync(0xffffffffu, tmax[hr], 2));
        const float m_new = (m_run[hr] == -INFINITY || tmax[hr] > m_run[hr] + 8.f) ? tmax[hr] : m_run[hr];
        const float m_use = m_new == -INFINITY ? 0.f : m_new;
        corr[hr] = m_run[hr] == -INFINITY ? 0.f : fast_exp2(m_run[hr] - m_use);
        m_run[hr] = m_new;
        tmax[hr] = m_use;
        l_run[hr] *= corr[hr];
    }
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < NW / 2; i += 2) {
        const int hr = (i >> 1) & 1;
        const float e0 = fast_exp2(s[i] - tmax[hr]), e1 = fast_exp2(s[i + 1] - tmax[hr]);
        lsum[hr] += e0 + e1;
        s[i] = e0;
        s[i + 1] = e1;
    }
#pragma unroll
    for (int i = NW / 2; i < 64; ++i) s[i] = 0.f;
    l_run[0] += lsum[0];
    l_run[1] += lsum[1];
}

template <bool HAS_BIAS, bool ROUND, int NW, bool EDGE>
__device__ __forceinline__ void attn64_softmax_cb(bool cb_on, float (&s)[64], int k0, int len, const int (&qrow)[2], int c0, const float* sBias,
                                                  int S, float cb, float scale_log2e, float (&m_run)[2], float (&l_run)[2], float (&corr)[2]) {
    if (HAS_BIAS && cb_on) attn64_softmax<HAS_BIAS, ROUND, NW, true, EDGE>(s, k0, len, qrow, c0, sBias, S, cb, scale_log2e, m_run, l_run, corr);
    else                   attn64_softmax<HAS_BIAS, ROUND, NW, false, EDGE>(s, k0, len, qrow, c0, sBias, S, cb, scale_log2e, m_run, l_run, corr);
}

// nw: valid keys of the tile rounded up to 32 (128 for every tile but the last)
template <bool HAS_BIAS, bool ROUND>
__device__ __forceinline__ void attn64_softmax_any(int nw, bool cb_on, float (&s)[64], int k0, int len, const int (&qrow)[2], int c0,
                                                   const float* sBias, int S, float cb, float scale_log2e, float (&m_run)[2], float (&l_run)[2],
                                                   float (&corr)[2]) {
    if (k0 + 128 <= len) attn64_softmax_cb<HAS_BIAS, ROUND, 128, false>(cb_on, s, k0, len, qrow, c0, sBias, S, cb, scale_log2e, m_run, l_run, corr);
    else if (nw == 128)  attn64_softmax_cb<HAS_BIAS, ROUND, 128, true>(cb_on, s, k0, len, qrow, c0, sBias, S, cb, scale_log2e, m_run, l_run, corr);
    else if (nw == 96)   attn64_softmax_cb<HAS_BIAS, ROUND, 96, true>(cb_on, s, k0, len, qrow, c0, sBias, S, cb, scale_log2e, m_run, l_run, corr);
    else if (nw == 64)   attn64_softmax_cb<HAS_BIAS, ROUND, 64, true>(cb_on, s, k0, len, qrow, c0, sBias, S, cb, scale_log2e, m_run, l_run, corr);
    else                 attn64_softmax_cb<HAS_BIAS, ROUND, 32, true>(cb_on, s, k0, len, qrow, c0, sBias, S, cb, scale_log2e, m_run, l_run, corr);
}

template <bool HAS_BIAS, bool ROUND>
__global__ void __launch_bounds__(A64_THREADS, 1)
attn64_ws_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const Attn64Params p) {
    pdl_launch_dependents();
    extern __shared__ uint8_t at_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;                                  // [2]
    uint8_t* sK = smem + 2 * A64_TILE;                   // [stages]
    uint8_t* sV = sK + p.stages * A64_TILE;              // [stages]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + p.stages * A64_TILE);
    uint64_t* q_full = bars;                             // [2]
    uint64_t* q_empty = bars + 2;                        // [2]
    uint64_t* kv_full = bars + 4;                        // [A64_MAX_STAGES]
    uint64_t* kv_empty = bars + 4 + A64_MAX_STAGES;      // [A64_MAX_STAGES]
    // HAS_BIAS: the current head's 2S-1 biases padded by A64_BIAS_PAD on either side (ROUND: rounded to bf16), times log2(e) unless ROUND.
    // Addressed from the __shared__ array itself so that its reads compile to LDS with immediate offsets.
    const uint32_t align_pad = (1024u - (smem_u32(at_smem_raw) & 1023u)) & 1023u;
    float* sBias = reinterpret_cast<float*>(at_smem_raw + align_pad + (2 + 2 * p.stages) * A64_TILE + 16 * sizeof(uint64_t));

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_qkv);
        for (int i = 0; i < 2; ++i) { mbar_init(&q_full[i], 1); mbar_init(&q_empty[i], 8); }
        for (int i = 0; i < p.stages; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }   // empty: one arrive per consumer warp
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();      // seq_lens / the bias table / qkv are outputs of earlier kernels

    const int per_b = p.n_qt, per_h = p.B * p.n_qt;
    const long long n_items = (long long)p.H * per_h;
    const int t_begin = (int)(n_items * blockIdx.x / gridDim.x), t_end = (int)(n_items * (blockIdx.x + 1) / gridDim.x);
    auto item = [&](int t, int& b, int& h, int& q0, int& len) {
        h = t / per_h;
        const int r = t - h * per_h;
        b = r / per_b;
        q0 = (r - b * per_b) * 128;
        len = p.seq_lens ? min(p.seq_lens[b], p.S) : p.S;
    };
    const int wg = threadIdx.x >> 7;

    if (wg == 0) {
        regs_dealloc<24>();
        if (threadIdx.x != 0) return;
        int st = 0, qs = 0;
        uint32_t kph = 0, qph = 0;
        for (int t = t_begin; t < t_end; ++t) {
            int b, h, q0, len;
            item(t, b, h, q0, len);
            if (q0 >= len) continue;
            const int row_base = b * p.S;
            mbar_wait(&q_empty[qs], qph ^ 1u);
            mbar_arrive_expect_tx(&q_full[qs], A64_TILE);
            tma_load_2d(sQ + qs * A64_TILE, &tmap_qkv, &q_full[qs], p.q_col0 + h * 64, row_base + q0);
            if (++qs == 2) { qs = 0; qph ^= 1u; }
            const int nkt = (len + 127) / 128;
            for (int j = 0; j < nkt; ++j) {
                mbar_wait(&kv_empty[st], kph ^ 1u);
                mbar_arrive_expect_tx(&kv_full[st], 2 * A64_TILE);
                tma_load_2d(sK + st * A64_TILE, &tmap_qkv, &kv_full[st], p.k_col0 + h * 64, row_base + j * 128);
                tma_load_2d(sV + st * A64_TILE, &tmap_qkv, &kv_full[st], p.v_col0 + h * 64, row_base + j * 128);
                if (++st == p.stages) { st = 0; kph ^= 1u; }
            }
        }
        return;
    }

    regs_alloc<240>();
    const int cw = wg - 1;                   // rows [64 cw, 64 cw + 64) of every item
    const int tid = threadIdx.x & 127;
    const int lane = tid & 31;
    // this thread's rows of the item (accumulator layout): r0 and r0 + 8; columns 8j + c0 + {0, 1}
    const int r0 = cw * 64 + (tid >> 5) * 16 + (lane >> 2);
    const int c0 = (lane & 3) * 2;
    const int width = 2 * p.S - 1;
    int st = 0, qs = 0, bias_h = -1;
    uint32_t kph = 0, qph = 0;

    for (int t = t_begin; t < t_end; ++t) {
        int b, h, q0, len;
        item(t, b, h, q0, len);
        const int row_base = b * p.S;
        const int qrow[2] = {q0 + r0, q0 + r0 + 8};
        auto store_rows = [&](const float (&o)[32], const float (&inv)[2]) {
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                const int qr = qrow[hr];
                if (qr >= p.S) continue;
                __nv_bfloat16* orow = p.o + (size_t)(row_base + qr) * p.ldo + h * 64;
#pragma unroll
                for (int jb = 0; jb < 8; ++jb)
                    *reinterpret_cast<uint32_t*>(orow + jb * 8 + c0) =
                        qr < len ? pack_bf16x2(o[jb * 4 + 2 * hr] * inv[hr], o[jb * 4 + 2 * hr + 1] * inv[hr]) : 0u;
            }
        };
        float o_acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
        float l_run[2] = {0.f, 0.f};
        if (q0 >= len) {                      // no valid query row: nothing was loaded for this item
            store_rows(o_acc, l_run);
            continue;
        }
        if constexpr (HAS_BIAS) {
            if (h != bias_h) {                // both consumer warpgroups walk the same items: they agree on when the head changes
                named_bar_sync(1, 256);       // the other warpgroup is done with the previous head's row
                const float* src = p.bias_table + (size_t)h * width;
                for (int x = threadIdx.x - 128; x < width + 2 * A64_BIAS_PAD; x += 256) {
                    const float v = __ldg(src + min(max(x - A64_BIAS_PAD, 0), width - 1));
                    sBias[x] = ROUND ? bf16_round(v) : v * 1.4426950408889634f;
                }
                named_bar_sync(1, 256);
                bias_h = h;
            }
        }
        const int nkt = (len + 127) / 128;
        const int qb = q0 + cw * 64;
        if (qb >= len) {                      // this warpgroup's rows are all padding: release the item's slots unread
            if (lane == 0) {
                for (int j = 0; j < nkt; ++j) {
                    mbar_wait(&kv_full[st], kph);
                    mbar_arrive(&kv_empty[st]);
                    if (++st == p.stages) { st = 0; kph ^= 1u; }
                }
                mbar_wait(&q_full[qs], qph);
                mbar_arrive(&q_empty[qs]);
            } else {
                for (int j = 0; j < nkt; ++j)
                    if (++st == p.stages) { st = 0; kph ^= 1u; }
            }
            if (++qs == 2) { qs = 0; qph ^= 1u; }
            store_rows(o_acc, l_run);
            continue;
        }

        // valid keys of the tile starting at k0, rounded up to 32: the width the softmax covers
        auto tile_nw = [&](int k0) { const int w = min(128, len - k0); return w > 96 ? 128 : w > 64 ? 96 : w > 32 ? 64 : 32; };
        // the bias of a (64-row block, key tile) pair is one table value when every valid pair lies on one side past bias_const_from
        float cb = 0.f;
        auto const_bias = [&](int k0) {
            if (!HAS_BIAS || p.bias_const_from <= 0) return false;
            const int C = p.bias_const_from;
            const int kend = min(k0 + 128, len) - 1;
            if (k0 - (qb + 63) >= C) { cb = sBias[A64_BIAS_PAD + min(p.S - 1 + C, width - 1)]; return true; }
            if (kend - qb <= -C)     { cb = sBias[A64_BIAS_PAD + max(p.S - 1 - C, 0)]; return true; }
            return false;
        };

        float m_run[2] = {-INFINITY, -INFINITY}, corr[2];
        float s[64];
        uint32_t pk[32];
        mbar_wait(&q_full[qs], qph);
        const uint32_t q_addr = smem_u32(sQ + qs * A64_TILE + cw * 64 * 128);

        mbar_wait(&kv_full[st], kph);
        int nw = tile_nw(0);
        wgmma_fence();
        attn64_qk(s, q_addr, smem_u32(sK + st * A64_TILE));
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
        bool cb_on = const_bias(0);
        attn64_softmax_any<HAS_BIAS, ROUND>(nw, cb_on, s, 0, len, qrow, c0, sBias, p.S, cb, p.scale_log2e, m_run, l_run, corr);
        // o_acc is still zero: the first tile's rescale is a no-op
#pragma unroll
        for (int i = 0; i < 64; i += 2) pk[i >> 1] = pack_bf16x2(s[i], s[i + 1]);
        int pst = st;
        if (++st == p.stages) { st = 0; kph ^= 1u; }

        for (int j = 1; j < nkt; ++j) {
            const int k0 = j * 128;
            mbar_wait(&kv_full[st], kph);
            nw = tile_nw(k0);
            wgmma_fence();
            attn64_qk(s, q_addr, smem_u32(sK + st * A64_TILE));
            wgmma_commit();
            attn64_pv(o_acc, pk, smem_u32(sV + pst * A64_TILE));
            wgmma_commit();
            wgmma_wait<1>();                  // S_j is in the registers; O += P_{j-1} V_{j-1} may still run
            fence_regs(s);
            cb_on = const_bias(k0);
            attn64_softmax_any<HAS_BIAS, ROUND>(nw, cb_on, s, k0, len, qrow, c0, sBias, p.S, cb, p.scale_log2e, m_run, l_run, corr);
            wgmma_wait<0>();
            fence_regs(o_acc);
            fence_regs(s);
            if (lane == 0) mbar_arrive(&kv_empty[pst]);
            if (corr[0] != 1.f || corr[1] != 1.f) {   // the reference of both rows moved (x * 1 is exact: skipping it changes nothing)
#pragma unroll
                for (int i = 0; i < 32; ++i) o_acc[i] *= corr[(i >> 1) & 1];
            }
#pragma unroll
            for (int i = 0; i < 64; i += 2) pk[i >> 1] = pack_bf16x2(s[i], s[i + 1]);
            pst = st;
            if (++st == p.stages) { st = 0; kph ^= 1u; }
        }
        wgmma_fence();
        attn64_pv(o_acc, pk, smem_u32(sV + pst * A64_TILE));
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o_acc);
        if (lane == 0) {
            mbar_arrive(&kv_empty[pst]);
            mbar_arrive(&q_empty[qs]);
        }
        if (++qs == 2) { qs = 0; qph ^= 1u; }

        // ---- epilogue: O / l (row sums reduced over the four threads of a row); rows at or past len are written as zeros
        float inv[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 1);
            l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 2);
            inv[hr] = l_run[hr] > 0.f ? 1.f / l_run[hr] : 0.f;
        }
        store_rows(o_acc, inv);
    }
}

template <bool HAS_BIAS, bool ROUND>
inline cudaError_t launch_attn64(const CUtensorMap& tm, const Attn64Params& p, dim3 grid, size_t smem, cudaStream_t stream) {
    constexpr auto kernel = attn64_ws_kernel<HAS_BIAS, ROUND>;
    const cudaError_t e = allow_smem<kernel>(smem);
    if (e != cudaSuccess) return e;
    return launch_pdl(kernel, grid, dim3(A64_THREADS), smem, stream, tm, p);
}

inline int sm_count() {
    static std::atomic<int> count[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    int n = count[dev & 63].load(std::memory_order_relaxed);
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
        count[dev & 63].store(n, std::memory_order_relaxed);
    }
    return n;
}

// head_dim 64. qkv: packed [B*S, ld] buffer; q/k/v head 0 start at columns q_col0/k_col0/v_col0.
// bias_const_from > 0: the caller guarantees bias_table[h][.] is constant for key - query >= bias_const_from and for key - query <=
// -bias_const_from (T5: relative_attention_max_distance); 0 makes no assumption.
// round_scores: reproduce the bf16 tensors of the reference's eager attention (scores, scores + bias) before the fp32 softmax.
inline cudaError_t launch_attn_tc(const __nv_bfloat16* qkv, int ld, int q_col0, int k_col0, int v_col0, __nv_bfloat16* o, int ldo,
                                  int B, int S, int H, const int* seq_lens, const float* bias_table, float scale, int bias_const_from,
                                  bool round_scores, cudaStream_t stream) {
    CUtensorMap tm;
    if (!tmap_bf16_2d_cached(&tm, qkv, (uint64_t)B * S, (uint64_t)ld, (uint64_t)ld, 128)) return cudaErrorInvalidValue;
    Attn64Params p = {};
    p.o = o; p.ldo = ldo; p.seq_lens = seq_lens;
    p.B = B; p.S = S; p.H = H; p.n_qt = (int)((S + 127LL) / 128);
    p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.bias_table = bias_table;
    p.bias_const_from = bias_const_from > 0 ? bias_const_from : 0;
    const long long n_items = (long long)H * B * p.n_qt;
    if (n_items > INT32_MAX) return cudaErrorInvalidValue;
    // the deepest K/V ring that fits next to the bias row: 4 stages up to S = attn64_max_bias_len(4), then 3, then 2 up to
    // attn64_max_bias_len(2); longer sequences with a bias table do not fit at all
    if (bias_table && S > attn64_max_bias_len(2)) return cudaErrorInvalidValue;
    const int bias_entries = bias_table ? 2 * S - 1 + 2 * A64_BIAS_PAD : 0;
    p.stages = A64_MAX_STAGES;
    while (bias_table && p.stages > 2 && S > attn64_max_bias_len(p.stages)) --p.stages;
    const size_t smem = attn64_smem_bytes(p.stages, bias_entries);
    if (smem > A64_SMEM_MAX) return cudaErrorInvalidValue;
    const int sms = sm_count();
    if (sms <= 0) return cudaErrorInvalidDevice;
    const dim3 grid((unsigned)std::min<long long>(n_items, sms));
    if (bias_table) return round_scores ? launch_attn64<true, true>(tm, p, grid, smem, stream) : launch_attn64<true, false>(tm, p, grid, smem, stream);
    return round_scores ? launch_attn64<false, true>(tm, p, grid, smem, stream) : launch_attn64<false, false>(tm, p, grid, smem, stream);
}

// head_dim 128. rows: total rows of the packed buffer; max_len: longest sequence (grid sizing); kv_prefix: see AttnParams (varlen mode only)
inline cudaError_t launch_attn_tc128(const __nv_bfloat16* qkv, int ld, long long rows, int q_col0, int k_col0, int v_col0,
                                     __nv_bfloat16* o, int ldo, int n_seq, int max_len, int S, int Hq, int kv_group,
                                     const int* cu_seqlens, const int* seq_lens, float scale, bool causal, cudaStream_t stream,
                                     const int* kv_prefix = nullptr, bool pair_sequences = false, int o_head_stride = 128, int d_out = 128) {
    CUtensorMap tm;
    if (!tmap_bf16_2d_cached(&tm, qkv, (uint64_t)rows, (uint64_t)ld, (uint64_t)ld, 128)) return cudaErrorInvalidValue;
    if (kv_prefix && !cu_seqlens) return cudaErrorInvalidValue;
    if (pair_sequences && (!cu_seqlens || causal || kv_prefix || max_len > 64)) return cudaErrorInvalidValue;
    if (d_out < 8 || d_out > 128 || (d_out & 7) || (o_head_stride & 7)) return cudaErrorInvalidValue;
    AttnParams p = {};
    p.pair = pair_sequences ? 1 : 0; p.n_seq = n_seq;
    p.o_head_stride = o_head_stride; p.d_out = d_out;
    p.o = o; p.ldo = ldo; p.cu_seqlens = cu_seqlens; p.seq_lens = seq_lens; p.S = S;
    p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0; p.kv_group = kv_group;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.kv_prefix = kv_prefix;
    const size_t smem = AttnSmem<128>::bytes();
    dim3 grid(pair_sequences ? 1 : (max_len + 127) / 128, Hq, pair_sequences ? (n_seq + 1) / 2 : n_seq);
    if (causal) return launch_attn_t<128, true>(tm, p, grid, smem, stream);
    return launch_attn_t<128, false>(tm, p, grid, smem, stream);
}

}  // namespace vqa

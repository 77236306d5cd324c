// Persistent, warp-specialised bf16 GEMM for sm_90a:  C[M,N] = epilogue( A[M,K] . W[N,K]^T )
//
//   * operands are both K-major (activations [M,K] row-major, nn.Linear weights [N,K] row-major), fetched
//     tile-by-tile from HBM/L2 by TMA into a 128B-swizzled shared-memory ring;
//   * CTA tile 128 x BLOCK_N: warpgroup 0 is the TMA producer, warpgroups 1 and 2 each own 64 rows of the tile and accumulate
//     them in registers with wgmma (m64 x BLOCK_N x k16, both operands read from shared memory);
//   * dense bf16 outputs (TMA_EPI): each consumer thread applies the fused epilogue (bias / activation / gated GELU or SiLU / residual
//     add) to the accumulator columns it holds, writes the bf16 results into a 128B-swizzled 64-row box with stmatrix, and a thread of
//     warpgroup 0 stores the box with TMA. That thread also TMA-loads the bf16 residual of each box ahead of the consumers, so the
//     consumers start the next tile's main loop without waiting on HBM in either direction;
//   * the other launches (fp32 C, split-K partials, batched GEMMs, scattered column groups, RMSNorm partial sums, the lm_head's online
//     log-sum-exp) stage 64-column fp32 slices of the accumulators through shared memory so that one thread owns one row's 32
//     consecutive columns before the only write to HBM.
//   The producer keeps loading the next tile's operands during either epilogue.
//
// Replaces the cuBLAS bf16 GEMMs that the reference reaches through nn.Linear
// (transformers/models/t5/modeling_t5.py:109-111,178-181; transformers/models/clip/modeling_clip.py:296-299,344-345).
#pragma once
#include "ptx.cuh"
#include <cuda.h>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <type_traits>
#include <unordered_map>

namespace vqa {

enum GemmEpilogue : int {
    EPI_STORE = 0,       // C = [residual +] bf16(acc [+ bias])
    EPI_QUICK_GELU = 1,  // C = quick_gelu(bf16(acc + bias))                 (CLIP MLP fc1)
    EPI_GELU_ERF = 2,    // C = gelu_erf(bf16(acc + bias))                   (mlp2x_gelu projector)
    EPI_GATED_GELU = 3,  // C = gelu_new(bf16(acc_gate)) * bf16(acc_up)      (T5 DenseGatedActDense wi_0/wi_1)
    EPI_LSE = 4,         // no C; per-row (max, sum exp) partials + label-logit gather (lm_head + CE)
    EPI_RELU = 5,        // C = relu(bf16(acc + bias))
    EPI_GATED_SILU = 6,  // C = silu(bf16(acc_gate + b_gate)) * bf16(acc_up + b_up)   (Qwen2.5-VL SwiGLU MLPs)
};
__host__ __device__ constexpr bool epi_is_gated(int epi) { return epi == EPI_GATED_GELU || epi == EPI_GATED_SILU; }

struct GemmParams {
    int M, N, K;              // N = number of OUTPUT columns of the logical GEMM (for GATED: 2 * out columns)
    __nv_bfloat16* C;         // [M, ldc]
    int ldc;
    const __nv_bfloat16* bias;      // [N] or nullptr
    const __nv_bfloat16* residual;  // [M, ldr] or nullptr
    int ldr;
    int c_f32;                // EPI_STORE only. 1: C and residual are fp32 buffers (ldc / ldr in floats): C = residual + bf16(acc + bias), unrounded
                              // 2: C is an fp32 buffer that receives the RAW accumulator (split-K partial sums: batches = K slices, reduced by
                              //    splitk_reduce_kernel, which also applies bias / rounding / residual)
                              // (the CLIP tower's residual stream stays fp32 under the reference's autocast: LayerNorm is on autocast's fp32 list)
    int gate_up_offset;       // GATED: row offset of the "up" weight block inside W (= d_ff)
    int c_group_in, c_group_out;   // EPI_STORE without residual, c_group_in > 0: logical output column c is stored at column
                              // (c / c_group_in) * c_group_out + c % c_group_in -- heads narrower than the attention kernel's 128-wide slots
                              // (Qwen2.5-VL vision tower, 80-wide) are produced at their native width and written into the slots; both multiples of 8
    // EPI_LSE
    float* lse_max;           // [M, num_n_tiles]
    float* lse_sum;           // [M, num_n_tiles]
    const int* labels;        // [M]
    float* label_logit;       // [M]
    float lse_scale;          // logits are multiplied by this (1 / temperature) after the bf16 rounding
    // optional repetition penalty (HF RepetitionPenaltyLogitsProcessor, generation/logits_process.py): bit n of row m's bitmap
    // set -> logit = logit < 0 ? logit * penalty : logit / penalty, applied to the bf16-rounded fp32 logit BEFORE the 1/T scale
    const uint32_t* penalty_bitmap;   // [M, penalty_words] or nullptr
    int penalty_words;
    float penalty;
    // RMSNorm folded into the GEMMs around it (T5LayerNorm modeling_t5.py:55-68 / Qwen2RMSNorm): the GEMM that WRITES the residual stream
    // (EPI_STORE with a residual) also emits, per row, the sum of squares of the bf16 values it stores for its slice of columns
    // (ssq_out[m * ssq_out_parts + n_tile * parts_per_tile + column_half]); the GEMM that CONSUMES the stream takes the un-normalised rows
    // as its A operand with gamma folded into W, sums the partials and multiplies its fp32 accumulator row by rsqrt(sum / dim + eps)
    // before the bf16 rounding of the Linear's output (EPI_STORE, EPI_GATED_*). No normalised copy of the stream is ever written.
    float* ssq_out;
    int ssq_out_parts;
    const float* ssq_in;
    int ssq_in_parts;
    float ssq_inv_dim, ssq_eps;
    // batching: `num_batches` independent GEMMs of the same M,N,K share one launch; batch b reads A at
    // (row + b*a_row_off, k + b*a_k_off), W at (row + b*w_row_off, k + b*w_k_off) and writes C + b*c_batch_stride.
    int num_batches;
    int a_row_off, a_k_off, w_row_off, w_k_off;
    long long c_batch_stride;
    // scheduling: W is cut into chunks of `chunk_n` N tiles; inside a chunk, groups of `group_m` M tiles sweep the chunk's N tiles
    int num_m_tiles, num_n_tiles, group_m, chunk_n;
    // L2 eviction priority of the two operand streams (ptx.cuh L2_EVICT_*), chosen per launch by launch_gemm_t
    unsigned long long a_policy, w_policy;
};

template <int BLOCK_N>
struct GemmConfig {
    static constexpr int BLOCK_M = 128;           // rows per CTA: two consumer warpgroups x 64
    static constexpr int BLOCK_K = 64;            // 64 bf16 = 128 B = one swizzle atom
    static constexpr int WGMMA_K = 16;
    static constexpr int B_HALF_ROWS = BLOCK_N / 2;
    static constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
    static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
    static constexpr int NUM_THREADS = 384;       // warpgroup 0: TMA; warpgroups 1, 2: wgmma + epilogue
    // epilogue staging area, the same size on both epilogue paths: per consumer warpgroup either one 64 x EPI_COLS fp32 slice of the
    // accumulators (staged path; 16-byte chunks XOR-swizzled by row, see stg_index), or two bf16 output boxes of 64 rows x <= 64 columns
    // (TMA-store path)
    static constexpr int EPI_COLS = BLOCK_N >= 64 ? 64 : 32;
    static constexpr int EPI_BYTES = 2 * 64 * EPI_COLS * 4;
    // one thread per (row, 32-column half of a staged slice): LSE_PARTS partial results per row and tile
    static constexpr int LSE_PARTS = EPI_COLS / 32;
    static constexpr int SMEM_LIMIT = 227 * 1024;  // H100: dynamic shared memory per block
    static constexpr int STAGES_RAW = (SMEM_LIMIT - EPI_BYTES - 1024 - 256) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(BLOCK_N >= 32 && BLOCK_N <= 256 && (BLOCK_N & (BLOCK_N - 1)) == 0, "BLOCK_N must be 32..256, pow2");
    static_assert(B_HALF_ROWS % 8 == 0, "B half tile must hold whole 8-row swizzle atoms");
    static_assert(STAGES >= 3, "pipeline too shallow");
    // the main loop keeps one wgmma group in flight, which holds two slots: a fourth stage gives the 256-wide tile's producer two k blocks of look-ahead
    static_assert(BLOCK_N != 256 || STAGES == 4, "the 256-wide tile runs a four-stage ring on both epilogue paths");
    static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory");
    // staged path: float index of (row r, column c) of a warpgroup's fp32 slice. Chunk c / 4 of row r sits at chunk (c / 4) ^ s(r) with
    // s(r) = 2 (r % 4) + (r / 4) % 2: the float2 writes in accumulator layout (rows r..r+3 of 8-aligned groups, two adjacent chunks per row)
    // and the float4 row reads (8 consecutive rows, one chunk) are both free of bank conflicts.
    __device__ static __forceinline__ int stg_index(int r, int c) {
        return r * EPI_COLS + ((((c >> 2) ^ (((r & 3) << 1) | ((r >> 2) & 1)))) << 2) + (c & 3);
    }
};

// TMA-store epilogue: columns of one bf16 output box (64 rows per consumer warpgroup). Gated epilogues write BLOCK_N / 2 columns per tile.
__host__ __device__ constexpr int gemm_out_box_cols(int block_n, int epi) {
    return (epi_is_gated(epi) ? block_n / 2 : block_n) >= 64 ? 64 : 32;
}

__device__ __forceinline__ float act_quick_gelu(float x) { return __fdividef(x, 1.0f + __expf(-1.702f * x)); }
__device__ __forceinline__ float act_silu(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float act_gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float act_gelu_new(float x) {
    // 0.5 * x * (1 + tanh(sqrt(2/pi) * (x + 0.044715 x^3)))  -- transformers/activations.py NewGELUActivation, evaluated in fp32 like the
    // reference does under CUDA autocast (torch.pow is on autocast's fp32 list, so everything downstream of it is fp32).
    // tanh(u) = 1 - 2 / (exp(2u) + 1) with ex2.approx + rcp.approx: relative error ~1e-6. (tanh.approx.f32 is 2^-11 absolute, i.e. a
    // SYSTEMATIC 5e-4 error in 48 FFNs -- too coarse for parity with the fp32-evaluated reference.)
    const float k = 0.7978845608028654f;
    const float inner = k * (x + 0.044715f * x * x * x);
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(inner * 2.8853900817779268f));   // exp(2u) = 2^(2u log2 e)
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    const float th = 1.0f - 2.0f * r;
    return 0.5f * x * (1.0f + th);
}
// CLIP's quick_gelu as eager bf16 tensor ops run it (`input * torch.sigmoid(1.702 * input)`, transformers/activations.py:117-123; none of
// the three ops is on an autocast list, so each produces a bf16 tensor): y bf16 -> bf16(1.702 y) -> bf16(sigmoid) -> product (rounded by caller)
__device__ __forceinline__ float act_quick_gelu_bf16_ops(float y) {
    const float a = bf16_round(1.702f * y);
    const float sg = bf16_round(__fdividef(1.0f, 1.0f + __expf(-a)));
    return y * sg;
}

// calls f(std::integral_constant<int, i>) for i = 0 .. N-1 (compile-time indices into register arrays)
template <int I, int N, typename F>
__device__ __forceinline__ void static_for_impl(F&& f) {
    if constexpr (I < N) {
        f(std::integral_constant<int, I>{});
        static_for_impl<I + 1, N>(f);
    }
}
template <int N, typename F>
__device__ __forceinline__ void static_for(F&& f) { static_for_impl<0, N>(f); }

// TMA_EPI: the TMA-store epilogue (dense bf16 C, not batched); tmap_c maps C as [M, n_out] with row stride ldc, tmap_r the bf16 residual
// the same way (both boxes of 64 rows x gemm_out_box_cols). Otherwise the staged epilogue, which serves EPI_STORE and EPI_LSE only, and
// the two maps are not read.
template <int BLOCK_N, int EPI, bool TMA_EPI>
__global__ void __launch_bounds__(384, 1)
gemm_bf16_sm90_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                      const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r, const GemmParams p) {
    using Cfg = GemmConfig<BLOCK_N>;
    static_assert(!epi_is_gated(EPI) || BLOCK_N >= 64, "gated epilogue pairs two >=32-column half tiles");
    static_assert(TMA_EPI ? EPI != EPI_LSE : (EPI == EPI_STORE || EPI == EPI_LSE), "the staged epilogue serves plain stores and the lm_head");
    pdl_launch_dependents();
    constexpr int STAGES = Cfg::STAGES;
    constexpr int BLOCK_M = Cfg::BLOCK_M;
    constexpr int BLOCK_K = Cfg::BLOCK_K;
    constexpr int OUT_TILE_COLS = epi_is_gated(EPI) ? BLOCK_N / 2 : BLOCK_N;
    constexpr int BOX_COLS = gemm_out_box_cols(BLOCK_N, EPI);
    constexpr int BOX_ROW_BYTES = BOX_COLS * 2;                  // 128 B (SWIZZLE_128B) or 64 B (SWIZZLE_64B)
    constexpr int BOX_BYTES = 64 * BOX_ROW_BYTES;
    constexpr int NBOX = OUT_TILE_COLS / BOX_COLS;               // boxes per consumer warpgroup and tile
    static_assert(4 * BOX_BYTES <= Cfg::EPI_BYTES, "two boxes per consumer warpgroup fit the staging area");
    static_assert((2 * STAGES + 8) * 8 <= 256, "mbarriers fit their 256 bytes");

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;                                      // [STAGES][128 x 64 bf16]
    uint8_t* smem_b = smem + STAGES * Cfg::A_STAGE_BYTES;        // [STAGES][BLOCK_N x 64 bf16]
    uint8_t* smem_epi = smem + STAGES * Cfg::STAGE_BYTES;        // staged: [2][64][EPI_COLS] fp32; TMA store: [2 warpgroups][2][BOX_BYTES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::EPI_BYTES);
    uint64_t* full_bar = bars;                 // [STAGES]
    uint64_t* empty_bar = bars + STAGES;       // [STAGES]
    // TMA-store epilogue, box buffer i = 2 * (consumer warpgroup) + (box count & 1):
    //   box_free[i]  (count 1)  buffer i may be written: holds the box's residual (expect_tx) or its previous store has read it (plain arrive)
    //   box_ready[i] (count 4)  each consumer warp has written its rows of the box into buffer i
    uint64_t* box_free = bars + 2 * STAGES;    // [4]
    uint64_t* box_ready = bars + 2 * STAGES + 4;   // [4]

    const uint32_t wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        if constexpr (TMA_EPI) {
            tma_prefetch_desc(&tmap_c);
            tma_prefetch_desc(&tmap_r);
        }
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);    // the producer's expect_tx
            mbar_init(&empty_bar[s], 8);   // one arrive per consumer warp
        }
        if constexpr (TMA_EPI) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                mbar_init(&box_free[i], 1);
                mbar_init(&box_ready[i], 4);
            }
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();      // everything above touched only this CTA's shared memory; from here on operands of earlier kernels are read

    const int num_k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
    const int tiles_per_batch = p.num_m_tiles * p.num_n_tiles;
    const int num_tiles = tiles_per_batch * p.num_batches;
    const int num_workers = gridDim.x;
    const int worker = blockIdx.x;
    const int tiles_per_chunk = p.num_m_tiles * p.chunk_n;

    // Tile order (L2 blocking): W chunk (chunk_n N tiles, sized to stay resident in L2) -> group of group_m M tiles -> the chunk's
    // N tiles -> the group's M tiles (fastest). One wave of CTAs therefore shares group_m A row panels and a few W panels, the W chunk
    // is re-read from L2 by every M group, and A streams through once per chunk.
    auto tile_coords = [&](int t, int& batch, int& m_blk, int& n_blk) {
        batch = t / tiles_per_batch;
        t -= batch * tiles_per_batch;
        const int c = t / tiles_per_chunk;
        t -= c * tiles_per_chunk;
        const int n_first = c * p.chunk_n;
        const int cn = min(p.chunk_n, p.num_n_tiles - n_first);
        const int tiles_per_group = p.group_m * cn;
        const int g = t / tiles_per_group;
        const int r = t - g * tiles_per_group;
        const int m_first = g * p.group_m;
        const int gm = min(p.group_m, p.num_m_tiles - m_first);
        m_blk = m_first + r % gm;
        n_blk = n_first + r / gm;
    };

    if (wg == 0) {
        // ===================== TMA producer =====================
        regs_dealloc<40>();
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = worker; t < num_tiles; t += num_workers) {
                int batch, m_blk, n_blk;
                tile_coords(t, batch, m_blk, n_blk);
                const int m_row = m_blk * BLOCK_M + batch * p.a_row_off;
                const int w_row_base = batch * p.w_row_off;
                for (int kb = 0; kb < num_k_blocks; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1u);
                    uint8_t* sa = smem_a + stage * Cfg::A_STAGE_BYTES;
                    uint8_t* sb = smem_b + stage * Cfg::B_STAGE_BYTES;
                    const int k0 = kb * BLOCK_K + batch * p.a_k_off;
                    const int k0w = kb * BLOCK_K + batch * p.w_k_off;
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    tma_load_2d_hint(sa, &tmap_a, &full_bar[stage], k0, m_row, p.a_policy);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int n_row = epi_is_gated(EPI) ? h * p.gate_up_offset + n_blk * Cfg::B_HALF_ROWS
                                                            : n_blk * BLOCK_N + h * Cfg::B_HALF_ROWS;
                        tma_load_2d_hint(sb + h * Cfg::B_HALF_ROWS * BLOCK_K * 2, &tmap_b, &full_bar[stage], k0w,
                                         n_row + w_row_base, p.w_policy);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
        if constexpr (TMA_EPI) {
            // ===================== box thread of consumer warpgroup cw (lane 0 of warp 1 + cw) =====================
            // Walks the same tiles as its consumer warpgroup; box q (q = 0, 1, ... over all of them) uses buffer b = q & 1 for the
            // u = q >> 1 th time. Protocol of buffer b (both barriers complete one phase per use, so use u waits on parity u & 1):
            //   box thread, box q:  if q >= 2: wait box_ready[b] (parity of use u - 1), TMA-store box q - 2, wait until the store
            //                       has read the buffer; then complete box_free[b] for use u -- with the residual's expect_tx and its
            //                       TMA load, or with a plain arrive when there is nothing to load;
            //   consumers,  box q:  wait box_free[b] (parity u & 1), read the residual, write the results in place, fence.proxy.async,
            //                       one arrive per warp on box_ready[b].
            // box_free[b] for use u + 1 needs box_ready[b] of use u, which needs box_free[b] of use u: neither barrier can run a phase
            // ahead of the wait that reads it. After the last box the thread stores the (up to) two pending boxes and waits for all of
            // its stores to complete before the CTA exits.
            if (threadIdx.x == 32 || threadIdx.x == 64) {
                const int cw = (int)(threadIdx.x >> 5) - 1;
                const int n_out = epi_is_gated(EPI) ? p.N / 2 : p.N;
                const bool load_residual = !epi_is_gated(EPI) && p.residual != nullptr;
                uint8_t* buf = smem_epi + cw * 2 * BOX_BYTES;
                uint64_t* free_bar = box_free + cw * 2;
                uint64_t* ready_bar = box_ready + cw * 2;
                auto store_box = [&](int q, int c0, int r0) {
                    mbar_wait(&ready_bar[q & 1], (uint32_t)(q >> 1) & 1u);
                    if (r0 < p.M && c0 < n_out) {   // a box wholly outside C is not stored
                        tma_store_2d(&tmap_c, buf + (q & 1) * BOX_BYTES, c0, r0);
                        bulk_commit_group();
                        bulk_wait_group_read<0>();
                    }
                };
                int q = 0;
                int c0_1 = 0, r0_1 = 0, c0_2 = 0, r0_2 = 0;   // boxes q - 1 and q - 2
                for (int t = worker; t < num_tiles; t += num_workers) {
                    int batch, m_blk, n_blk;
                    tile_coords(t, batch, m_blk, n_blk);
                    const int r0 = m_blk * BLOCK_M + cw * 64;
                    for (int s = 0; s < NBOX; ++s, ++q) {
                        const int c0 = n_blk * OUT_TILE_COLS + s * BOX_COLS;
                        if (q >= 2) store_box(q - 2, c0_2, r0_2);
                        if (load_residual && r0 < p.M && c0 < n_out) {
                            mbar_arrive_expect_tx(&free_bar[q & 1], BOX_BYTES);
                            tma_load_2d(buf + (q & 1) * BOX_BYTES, &tmap_r, &free_bar[q & 1], c0, r0);
                        } else {
                            mbar_arrive(&free_bar[q & 1]);
                        }
                        c0_2 = c0_1; r0_2 = r0_1; c0_1 = c0; r0_1 = r0;
                    }
                }
                if (q >= 2) store_box(q - 2, c0_2, r0_2);
                if (q >= 1) store_box(q - 1, c0_1, r0_1);
                bulk_wait_group<0>();
            }
        }
    } else {
        // ===================== consumers: wgmma main loop, then the epilogue of the tile =====================
        regs_alloc<232>();
        const int cw = (int)wg - 1;                  // rows [64 cw, 64 cw + 64) of every tile
        const int tid = (int)threadIdx.x - 128 * (int)wg;
        const int lane = tid & 31;
        float* stg = reinterpret_cast<float*>(smem_epi) + cw * 64 * Cfg::EPI_COLS;
        // accumulator fragment of this thread: rows fr and fr + 8, columns 8j + fc + {0, 1}
        const int fr = (tid >> 5) * 16 + (lane >> 2);
        const int fc = (lane & 3) * 2;
        // staged epilogue ownership: row er of the warpgroup's 64, 32-column half esub of each staged slice
        const int er = tid & 63;
        const int esub = tid >> 6;
        constexpr int NSLICE = BLOCK_N / Cfg::EPI_COLS;   // staged slices per tile
        const bool e_active = esub < Cfg::LSE_PARTS;
        // TMA-store epilogue: this lane's row address in the x4 matrix moves (matrix i = lane / 8: rows +8 (i & 1), 8-column chunk +(i >> 1))
        const int mx_row = (tid >> 5) * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
        const int mx_chunk = lane >> 4;
        uint8_t* box_buf = smem_epi + cw * 2 * BOX_BYTES;
        int box_q = 0;                               // boxes this warpgroup has written (see the box thread's protocol)
        // fused RMSNorm of the A rows (consumer side): rsqrt(mean of squares + eps) of row m
        auto row_scale_of = [&](int m) {
            if (!p.ssq_in || m >= p.M) return 1.0f;
            const float* sp = p.ssq_in + (size_t)m * p.ssq_in_parts;
            float ssum = 0.f;
            for (int i = 0; i < p.ssq_in_parts; i += 4) {
                const float4 v4 = __ldg(reinterpret_cast<const float4*>(sp + i));
                ssum += (v4.x + v4.y) + (v4.z + v4.w);
            }
            return rsqrtf(ssum * p.ssq_inv_dim + p.ssq_eps);
        };
        float acc[BLOCK_N / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int t = worker; t < num_tiles; t += num_workers) {
            int batch, m_blk, n_blk;
            tile_coords(t, batch, m_blk, n_blk);
            int prev_stage = 0;
            for (int kb = 0; kb < num_k_blocks; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint64_t adesc = make_sw128_desc(smem_u32(smem_a + stage * Cfg::A_STAGE_BYTES + cw * 64 * 128));
                const uint64_t bdesc = make_sw128_desc(smem_u32(smem_b + stage * Cfg::B_STAGE_BYTES));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BLOCK_K / Cfg::WGMMA_K; ++k)
                    // advance 16 elements (32 B) along K inside the swizzle atom: +2 in 16-byte units
                    wgmma_ss<BLOCK_N>(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
                wgmma_commit();
                if (kb > 0) {
                    wgmma_wait<1>();                                   // the previous k block's wgmmas have read their slot
                    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
                }
                prev_stage = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1u; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

            if constexpr (TMA_EPI) {
                // ---------------- TMA-store epilogue: the math in the accumulator layout, bf16 results into the box buffers
                const int m0 = m_blk * BLOCK_M + cw * 64 + fr;
                const float rs[2] = {row_scale_of(m0), row_scale_of(m0 + 8)};
                static_for<NBOX>([&](auto s_c) {
                    constexpr int s = decltype(s_c)::value;
                    const int b = box_q & 1;
                    uint8_t* box = box_buf + b * BOX_BYTES;
                    mbar_wait(&box_free[cw * 2 + b], (uint32_t)(box_q >> 1) & 1u);
                    static_for<BOX_COLS / 16>([&](auto t_c) {
                        constexpr int t = decltype(t_c)::value;
                        // swizzled address of (row mx_row, 16-byte chunk 2t + mx_chunk): the box's 16-byte chunk c of row r sits at chunk
                        // c ^ ((row byte offset / 128) % (BOX_ROW_BYTES / 16)), the pattern TMA's 128B / 64B swizzle reads and writes
                        const uint32_t off = (uint32_t)(mx_row * BOX_ROW_BYTES + (2 * t + mx_chunk) * 16);
                        const uint32_t addr = smem_u32(box) + (off ^ (((off >> 7) & (BOX_ROW_BYTES / 16 - 1)) << 4));
                        uint32_t v[4] = {0u, 0u, 0u, 0u};
                        if (!epi_is_gated(EPI) && p.residual) ldmatrix_x4(addr, v);   // the TMA-loaded residual of the same elements
                        static_for<4>([&](auto k_c) {
                            constexpr int k = decltype(k_c)::value;
                            constexpr int jo = s * (BOX_COLS / 8) + 2 * t + (k >> 1);   // output 8-column chunk of the tile
                            constexpr int h = k & 1;                                   // row fr + 8h
                            constexpr int ia = 4 * jo + 2 * h;                         // acc index of the pair's first column
                            const int n = n_blk * OUT_TILE_COLS + 8 * jo + fc;        // output column of the pair
                            if constexpr (epi_is_gated(EPI)) {
                                // gate column n at acc[ia], its up column (BLOCK_N / 2 accumulator columns further) at acc[ia + BLOCK_N / 4]
                                float g0 = acc[ia] * rs[h], g1 = acc[ia + 1] * rs[h];
                                float u0 = acc[ia + BLOCK_N / 4] * rs[h], u1 = acc[ia + BLOCK_N / 4 + 1] * rs[h];
                                if (p.bias) {   // [gate bias | up bias], `gate_up_offset` apart like the weight rows
                                    if (n < p.N / 2) {
                                        const float2 bg = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.bias + n));
                                        const float2 bu = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.bias + p.gate_up_offset + n));
                                        g0 += bg.x; g1 += bg.y; u0 += bu.x; u1 += bu.y;
                                    }
                                }
                                g0 = bf16_round(g0); g1 = bf16_round(g1); u0 = bf16_round(u0); u1 = bf16_round(u1);
                                float h0, h1;
                                if constexpr (EPI == EPI_GATED_GELU) {
                                    // T5DenseGatedActDense under CUDA autocast: act(wi_0 x) comes out in fp32 (pow -> fp32), the product
                                    // with the bf16 wi_1 x is fp32, and the single rounding is the cast in front of `wo` (modeling_t5.py:115-131)
                                    h0 = act_gelu_new(g0) * u0;
                                    h1 = act_gelu_new(g1) * u1;
                                } else {
                                    h0 = bf16_round(act_silu(g0)) * u0;
                                    h1 = bf16_round(act_silu(g1)) * u1;
                                }
                                v[k] = pack_bf16x2(h0, h1);
                            } else {
                                float f0 = acc[ia] * rs[h], f1 = acc[ia + 1] * rs[h];
                                const float2 bb = (p.bias && n < p.N) ? unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n)))
                                                                      : make_float2(0.f, 0.f);
                                f0 += bb.x; f1 += bb.y;
                                float y[2] = {bf16_round(f0), bf16_round(f1)};   // the Linear's bf16 output in the reference
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    if constexpr (EPI == EPI_QUICK_GELU) y[e] = act_quick_gelu_bf16_ops(y[e]);
                                    if constexpr (EPI == EPI_GELU_ERF) y[e] = act_gelu_erf(y[e]);
                                    if constexpr (EPI == EPI_RELU) y[e] = fmaxf(y[e], 0.f);
                                }
                                const float2 r = unpack_bf16x2(v[k]);   // zero without a residual
                                f0 = y[0]; f1 = y[1];
                                f0 += r.x; f1 += r.y;
                                v[k] = pack_bf16x2(f0, f1);
                            }
                        });
                        stmatrix_x4(addr, v);
                    });
                    fence_proxy_async_shared();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&box_ready[cw * 2 + b]);
                    ++box_q;
                });
                continue;
            }
            // ---------------- staged epilogue
            const long long c_off = (long long)batch * p.c_batch_stride;
            const int m = m_blk * BLOCK_M + cw * 64 + er;
            const bool row_ok = m < p.M;
            const float row_scale = row_scale_of(m);
            // accumulator columns [src, src + 8 * n8) -> staging columns [dst, ...) of this warpgroup's 64 rows
            auto stage_out = [&](auto src_c, int dst, auto n8_c) {
                constexpr int src = decltype(src_c)::value;
                constexpr int n8 = decltype(n8_c)::value;
#pragma unroll
                for (int j = 0; j < n8; ++j) {
                    const int b = (src / 8 + j) * 4;
                    *reinterpret_cast<float2*>(stg + Cfg::stg_index(fr, dst + 8 * j + fc)) = make_float2(acc[b], acc[b + 1]);
                    *reinterpret_cast<float2*>(stg + Cfg::stg_index(fr + 8, dst + 8 * j + fc)) = make_float2(acc[b + 2], acc[b + 3]);
                }
            };
            auto load_row = [&](int col, auto n_c, uint32_t* v) {
                constexpr int n = decltype(n_c)::value;
#pragma unroll
                for (int i = 0; i < n; i += 4) {
                    const float4 f = *reinterpret_cast<const float4*>(stg + Cfg::stg_index(er, col + i));
                    v[i] = __float_as_uint(f.x); v[i + 1] = __float_as_uint(f.y); v[i + 2] = __float_as_uint(f.z); v[i + 3] = __float_as_uint(f.w);
                }
            };
            float run_max = -INFINITY, run_sum = 0.f;   // EPI_LSE
            float ssq_acc = 0.f;                        // producer side of the fused RMSNorm: sum of squares of the bf16 values this thread stores
            const int label = (EPI == EPI_LSE && row_ok) ? p.labels[m] : -1;
            static_for<NSLICE>([&](auto s_c) {
                constexpr int s = decltype(s_c)::value;
                named_bar_sync(1 + cw, 128);            // the previous slice has been read
                stage_out(std::integral_constant<int, s * Cfg::EPI_COLS>{}, 0, std::integral_constant<int, Cfg::EPI_COLS / 8>{});
                named_bar_sync(1 + cw, 128);
                if (!e_active) return;
                {
                    uint32_t v[32];
                    load_row(esub * 32, std::integral_constant<int, 32>{}, v);
                    const int nc = n_blk * BLOCK_N + s * Cfg::EPI_COLS + esub * 32;   // first column of this thread's 32
                    if constexpr (EPI == EPI_LSE) {
                        float x[32];
                        float cmax = -INFINITY;
                        const uint32_t pen_bits = (p.penalty_bitmap && row_ok && nc < p.N)
                                                      ? p.penalty_bitmap[(size_t)m * p.penalty_words + (nc >> 5)] : 0u;
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int n = nc + j;
                            float raw = bf16_round(__uint_as_float(v[j]));                  // reference logits are bf16, then fp32
                            if (pen_bits && ((pen_bits >> j) & 1u)) raw = raw < 0.f ? raw * p.penalty : __fdiv_rn(raw, p.penalty);
                            float val = raw * p.lse_scale;                                   // ... / T in fp32
                            x[j] = (n < p.N) ? val : -INFINITY;
                            cmax = fmaxf(cmax, x[j]);
                            if (n == label) p.label_logit[m] = val;
                        }
                        if (cmax > -INFINITY) {
                            const float new_max = fmaxf(run_max, cmax);
                            float sacc = 0.f;
#pragma unroll
                            for (int j = 0; j < 32; ++j) sacc += __expf(x[j] - new_max);
                            run_sum = run_sum * __expf(run_max - new_max) + sacc;
                            run_max = new_max;
                        }
                    } else if (EPI == EPI_STORE && p.c_f32) {
                        float* Cf = reinterpret_cast<float*>(p.C);
                        const float* Rf = reinterpret_cast<const float*>(p.residual);
                        if (row_ok && nc < p.N) {
                            float* crow = Cf + c_off + (size_t)m * p.ldc + nc;
                            const float* rrow = Rf ? Rf + c_off + (size_t)m * p.ldr + nc : nullptr;
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                if (nc + j * 4 < p.N) {
                                    if (p.c_f32 == 2) {
                                        *reinterpret_cast<float4*>(crow + j * 4) = make_float4(__uint_as_float(v[j * 4]), __uint_as_float(v[j * 4 + 1]),
                                                                                              __uint_as_float(v[j * 4 + 2]), __uint_as_float(v[j * 4 + 3]));
                                        continue;
                                    }
                                    float4 r = rrow ? *reinterpret_cast<const float4*>(rrow + j * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                                    float b[4] = {0.f, 0.f, 0.f, 0.f};
                                    if (p.bias) {
                                        const uint2 bb = __ldg(reinterpret_cast<const uint2*>(p.bias + nc + j * 4));
                                        const float2 b0 = unpack_bf16x2(bb.x), b1 = unpack_bf16x2(bb.y);
                                        b[0] = b0.x; b[1] = b0.y; b[2] = b1.x; b[3] = b1.y;
                                    }
                                    r.x += bf16_round(__uint_as_float(v[j * 4]) + b[0]);
                                    r.y += bf16_round(__uint_as_float(v[j * 4 + 1]) + b[1]);
                                    r.z += bf16_round(__uint_as_float(v[j * 4 + 2]) + b[2]);
                                    r.w += bf16_round(__uint_as_float(v[j * 4 + 3]) + b[3]);
                                    *reinterpret_cast<float4*>(crow + j * 4) = r;
                                }
                            }
                        }
                    } else {
                        if (row_ok && nc < p.N) {
                            __nv_bfloat16* crow = p.C + c_off + (size_t)m * p.ldc + nc;
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                if (nc + j * 8 < p.N) {
                                    const uint4 bq = p.bias ? __ldg(reinterpret_cast<const uint4*>(p.bias + nc + j * 8)) : make_uint4(0, 0, 0, 0);
                                    const uint4 rq = p.residual ? *reinterpret_cast<const uint4*>(p.residual + c_off + (size_t)m * p.ldr + nc + j * 8)
                                                                : make_uint4(0, 0, 0, 0);
                                    float f[8];
#pragma unroll
                                    for (int e = 0; e < 8; ++e) f[e] = __uint_as_float(v[j * 8 + e]) * row_scale;
                                    {
                                        float2 b0 = unpack_bf16x2(bq.x), b1 = unpack_bf16x2(bq.y);
                                        float2 b2 = unpack_bf16x2(bq.z), b3 = unpack_bf16x2(bq.w);
                                        f[0] += b0.x; f[1] += b0.y; f[2] += b1.x; f[3] += b1.y;
                                        f[4] += b2.x; f[5] += b2.y; f[6] += b3.x; f[7] += b3.y;
                                    }
#pragma unroll
                                    for (int e = 0; e < 8; ++e) f[e] = bf16_round(f[e]);   // the Linear's bf16 output in the reference
                                    {
                                        float2 r0 = unpack_bf16x2(rq.x), r1 = unpack_bf16x2(rq.y);
                                        float2 r2 = unpack_bf16x2(rq.z), r3 = unpack_bf16x2(rq.w);
                                        f[0] += r0.x; f[1] += r0.y; f[2] += r1.x; f[3] += r1.y;
                                        f[4] += r2.x; f[5] += r2.y; f[6] += r3.x; f[7] += r3.y;
                                    }
                                    uint4 o = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]),
                                                         pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
                                    __nv_bfloat16* dst = crow + j * 8;
                                    if (p.c_group_in > 0) {
                                        const int cc = nc + j * 8;
                                        dst = p.C + c_off + (size_t)m * p.ldc + (cc / p.c_group_in) * p.c_group_out + cc % p.c_group_in;
                                    }
                                    *reinterpret_cast<uint4*>(dst) = o;
                                    if (p.ssq_out) {
                                        const float2 s0 = unpack_bf16x2(o.x), s1 = unpack_bf16x2(o.y), s2 = unpack_bf16x2(o.z), s3 = unpack_bf16x2(o.w);
                                        ssq_acc += (s0.x * s0.x + s0.y * s0.y) + (s1.x * s1.x + s1.y * s1.y) + (s2.x * s2.x + s2.y * s2.y) +
                                                   (s3.x * s3.x + s3.y * s3.y);
                                    }
                                }
                            }
                        }
                    }
                }
            });
            if (e_active && row_ok) {
                // one partial per (row, n tile, 32-column half of the staged slices)
                if constexpr (EPI == EPI_LSE) {
                    const size_t slot = ((size_t)m * p.num_n_tiles + n_blk) * Cfg::LSE_PARTS + esub;
                    p.lse_max[slot] = run_max;
                    p.lse_sum[slot] = run_sum;
                } else if (EPI == EPI_STORE) {
                    if (p.ssq_out) p.ssq_out[(size_t)m * p.ssq_out_parts + n_blk * Cfg::LSE_PARTS + esub] = ssq_acc;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    return fn;
}

// bf16 row-major [rows, cols] (row stride ld elements) -> 2-D map, box {box_cols, box_rows}; box_cols 64 (128B swizzle) or 32 (64B swizzle).
inline bool make_tmap_bf16_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                              uint32_t box_rows, uint32_t box_cols = 64) {
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc || (box_cols != 64 && box_cols != 32)) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// process-wide tuning overrides (vqa_set_gemm_schedule); 0 = automatic
static int g_gemm_group_rows_override = 0;
static int g_gemm_chunk_rows_override = 0;

// The same (base, shape) pairs come back on every forward (weights and workspace slices are stable), and encoding a CUtensorMap costs
// a driver call: keep the encoded maps per thread. The map only describes address + extents, so a hit is valid whatever lives there.
struct TmapKey {
    const void* base; uint64_t rows, cols, ld; uint32_t box_rows, box_cols;
    bool operator==(const TmapKey& o) const {
        return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && box_cols == o.box_cols;
    }
};
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        uint64_t h = reinterpret_cast<uint64_t>(k.base) * 0x9E3779B97F4A7C15ull;
        h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
        h ^= (k.cols * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2));
        h ^= (k.ld * 0x165667B19E3779F9ull + k.box_rows + ((uint64_t)k.box_cols << 32) + (h << 6) + (h >> 2));
        return (size_t)h;
    }
};
inline bool tmap_bf16_2d_cached(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                                uint32_t box_cols = 64) {
    static thread_local std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
    const TmapKey key{base, rows, cols, ld, box_rows, box_cols};
    auto it = cache.find(key);
    if (it != cache.end()) { memcpy(map, &it->second, sizeof(CUtensorMap)); return true; }
    if (!make_tmap_bf16_2d(map, base, rows, cols, ld, box_rows, box_cols)) return false;
    if (cache.size() > 16384) cache.clear();
    cache.emplace(key, *map);
    return true;
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per (function, device): remember which devices have it for this kernel.
struct PerDeviceOnce {
    std::atomic<uint64_t> done{0};
    template <typename F>
    cudaError_t ensure(F&& set) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        const uint64_t bit = 1ull << (dev & 63);
        if (done.load(std::memory_order_acquire) & bit) return cudaSuccess;
        e = set();
        if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_release);
        return e;
    }
};

// number of (row) partial sums a residual-writing GEMM of N columns emits with this tile shape (GemmParams::ssq_out_parts)
template <int BLOCK_N>
inline int gemm_ssq_parts(int N) { return ((N + BLOCK_N - 1) / BLOCK_N) * GemmConfig<BLOCK_N>::LSE_PARTS; }

struct GemmLaunch {
    const __nv_bfloat16* A; int lda;   // [a_rows, a_cols] visible to TMA (defaults: M x K)
    const __nv_bfloat16* W; int ldw;   // [w_rows, w_cols] visible to TMA (defaults: N x K; 2*d_ff rows for GATED)
    int w_rows;
    long long a_rows = 0, a_cols = 0, w_cols = 0;   // 0 = default
    GemmParams p;
};

// TMA_EPI: the TMA-store epilogue (dense bf16 C and residual, one batch); C and the residual must start on 16 bytes and have row strides
// that are multiples of 8 elements.
template <int BLOCK_N, int EPI, bool TMA_EPI>
inline cudaError_t launch_gemm_t(const GemmLaunch& g, int num_sms, cudaStream_t stream) {
    using Cfg = GemmConfig<BLOCK_N>;
    auto kernel = gemm_bf16_sm90_kernel<BLOCK_N, EPI, TMA_EPI>;
    static PerDeviceOnce attr;
    {
        cudaError_t e = attr.ensure([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES); });
        if (e != cudaSuccess) return e;
    }
    CUtensorMap ta, tb;
    const uint64_t a_rows = g.a_rows ? (uint64_t)g.a_rows : (uint64_t)g.p.M;
    const uint64_t a_cols = g.a_cols ? (uint64_t)g.a_cols : (uint64_t)g.p.K;
    const uint64_t w_cols = g.w_cols ? (uint64_t)g.w_cols : (uint64_t)g.p.K;
    if (!tmap_bf16_2d_cached(&ta, g.A, a_rows, a_cols, (uint64_t)g.lda, Cfg::BLOCK_M)) return cudaErrorInvalidValue;
    if (!tmap_bf16_2d_cached(&tb, g.W, (uint64_t)g.w_rows, w_cols, (uint64_t)g.ldw, Cfg::B_HALF_ROWS))
        return cudaErrorInvalidValue;
    CUtensorMap tc = ta, tr = ta;   // not read by the staged epilogue
    if constexpr (TMA_EPI) {
        // extents [M, n_out]: the hardware clips the ragged last tiles, and columns n_out .. ldc - 1 are never written
        const GemmParams& q = g.p;
        const uint64_t n_out = epi_is_gated(EPI) ? q.N / 2 : q.N;
        constexpr uint32_t box_cols = gemm_out_box_cols(BLOCK_N, EPI);
        auto tma_ok = [](const void* ptr, int ld) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && ld > 0 && ld % 8 == 0; };
        if (g.p.num_batches > 1 || !tma_ok(q.C, q.ldc) || (q.residual && !tma_ok(q.residual, q.ldr))) return cudaErrorInvalidValue;
        if (!tmap_bf16_2d_cached(&tc, q.C, (uint64_t)q.M, n_out, (uint64_t)q.ldc, 64, box_cols)) return cudaErrorInvalidValue;
        if (q.residual && !tmap_bf16_2d_cached(&tr, q.residual, (uint64_t)q.M, n_out, (uint64_t)q.ldr, 64, box_cols)) return cudaErrorInvalidValue;
    }
    GemmParams p = g.p;
    if (p.num_batches < 1) p.num_batches = 1;
    const int rows_per_tile = Cfg::BLOCK_M;
    p.num_m_tiles = (p.M + rows_per_tile - 1) / rows_per_tile;
    p.num_n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
    // Tile order = L2 blocking (see tile_coords). Either the W chunk or the A row group is the L2-resident operand:
    //   * W-stationary: W cut into chunks of <= ~14 MB, small A groups stream past each chunk;
    //   * A-stationary: one chunk (all of W streams), A groups of ~12 MB.
    // Sizes chosen for the H100's 50 MB L2. Measured against other orders at the clip-flant5-xxl encoder shapes (M = 43008, isolated CUDA-event
    // times; DESIGN.md section 8): best or within 3 % for qkv / o / wo; for the FFN wi GEMM, W-stationary 32 MB chunks won one of three runs
    // against this order and lost the other two, so the order stays.
    // vqa_set_gemm_schedule() / VQA_GEMM_GROUP_ROWS / VQA_GEMM_CHUNK_ROWS override (tuning).
    static const int env_rows = [] { const char* v = getenv("VQA_GEMM_GROUP_ROWS"); return (v && v[0]) ? atoi(v) : 0; }();
    static const int env_chunk = [] { const char* v = getenv("VQA_GEMM_CHUNK_ROWS"); return (v && v[0]) ? atoi(v) : 0; }();
    const int ov_rows = g_gemm_group_rows_override > 0 ? g_gemm_group_rows_override : env_rows;
    const int ov_chunk = g_gemm_chunk_rows_override != 0 ? g_gemm_chunk_rows_override : env_chunk;
    const long long w_bytes = (long long)g.w_rows * p.K * 2;
    const long long resident = 14ll << 20;
    const long long a_group_bytes = 12ll << 20;
    int group_rows, chunk_rows;   // chunk_rows < 0: no chunking (all N tiles in one chunk)
    if (w_bytes <= resident) {
        group_rows = 1024; chunk_rows = -1;                       // W stays in L2 as a whole, A streams once
    } else {
        const long long n_chunks = (w_bytes + resident - 1) / resident;
        if (n_chunks <= 3) {
            // W-stationary: up to three L2-resident chunks, A streams once per chunk
            const long long rows = ((long long)g.w_rows + n_chunks - 1) / n_chunks;
            chunk_rows = (int)((rows + BLOCK_N - 1) / BLOCK_N * BLOCK_N);
            group_rows = 1024;
        } else {
            // W much larger than L2: A-stationary groups, all of W streams past each
            chunk_rows = -1;
            group_rows = max(512, min(8192, (int)(a_group_bytes / ((long long)p.K * 2)) / 256 * 256));
        }
    }
    if (ov_rows > 0) group_rows = ov_rows;
    if (ov_chunk != 0) chunk_rows = ov_chunk;
    p.group_m = max(1, group_rows / rows_per_tile);
    // the gated epilogue's W tile holds BLOCK_N/2 gate rows + BLOCK_N/2 up rows: a chunk of `chunk_rows` W rows = chunk_rows / BLOCK_N tiles either way
    p.chunk_n = chunk_rows > 0 ? max(1, chunk_rows / BLOCK_N) : p.num_n_tiles;
    if (p.chunk_n > p.num_n_tiles) p.chunk_n = p.num_n_tiles;
    // L2 eviction hints on the operand streams: evict_normal on both by default (an evict_first tile can be dropped before the sibling
    // CTAs that share it have fetched it). VQA_GEMM_L2_POLICY=<a><w> with digits 0 normal / 1 first / 2 last overrides (tuning).
    static const int env_pol = [] { const char* v = getenv("VQA_GEMM_L2_POLICY"); return (v && v[0] && v[1]) ? (v[0] - '0') * 10 + (v[1] - '0') : -1; }();
    const unsigned long long pol[3] = {L2_EVICT_NORMAL, L2_EVICT_FIRST, L2_EVICT_LAST};
    p.a_policy = p.w_policy = L2_EVICT_NORMAL;
    if (env_pol >= 0 && env_pol / 10 < 3 && env_pol % 10 < 3) {
        p.a_policy = pol[env_pol / 10]; p.w_policy = pol[env_pol % 10];
    }
    const int num_tiles = p.num_m_tiles * p.num_n_tiles * p.num_batches;
    int workers = num_sms;
    if (workers > num_tiles) workers = num_tiles;
    if (workers < 1) workers = 1;

    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(workers);
    cfg.blockDim = dim3(Cfg::NUM_THREADS);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, ta, tb, tc, tr, p);
}

}  // namespace vqa

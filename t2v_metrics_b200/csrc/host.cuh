// Host layer shared by the model forwards: the handle, errors, profiling, GEMM and norm dispatch, the workspace plan and the
// forward context every launch of a forward goes through.
#pragma once
#include "../../include/vqa_b200.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <unordered_map>
#include <vector>

#include "ptx.cuh"
#include "gemm_sm90.cuh"
#include "elementwise.cuh"

using namespace vqa;
typedef __nv_bfloat16 bf16;

// bits of vqa_clipt5_config::emulate_bf16_rounding (see include/vqa_b200.h)
constexpr int VQA_FLAG_ROUND_DECODER = 1, VQA_FLAG_ROUND_ATTN_SCORES = 2, VQA_FLAG_FUSE_NORMS = 4;

// ------------------------------------------------------------------------------------------------ handle
struct BoundTensor {
    const void* data = nullptr;
    int64_t shape[4] = {0, 0, 0, 0};
    int ndim = 0;
};

struct VitLayerW {
    const bf16 *ln1_w, *ln1_b, *qkv_w, *qkv_b, *out_w, *out_b, *ln2_w, *ln2_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
};
struct T5EncLayerW {
    const bf16 *ln0, *qkv, *o, *ln1, *wi, *wo;
    const bf16 *qkv_g = nullptr, *wi_g = nullptr;   // fused-norm mode: qkv . diag(ln0), wi . diag(ln1) (gamma folded into the weight's K axis)
};
struct T5DecLayerW {
    const bf16 *ln0, *qkv, *o, *ln1, *cq, *ckv, *co, *ln2, *wi, *wo;
    const bf16* ckT;   // Wk^T [d_model, inner] for the absorbed cross-attention (optional)
};

struct QwenState;
struct vqa_handle {
    int kind = 0;               // 0: CLIP-FlanT5, 1: Qwen2.5-VL
    QwenState* qwen = nullptr;
    vqa_clipt5_config cfg;
    int num_sms = 132;
    std::string err;
    std::unordered_map<std::string, BoundTensor> tensors;
    bool finalized = false;
    int64_t launches = 0;
    int kpad = 0;  // padded K of the patch-embedding GEMM
    // resolved weights
    const bf16 *patch_w = nullptr, *cls = nullptr, *pos = nullptr, *pre_ln_w = nullptr, *pre_ln_b = nullptr;
    std::vector<VitLayerW> vit;
    const bf16 *proj0_w = nullptr, *proj0_b = nullptr, *proj2_w = nullptr, *proj2_b = nullptr;
    const bf16 *shared = nullptr, *enc_rel = nullptr, *dec_rel = nullptr, *enc_final_ln = nullptr,
               *dec_final_ln = nullptr, *lm_head = nullptr;
    std::vector<T5EncLayerW> enc;
    std::vector<T5DecLayerW> dec;
    // relative-position bucket LUTs (device), index rel + max_dist, rel clamped to [-max_dist, max_dist]
    int* lut_bidir = nullptr;
    int* lut_unidir = nullptr;
    // optional per-category device timing (vqa_set_profile): CUDA events around every launch of the forward
    bool profile = false;
    std::vector<cudaEvent_t> ev_pool;
    struct ProfRec { int cat; double flops; double bytes; int ev0, ev1; };
    std::vector<ProfRec> prof;
    size_t ev_used = 0;
};

enum ProfCat { CAT_GEMM = 0, CAT_ATTENTION = 1, CAT_NORM = 2, CAT_OTHER = 3, CAT_COUNT = 4 };

static thread_local std::string g_global_err;

static int fail(vqa_handle* h, int code, const std::string& msg) {
    if (h) h->err = msg; else g_global_err = msg;
    return code;
}

// VQA_OK, or VQA_ERR_CUDA with "what: <CUDA error>"
static int cuda_status(vqa_handle* h, cudaError_t e, const char* what) {
    return e == cudaSuccess ? VQA_OK : fail(h, VQA_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------ GEMM dispatch
static int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && v[0]) ? atoi(v) : dflt;
}

// Tile variants are named <BLOCK_N><rows / 128> (ABI values of vqa_op_gemm_bf16 and VQA_GEMM_VARIANT). sm_90a has no CTA-pair MMA, so the
// two-CTA names 2562 / 1282 select the same 128-row tile as 2561 / 1281.
template <int EPI, bool TMA_EPI>
static cudaError_t gemm_dispatch_variant(const GemmLaunch& g, int variant, int num_sms, cudaStream_t st) {
    switch (variant) {
        case 2562:
        case 2561: return launch_gemm_t<256, EPI, TMA_EPI>(g, num_sms, st);
        case 1282:
        case 1281: return launch_gemm_t<128, EPI, TMA_EPI>(g, num_sms, st);
        case 641:  return launch_gemm_t<64, EPI, TMA_EPI>(g, num_sms, st);
        case 321:
            if constexpr (epi_is_gated(EPI)) return cudaErrorInvalidValue;
            else return launch_gemm_t<32, EPI, TMA_EPI>(g, num_sms, st);
        default:   return cudaErrorInvalidValue;
    }
}

static int pick_variant(int M, int N, int epi) {
    static const int forced = env_int("VQA_GEMM_VARIANT", 0);
    if (forced) return forced;
    if (M <= 128) {
        // skinny (decoder rows): pure weight streaming; favour many CTAs. The gated epilogue pairs two half tiles of
        // BLOCK_N/2 >= 32 columns, so it needs BLOCK_N >= 64.
        if (epi_is_gated(epi)) return N <= 16384 ? 641 : 1281;
        if (N <= 4096) return 321;
        if (N <= 12288) return 641;
        return 1281;
    }
    // Measured on H100 (isolated CUDA-event times, one run): the 256-wide tile is 15-20 % faster at the encoder / vision shapes
    // (M >= 36928, N >= 1024, K = 4096: 686-693 vs 575-582 TFLOP/s); for M <= 4096 with N <= 1024 the two tiles are within a few percent
    // (M=4096 N=1024 K=4096: 599 with 128 vs 586 with 256; M=2308 N=1024 K=1024: 213 vs 233), and the 128-wide tile gives more CTAs.
    if (M <= 4096 && N <= 1024) return 1281;
    return 2561;
}

// partial sums per row that a residual-writing GEMM with this tile variant emits for N output columns (GemmParams::ssq_out)
static int ssq_parts_for(int variant, int N) {
    switch (variant) {
        case 2562:
        case 2561: return gemm_ssq_parts<256>(N);
        case 1282:
        case 1281: return gemm_ssq_parts<128>(N);
        case 641:  return gemm_ssq_parts<64>(N);
        default:   return gemm_ssq_parts<32>(N);
    }
}

// Split-K for skinny GEMMs (M <= 128 decoder rows x a 4096-row weight): 32 N tiles alone leave 100 of 132 SMs idle and cannot stream the
// weight at full HBM bandwidth, so the K range is cut into `splits` slices that run as the batches of ONE launch (fp32 partial tiles in `ws`),
// and this kernel adds the slices: C = [residual +] bf16(sum_s partial_s + bias) -- the Linear's bf16 output, then the residual add, like EPI_STORE.
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, int M, int N, const bf16* __restrict__ bias,
                                     const bf16* __restrict__ residual, int ldr, bf16* __restrict__ C, int ldc) {
    pdl_launch_dependents();
    const int nv = N / 8;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)M * nv) return;
    const int m = (int)(i / nv), n = (int)(i % nv) * 8;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < splits; ++s) {
        const float4* src = reinterpret_cast<const float4*>(part + ((size_t)s * M + m) * N + n);
        const float4 a = src[0], b = src[1];
        acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w; acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
    }
    if (bias) {
        const uint4 bb = __ldg(reinterpret_cast<const uint4*>(bias + n));
        const float2 b0 = unpack_bf16x2(bb.x), b1 = unpack_bf16x2(bb.y), b2 = unpack_bf16x2(bb.z), b3 = unpack_bf16x2(bb.w);
        acc[0] += b0.x; acc[1] += b0.y; acc[2] += b1.x; acc[3] += b1.y; acc[4] += b2.x; acc[5] += b2.y; acc[6] += b3.x; acc[7] += b3.y;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = bf16_round(acc[e]);
    if (residual) {
        const uint4 rr = *reinterpret_cast<const uint4*>(residual + (size_t)m * ldr + n);
        const float2 r0 = unpack_bf16x2(rr.x), r1 = unpack_bf16x2(rr.y), r2 = unpack_bf16x2(rr.z), r3 = unpack_bf16x2(rr.w);
        acc[0] += r0.x; acc[1] += r0.y; acc[2] += r1.x; acc[3] += r1.y; acc[4] += r2.x; acc[5] += r2.y; acc[6] += r3.x; acc[7] += r3.y;
    }
    *reinterpret_cast<uint4*>(C + (size_t)m * ldc + n) = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                                     pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
}

// number of K slices a skinny store-GEMM is cut into (1 = not worth it / not possible)
static int splitk_slices(int M, int N, int K, int num_sms) {
    static const int off = env_int("VQA_GEMM_SPLITK", 1) == 0;
    if (off || M > 128 || N % 8 || K < 2048) return 1;
    const int n_tiles = (N + 127) / 128;
    int s = num_sms / n_tiles;
    if (s > 8) s = 8;
    while (s >= 2 && K % (s * 64) != 0) --s;
    return s >= 2 ? s : 1;
}

constexpr int LMHEAD_BN = 128;
constexpr int LMHEAD_PARTS = GemmConfig<LMHEAD_BN>::LSE_PARTS;   // (max, sum) partials per (row, n tile)

struct NormFuse {            // fused RMSNorm hooks of one GEMM launch (see GemmParams::ssq_*)
    float* ssq_out = nullptr;       // producer: partial sums of squares of the rows this GEMM writes ([M, ssq_stride])
    const float* ssq_in = nullptr;  // consumer: partial sums of the rows of A
    int stride = 0;                 // floats per row in both buffers (multiple of 4; unused slots are zero)
    float inv_dim = 0.f, eps = 0.f;
};
// Batched launch: `nb` independent GEMMs sharing one tensor map per operand (see GemmParams::num_batches).
struct BatchSpec {
    int nb; int a_row_off, a_k_off, w_row_off, w_k_off; long long c_stride;
    long long a_rows, a_cols, w_rows, w_cols;   // full extents visible to TMA
};

// The kernel reads K in whole 64-column k blocks and clips them only at the operands' tensor-map extents (a_cols / w_cols, not K): with
// K % 64 != 0 the last k block of every batch multiplies columns K .. roundup(K, 64) of its A and W rows. Those products vanish only when
// one operand's extent ends at K, so that its tail reads TMA zero fill (that extent is then K wide, so the extents check has already
// forced its batches to k offset 0).
static bool batched_k_tail_ok(long long K, long long a_cols, long long w_cols) { return K % 64 == 0 || a_cols == K || w_cols == K; }

// One GEMM: C[M, N] = epi(A[M, K] . W[N, K]^T) and its optional parts. The constructor sets the dense layout (lda = ldw = K, N weight
// rows, ldc = N); the setters name what differs from it.
struct Gemm {
    const bf16* A; int lda;
    const bf16* W; int ldw, w_rows;
    void* C; int ldc;                          // bf16, fp32 with c_f32; unused by EPI_LSE
    int M, N, K;                               // N: columns of A W^T (2 x the output columns for the gated epilogues)
    int epi = EPI_STORE, gate_up_offset = 0;
    int variant = 0;                           // tile variant; 0 = pick_variant
    const bf16* bias = nullptr;
    const void* residual = nullptr; int ldr = 0;
    bool c_f32 = false;                        // EPI_STORE: C and the residual are fp32 (GemmParams::c_f32 = 1)
    int c_group_in = 0, c_group_out = 0;       // GemmParams::c_group_in
    NormFuse nf;
    BatchSpec batch = {};                      // batch.nb > 0: batched launch
    int k_slices = 0; float* splitk_ws = nullptr;   // > 0: split-K (splitk_reduce_kernel adds the fp32 slices in splitk_ws; two launches)
    // EPI_LSE (lm_head + log-softmax gather)
    const int* labels = nullptr; float *lse_max = nullptr, *lse_sum = nullptr, *label_logit = nullptr;
    float lse_scale = 1.0f; const uint32_t* penalty_bitmap = nullptr; int penalty_words = 0; float penalty = 1.0f;

    Gemm(const bf16* A_, const bf16* W_, void* C_, int M_, int N_, int K_)
        : A(A_), lda(K_), W(W_), ldw(K_), w_rows(N_), C(C_), ldc(N_), M(M_), N(N_), K(K_) {}
    Gemm& with_bias(const bf16* b) { bias = b; return *this; }
    Gemm& with_residual(const void* r) { residual = r; ldr = ldc; return *this; }        // same layout as C
    Gemm& with_epilogue(int e, int gate_up = 0) {   // a gated epilogue writes N / 2 dense columns
        epi = e; gate_up_offset = gate_up;
        if (epi_is_gated(e)) ldc = N / 2;
        return *this;
    }
    Gemm& accumulate_f32() { c_f32 = true; return with_residual(C); }                     // fp32 C += bf16(A W^T + bias)
    Gemm& with_norm(const NormFuse& n) { nf = n; return *this; }
    Gemm& batched(const BatchSpec& b, int tile_variant) { batch = b; variant = tile_variant; return *this; }
    Gemm& split_k(int slices, float* ws) { k_slices = slices; splitk_ws = ws; return *this; }
    Gemm& lse(const int* labels_, float* max, float* sum, float* label) {
        epi = EPI_LSE; labels = labels_; lse_max = max; lse_sum = sum; label_logit = label;
        return *this;
    }
    // the Qwen score's logit processing in the EPI_LSE epilogue: HF's repetition penalty on the ids set in bitmap [M, ceil(N / 32)] (none
    // when rep_penalty is 1), then 1 / temperature
    Gemm& processed(float temperature, const uint32_t* bitmap, float rep_penalty) {
        lse_scale = 1.0f / temperature;
        penalty_bitmap = rep_penalty != 1.0f ? bitmap : nullptr; penalty_words = (N + 31) / 32; penalty = rep_penalty;
        return *this;
    }
    // algorithmic work: A and W read once, C written once (+ residual read once); elem = bytes per C element, none for the lm_head
    double flops() const { return (batch.nb > 0 ? batch.nb : 1) * 2.0 * M * (double)N * K; }
    double bytes() const {
        const double n_out = epi_is_gated(epi) ? N / 2 : N, elem = epi == EPI_LSE ? 0 : c_f32 ? 4 : 2;
        return (batch.nb > 0 ? batch.nb : 1) * (2.0 * ((double)M * K + (double)N * K) + M * n_out * elem * (residual ? 2 : 1));
    }
};

// Validates and launches one GEMM (two launches for split-K). Returns cudaError_t.
static cudaError_t run_gemm(const Gemm& g, int num_sms, cudaStream_t st) {
    GemmLaunch L;
    L.A = g.A; L.lda = g.lda; L.W = g.W; L.ldw = g.ldw; L.w_rows = g.w_rows;
    GemmParams& p = L.p;
    memset(&p, 0, sizeof(p));
    p.M = g.M; p.N = g.N; p.K = g.K;
    if (g.epi == EPI_LSE) {
        if (!g.labels || !g.lse_max || !g.lse_sum || !g.label_logit) return cudaErrorInvalidValue;
        p.lse_max = g.lse_max; p.lse_sum = g.lse_sum; p.labels = g.labels; p.label_logit = g.label_logit; p.lse_scale = g.lse_scale;
        p.penalty_bitmap = g.penalty_bitmap; p.penalty_words = g.penalty_words; p.penalty = g.penalty;
        return launch_gemm_t<LMHEAD_BN, EPI_LSE, false>(L, num_sms, st);
    }
    bf16* C = static_cast<bf16*>(g.C);
    const bf16* residual = static_cast<const bf16*>(g.residual);
    if (g.k_slices > 0) {   // the K slices are the batches of one launch writing raw fp32 partial tiles
        const int Ks = g.K / g.k_slices;
        L.a_rows = g.M; L.a_cols = g.K; L.w_cols = g.K;
        p.K = Ks; p.C = reinterpret_cast<bf16*>(g.splitk_ws); p.ldc = g.N; p.c_f32 = 2;
        p.num_batches = g.k_slices; p.a_k_off = Ks; p.w_k_off = Ks; p.c_batch_stride = (long long)g.M * g.N;
        cudaError_t e = gemm_dispatch_variant<EPI_STORE, false>(L, 1281, num_sms, st);
        if (e != cudaSuccess) return e;
        const long long n = (long long)g.M * (g.N / 8);
        splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g.splitk_ws, g.k_slices, g.M, g.N, g.bias, residual, g.ldr, C, g.ldc);
        return cudaGetLastError();
    }
    if (g.batch.nb > 0) {
        const BatchSpec& bs = g.batch;
        if (!batched_k_tail_ok(g.K, bs.a_cols, bs.w_cols)) return cudaErrorInvalidValue;
        L.w_rows = (int)bs.w_rows; L.a_rows = bs.a_rows; L.a_cols = bs.a_cols; L.w_cols = bs.w_cols;
        p.num_batches = bs.nb; p.a_row_off = bs.a_row_off; p.a_k_off = bs.a_k_off; p.w_row_off = bs.w_row_off;
        p.w_k_off = bs.w_k_off; p.c_batch_stride = bs.c_stride;
    }
    p.C = C; p.ldc = g.ldc; p.bias = g.bias; p.residual = residual; p.ldr = g.ldr; p.gate_up_offset = g.gate_up_offset;
    if (g.c_f32 && g.epi != EPI_STORE) return cudaErrorInvalidValue;
    p.c_f32 = g.c_f32 ? 1 : 0;
    if (g.c_group_in > 0) {   // narrow output column groups written into wider slots (GemmParams::c_group_in)
        if (g.epi != EPI_STORE || residual || g.c_f32 || (g.c_group_in & 7) || (g.c_group_out & 7) || g.c_group_out < g.c_group_in ||
            g.N % g.c_group_in)
            return cudaErrorInvalidValue;
        p.c_group_in = g.c_group_in; p.c_group_out = g.c_group_out;
    }
    const NormFuse& nf = g.nf;
    p.ssq_out = nf.ssq_out; p.ssq_in = nf.ssq_in; p.ssq_out_parts = p.ssq_in_parts = nf.stride;
    p.ssq_inv_dim = nf.inv_dim; p.ssq_eps = nf.eps;
    if (nf.ssq_out && (g.epi != EPI_STORE || g.c_f32)) return cudaErrorInvalidValue;
    const int variant = g.variant ? g.variant : pick_variant(g.M, g.N, g.epi);
    // Dense bf16 outputs take the TMA-store epilogue. The staged one keeps what a box store cannot do with the same bits: fp32 C, the
    // batched launches (whose gap rows between batches keep their contents), the scattered column groups and the per-row sums of squares
    // (their summation order). Those are plain stores; the other epilogues have only the TMA-store path.
    if (g.batch.nb > 0 || g.c_f32 || g.c_group_in > 0 || nf.ssq_out)
        return g.epi == EPI_STORE ? gemm_dispatch_variant<EPI_STORE, false>(L, variant, num_sms, st) : cudaErrorInvalidValue;
    switch (g.epi) {
        case EPI_STORE:      return gemm_dispatch_variant<EPI_STORE, true>(L, variant, num_sms, st);
        case EPI_QUICK_GELU: return gemm_dispatch_variant<EPI_QUICK_GELU, true>(L, variant, num_sms, st);
        case EPI_GELU_ERF:   return gemm_dispatch_variant<EPI_GELU_ERF, true>(L, variant, num_sms, st);
        case EPI_GATED_GELU: return gemm_dispatch_variant<EPI_GATED_GELU, true>(L, variant, num_sms, st);
        case EPI_RELU:       return gemm_dispatch_variant<EPI_RELU, true>(L, variant, num_sms, st);
        case EPI_GATED_SILU: return gemm_dispatch_variant<EPI_GATED_SILU, true>(L, variant, num_sms, st);
        default:             return cudaErrorInvalidValue;
    }
}

// ------------------------------------------------------------------------------------------------ norm dispatch
static cudaError_t run_rmsnorm(const bf16* x, const bf16* w, bf16* y, int rows, int D, float eps, cudaStream_t st) {
    if (rows <= 0) return cudaSuccess;
    if (D % 256 == 0 && D < 4096) {
        const int blocks = (rows + 7) / 8;      // one warp per row
#define VQA_RMS_CASE(NV) case NV: t5_rmsnorm_warp_kernel<NV><<<blocks, 256, 0, st>>>(x, w, y, rows, eps); break;
        switch (D / 256) {
            VQA_RMS_CASE(1) VQA_RMS_CASE(2) VQA_RMS_CASE(3) VQA_RMS_CASE(4) VQA_RMS_CASE(5) VQA_RMS_CASE(6) VQA_RMS_CASE(7) VQA_RMS_CASE(8)
            VQA_RMS_CASE(9) VQA_RMS_CASE(10) VQA_RMS_CASE(11) VQA_RMS_CASE(12) VQA_RMS_CASE(13) VQA_RMS_CASE(14) VQA_RMS_CASE(15)
        }
#undef VQA_RMS_CASE
        return cudaGetLastError();
    }
    const int nvec = D / 8;
    if (D % 8) return cudaErrorInvalidValue;
    if (nvec <= 256)       t5_rmsnorm_kernel<1><<<rows, 256, 0, st>>>(x, w, y, D, eps);
    else if (nvec <= 512)  t5_rmsnorm_kernel<2><<<rows, 256, 0, st>>>(x, w, y, D, eps);
    else if (nvec <= 1024) t5_rmsnorm_kernel<4><<<rows, 256, 0, st>>>(x, w, y, D, eps);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}
// LayerNorm of an fp32 stream (the CLIP residual under autocast) -> bf16
static cudaError_t run_layernorm_f32(const float* x, const bf16* g, const bf16* b, bf16* y, int rows, int D, float eps, cudaStream_t st) {
    const int blocks = (rows + 7) / 8;
    if (D == 1024)      layernorm_kernel<1024, float><<<blocks, 256, 0, st>>>(x, g, b, y, rows, eps);
    else if (D == 256)  layernorm_kernel<256, float><<<blocks, 256, 0, st>>>(x, g, b, y, rows, eps);
    else if (D == 512)  layernorm_kernel<512, float><<<blocks, 256, 0, st>>>(x, g, b, y, rows, eps);
    else if (D == 768)  layernorm_kernel<768, float><<<blocks, 256, 0, st>>>(x, g, b, y, rows, eps);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ weights and workspace plan
static const bf16* need(vqa_handle* h, const std::string& name, int64_t d0, int64_t d1, bool& ok) {
    auto it = h->tensors.find(name);
    if (it == h->tensors.end()) {
        if (ok) h->err = "missing weight: " + name;
        ok = false;
        return nullptr;
    }
    const BoundTensor& b = it->second;
    int64_t numel = 1;
    for (int d = 0; d < b.ndim; ++d) numel *= b.shape[d];
    if (numel != d0 * d1) {
        if (ok) {
            char buf[256];
            snprintf(buf, sizeof buf, "weight %s: expected %lld x %lld elements, got %lld", name.c_str(), (long long)d0,
                     (long long)d1, (long long)numel);
            h->err = buf;
        }
        ok = false;
        return nullptr;
    }
    return reinterpret_cast<const bf16*>(b.data);
}

struct Plan {
    size_t off = 0;
    size_t take(size_t bytes) {
        size_t o = off;
        off += (bytes + 255) & ~size_t(255);
        return o;
    }
};

// ------------------------------------------------------------------------------------------------ forward context
// Everything a forward enqueues goes through one of these calls. Each counts its own launches (vqa_last_launch_count), opens a profiling
// scope of its category when profiling is on, and turns a launch error into VQA_ERR_CUDA naming the stage. Returns a vqa_status.
struct Forward {
    vqa_handle* h;
    cudaStream_t st;
    uint8_t* ws;
    int nsm;
    int depth = 0;   // open profiling scopes

    Forward(vqa_handle* h_, void* workspace, cudaStream_t st_) : h(h_), st(st_), ws(static_cast<uint8_t*>(workspace)), nsm(h_->num_sms) {
        h->launches = 0;
        h->prof.clear();
        h->ev_used = 0;
    }
    template <typename T = bf16>
    T* at(size_t off) const { return reinterpret_cast<T*>(ws + off); }

    // Records an event pair around the launches issued in its lifetime (profile mode only). A scope opened inside another one records
    // nothing: a group of launches counts as one scope of the outer category.
    struct Scope {
        Forward& f;
        int idx = -1;
        Scope(Forward& f_, int cat, double flops = 0.0, double bytes = 0.0) : f(f_) {
            vqa_handle* h = f.h;
            if (f.depth++ > 0 || !h->profile) return;
            while (h->ev_pool.size() < h->ev_used + 2) {
                cudaEvent_t e;
                if (cudaEventCreate(&e) != cudaSuccess) return;
                h->ev_pool.push_back(e);
            }
            vqa_handle::ProfRec r{cat, flops, bytes, (int)h->ev_used, (int)h->ev_used + 1};
            h->ev_used += 2;
            cudaEventRecord(h->ev_pool[r.ev0], f.st);
            idx = (int)h->prof.size();
            h->prof.push_back(r);
        }
        ~Scope() {
            --f.depth;
            if (idx >= 0) cudaEventRecord(f.h->ev_pool[f.h->prof[idx].ev1], f.st);
        }
    };
    Scope group(int cat) { return Scope(*this, cat); }

    // `n` launches issued by enqueue() (returns cudaError_t) as one scope
    template <typename F>
    int op(int cat, double flops, double bytes, int n, const char* what, F&& enqueue) {
        Scope s(*this, cat, flops, bytes);
        h->launches += n;
        return cuda_status(h, enqueue(), what);
    }
    template <typename... KArgs, typename... Args>
    int launch(int cat, double flops, const char* what, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args... args) {
        return op(cat, flops, 0.0, 1, what, [&] {
            kernel<<<grid, block, smem, st>>>(args...);
            return cudaGetLastError();
        });
    }
    int memset0(void* p, size_t bytes, const char* what) {
        return op(CAT_OTHER, 0.0, 0.0, 1, what, [&] { return cudaMemsetAsync(p, 0, bytes, st); });
    }
    int copy(void* dst, const void* src, size_t bytes, const char* what) {
        return op(CAT_OTHER, 0.0, 0.0, 1, what, [&] { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st); });
    }
    int gemm(const Gemm& g, const char* what = "gemm") {
        return op(CAT_GEMM, g.flops(), g.bytes(), g.k_slices > 0 ? 2 : 1, what, [&] { return run_gemm(g, nsm, st); });
    }
    // one launch of launch_attn_tc / launch_attn_tc128 on this->st
    template <typename F>
    int attention(double flops, const char* what, F&& enqueue) { return op(CAT_ATTENTION, flops, 0.0, 1, what, enqueue); }
    int rmsnorm(const bf16* x, const bf16* w, bf16* y, int rows, int D, float eps) {
        return op(CAT_NORM, 0.0, 0.0, 1, "rmsnorm", [&] { return run_rmsnorm(x, w, y, rows, D, eps, st); });
    }
    int layernorm_f32(const float* x, const bf16* g, const bf16* b, bf16* y, int rows, int D, float eps) {
        return op(CAT_NORM, 0.0, 0.0, 1, "layernorm", [&] { return run_layernorm_f32(x, g, b, y, rows, D, eps, st); });
    }
};
#define TRY(x) do { int _rc = (x); if (_rc) return _rc; } while (0)

// The score's tail of both forwards: the EPI_LSE lm_head GEMM g (M = B * T rows) with its (max, sum) partials and label logits, then
// lse_finalize_kernel into scores [B] and, unless NULL, logprobs [B * T].
static int lmhead_score(Forward& f, Gemm g, const int* labels, float* lse_max, float* lse_sum, float* label_logit, float* scores,
                        float* logprobs, int B, int T) {
    const int ntiles = LMHEAD_PARTS * ((g.N + LMHEAD_BN - 1) / LMHEAD_BN);
    TRY(f.gemm(g.lse(labels, lse_max, lse_sum, label_logit), "lm_head"));
    return f.launch(CAT_OTHER, 0, "lse finalize", lse_finalize_kernel, (B + 3) / 4, 128, 0, (const float*)lse_max, (const float*)lse_sum,
                    (const float*)label_logit, labels, scores, logprobs, B, T, ntiles);
}

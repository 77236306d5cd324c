// Host-side orchestration of the Qwen2.5-VL VQAScore forward: P(answer token | image, question) for a batch of prompts
// in ONE prefill (the reference runs generate(max_new_tokens=1) per sample: qwen2vl_model.py:190-230).
#pragma once
#include "host.cuh"
#include "attention_sm90.cuh"
#include "qwen_kernels.cuh"
#include "qwen_decode.cuh"

struct QwenVisLayerW {
    const bf16 *norm1, *norm2, *qkv_w, *qkv_b, *proj_w, *proj_b, *gu_w, *gu_b, *down_w, *down_b;
};
struct QwenLlmLayerW {
    const bf16 *ln1, *ln2, *qkv_w, *qkv_b, *o_w, *gu_w, *down_w;
};
struct QwenState {
    vqa_qwen25vl_config cfg;
    const bf16 *patch_w = nullptr, *merger_ln = nullptr, *fc1_w = nullptr, *fc1_b = nullptr, *fc2_w = nullptr, *fc2_b = nullptr;
    const bf16 *embed = nullptr, *final_norm = nullptr, *lm_head = nullptr;
    std::vector<QwenVisLayerW> vis;
    std::vector<QwenLlmLayerW> llm;
    // rotary metadata (device): axis of each frequency index and its inverse frequency
    int *text_axis = nullptr, *vis_axis = nullptr;
    float *text_inv_freq = nullptr, *vis_inv_freq = nullptr;
    bool rope_set = false;
};

static inline int qwen_mlp_pad(int mlp) { return (mlp + 127) / 128 * 128; }

struct QwenWorkspace {
    size_t patches, vx, vxn, vqkv, vattn, vff, vmerge_in, vfc1, vfeat, vfeat_orig, vcos, vsin;
    size_t x, xn, qkv, attn, ff, cos, sin, last, lastn, lse_max, lse_sum, label_logit, logprob, pen_bitmap, trace_logits;
    size_t total;
};
// B = prompts scored, M = token rows of the language model (B * S in the padded layout; fewer when prompts share a vision prefix)
static QwenWorkspace qwen_plan_rows(const vqa_qwen25vl_config& c, int B, size_t M, int n_patches) {
    Plan pl;
    QwenWorkspace w;
    const size_t L = n_patches;
    const size_t unit = (size_t)c.spatial_merge * c.spatial_merge;
    const size_t Dv = c.vit_hidden, Hv = c.vit_heads;
    const size_t mlp_pad = qwen_mlp_pad(c.vit_mlp);
    w.patches = pl.take(L * c.patch_dim * 2);
    w.vx = pl.take(L * Dv * 2);
    w.vxn = pl.take(L * Dv * 2);
    w.vqkv = pl.take(L * 3 * Hv * 128 * 2);
    w.vattn = pl.take(L * Hv * 128 * 2);      // used as [L, Hv * head_dim] (compact heads)
    w.vff = pl.take(L * mlp_pad * 2);
    w.vmerge_in = pl.take(L * Dv * 2);
    w.vfc1 = pl.take(L / unit * (Dv * unit) * 2);
    w.vfeat = pl.take(L / unit * c.out_hidden * 2);
    w.vfeat_orig = pl.take(L / unit * c.out_hidden * 2);
    w.vcos = pl.take(L * c.vit_head_dim * 4);
    w.vsin = pl.take(L * c.vit_head_dim * 4);
    const size_t qkv_cols = (size_t)(c.heads + 2 * c.kv_heads) * 128;
    w.x = pl.take(M * c.hidden * 2);
    w.xn = pl.take(M * c.hidden * 2);
    w.qkv = pl.take(M * qkv_cols * 2);
    w.attn = pl.take(M * c.heads * 128 * 2);
    w.ff = pl.take(M * c.mlp * 2);
    w.cos = pl.take(M * 128 * 4);
    w.sin = pl.take(M * 128 * 4);
    w.last = pl.take((size_t)B * c.hidden * 2);
    w.lastn = pl.take((size_t)B * c.hidden * 2);
    const size_t ntiles = (size_t)LMHEAD_PARTS * ((c.vocab + LMHEAD_BN - 1) / LMHEAD_BN);
    w.lse_max = pl.take((size_t)B * ntiles * 4);
    w.lse_sum = pl.take((size_t)B * ntiles * 4);
    w.label_logit = pl.take((size_t)B * 4);
    w.logprob = pl.take((size_t)B * 4);
    w.pen_bitmap = pl.take((size_t)B * ((c.vocab + 31) / 32) * 4);
    w.trace_logits = pl.take((size_t)B * c.vocab * 2);      // only written by vqa_qwen25vl_topk (trace output); the scoring path never stores logits
    w.total = pl.off;
    return w;
}

static int qwen_finalize(vqa_handle* h, QwenState& q) {
    const vqa_qwen25vl_config& c = q.cfg;
    bool ok = true;
    const int Dv = c.vit_hidden, Hv = c.vit_heads, unit = c.spatial_merge * c.spatial_merge, mlp_pad = qwen_mlp_pad(c.vit_mlp);
    q.patch_w = need(h, "vis.patch_embed", Dv, c.patch_dim, ok);
    q.vis.resize(c.vit_depth);
    for (int i = 0; i < c.vit_depth; ++i) {
        const std::string p = "vis." + std::to_string(i) + ".";
        QwenVisLayerW& L = q.vis[i];
        L.norm1 = need(h, p + "norm1", Dv, 1, ok); L.norm2 = need(h, p + "norm2", Dv, 1, ok);
        // native head width (80 for Qwen2.5-VL): the HF qkv weight is already ordered (q|k|v, head, dim); the GEMM epilogue scatters each head's
        // columns into the 128-wide slots the attention kernel reads, the attention writes compact heads, proj contracts over Hv * head_dim
        L.qkv_w = need(h, p + "qkv.weight", 3 * Hv * c.vit_head_dim, Dv, ok); L.qkv_b = need(h, p + "qkv.bias", 3 * Hv * c.vit_head_dim, 1, ok);
        L.proj_w = need(h, p + "proj.weight", Dv, Hv * c.vit_head_dim, ok); L.proj_b = need(h, p + "proj.bias", Dv, 1, ok);
        L.gu_w = need(h, p + "gate_up.weight", 2 * mlp_pad, Dv, ok); L.gu_b = need(h, p + "gate_up.bias", 2 * mlp_pad, 1, ok);
        L.down_w = need(h, p + "down.weight", Dv, mlp_pad, ok); L.down_b = need(h, p + "down.bias", Dv, 1, ok);
    }
    q.merger_ln = need(h, "vis.merger.ln_q", Dv, 1, ok);
    q.fc1_w = need(h, "vis.merger.fc1.weight", Dv * unit, Dv * unit, ok); q.fc1_b = need(h, "vis.merger.fc1.bias", Dv * unit, 1, ok);
    q.fc2_w = need(h, "vis.merger.fc2.weight", c.out_hidden, Dv * unit, ok); q.fc2_b = need(h, "vis.merger.fc2.bias", c.out_hidden, 1, ok);
    const int D = c.hidden, qkv_rows = (c.heads + 2 * c.kv_heads) * 128;
    q.embed = need(h, "llm.embed", c.vocab, D, ok);
    q.final_norm = need(h, "llm.norm", D, 1, ok);
    q.lm_head = need(h, "llm.lm_head", c.vocab, D, ok);
    q.llm.resize(c.layers);
    for (int i = 0; i < c.layers; ++i) {
        const std::string p = "llm." + std::to_string(i) + ".";
        QwenLlmLayerW& L = q.llm[i];
        L.ln1 = need(h, p + "ln1", D, 1, ok); L.ln2 = need(h, p + "ln2", D, 1, ok);
        L.qkv_w = need(h, p + "qkv.weight", qkv_rows, D, ok); L.qkv_b = need(h, p + "qkv.bias", qkv_rows, 1, ok);
        L.o_w = need(h, p + "o.weight", D, c.heads * 128, ok);
        L.gu_w = need(h, p + "gate_up.weight", 2 * c.mlp, D, ok);
        L.down_w = need(h, p + "down.weight", D, c.mlp, ok);
    }
    if (!ok) return VQA_ERR_MISSING_WEIGHT;
    if (!q.rope_set) return fail(h, VQA_ERR_INVALID_ARG, "vqa_qwen25vl_set_rope has not been called");
    return VQA_OK;
}

// ------------------------------------------------------------------------------------------------ glue launches (see clipt5.cuh)

// cos / sin tables [rows, 2 * half] of the positions pos [n_axes, rows]; round_bf16: the text model's bf16 tables.
static int qwen_rope_table(Forward& f, const char* what, const int* pos, int rows, const int* axis_of_dim, const float* inv_freq, int half,
                           float* cos_t, float* sin_t, int round_bf16) {
    return f.launch(CAT_OTHER, 0, what, rope_table_kernel, (unsigned)(((long long)rows * half + GLUE_THREADS - 1) / GLUE_THREADS), GLUE_THREADS,
                    0, pos, rows, axis_of_dim, inv_freq, half, cos_t, sin_t, round_bf16);
}

// In-place rotary embedding of n_heads heads (head h at column col0 + h * head_stride) of x [rows, ld] with the tables of qwen_rope_table.
static int qwen_rope(Forward& f, const char* what, bf16* x, int ld, int col0, int n_heads, int head_stride, int head_dim, const float* cos_t,
                     const float* sin_t, long long rows, int bf16_products) {
    return f.launch(CAT_OTHER, 0, what, rope_inplace_kernel, (unsigned)((rows * n_heads * (head_dim / 16) + GLUE_THREADS - 1) / GLUE_THREADS),
                    GLUE_THREADS, 0, x, ld, col0, n_heads, head_stride, head_dim, cos_t, sin_t, rows, bf16_products);
}

// dst row r = src row index[r / group] * group + r % group, for r < rows.
static int qwen_gather_rows(Forward& f, const char* what, const bf16* src, bf16* dst, const int* index, int rows, int group, int D) {
    return f.launch(CAT_OTHER, 0, what, gather_rows_kernel, rows, ROW_COPY_THREADS, 0, src, dst, index, group, D);
}

// The language model's input out [rows, D]: row b * S + s < seq_lens[b] takes feats[feat_index] or embed[ids], the rest zero.
static int qwen_embed(Forward& f, const int* ids, const int* feat_index, const int* seq_lens, const bf16* embed, const bf16* feats, bf16* out,
                      int rows, int S, int D) {
    return f.launch(CAT_OTHER, 0, "llm embed", qwen_embed_kernel, rows, ROW_COPY_THREADS, 0, ids, feat_index, seq_lens, embed, feats, out, S, D);
}

// The prompt ids OR-ed into the repetition-penalty bitmap [B, ceil(vocab / 32)]: padded rows ids [B, S] up to seq_lens[b] ...
static int qwen_token_bitmap(Forward& f, const int* ids, const int* seq_lens, int B, int S, int vocab, uint32_t* bitmap) {
    return f.launch(CAT_OTHER, 0, "penalty bitmap", token_bitmap_kernel, (unsigned)(((long long)B * S + GLUE_THREADS - 1) / GLUE_THREADS),
                    GLUE_THREADS, 0, ids, seq_lens, B, S, vocab, bitmap, token_bitmap_words(vocab));
}
// ... or packed rows: pair b's prompt is its prefix sequence (kv_prefix[pair_seq[b]], if any) and its own sequence
static int qwen_token_bitmap_packed(Forward& f, const int* ids, const int* cu_seqlens, const int* kv_prefix, const int* pair_seq, int max_prompt_len,
                                    int B, int vocab, uint32_t* bitmap) {
    return f.launch(CAT_OTHER, 0, "penalty bitmap", token_bitmap_packed_kernel, dim3((max_prompt_len + GLUE_THREADS - 1) / GLUE_THREADS, B),
                    GLUE_THREADS, 0, ids, cu_seqlens, kv_prefix, pair_seq, vocab, bitmap, token_bitmap_words(vocab));
}

// The K most probable ids of every row of logits [B, ldl] (first V columns) under the score's processing: the repetition penalty on the
// ids set in pen_bitmap (none when the penalty is 1), then 1 / temperature.
static int qwen_topk_softmax(Forward& f, const bf16* logits, long long ldl, int B, int V, float temperature, const uint32_t* pen_bitmap,
                             float penalty, int K, int* out_ids, float* out_probs) {
    return f.launch(CAT_OTHER, 0, "top-k softmax", topk_softmax_kernel, B, GLUE_THREADS, 0, logits, ldl, V, 1.0f / temperature,
                    penalty != 1.0f ? pen_bitmap : nullptr, token_bitmap_words(V), penalty, K, out_ids, out_probs);
}

// ------------------------------------------------------------------------------------------------ forward
// K/V cache of a generate prefill: layer l's K and V at kc + l * layer_elems and vc + l * layer_elems, each [B, Hkv, cap, 128]
struct QwenKVCache {
    bf16 *kc, *vc;
    size_t layer_elems;
    int cap;
};

// Vision tower, embedding splice and every language-model layer of one prefill, into w.x. With `kv`, each layer's post-rope K/V rows are
// also stored in the cache (one launch per layer after the rope).
static int qwen_prefill(Forward& f, QwenState& q, const QwenWorkspace& w, const vqa_qwen25vl_prompts& in, const vqa_qwen25vl_packed* pk,
                        const QwenKVCache* kv = nullptr) {
    const vqa_qwen25vl_config& c = q.cfg;
    cudaStream_t st = f.st;
    const void* pixel_patches = in.pixel_patches;
    const int pixel_dtype = in.pixel_dtype, n_patches = in.n_patches, B = in.batch, S = pk ? pk->total_rows : in.seq_len;
    const int *vis_pos_hw = in.vis_pos_hw, *window_index = in.window_index, *reverse_index = in.reverse_index, *cu_window = in.cu_window;
    const int n_windows = in.n_windows, max_window_len = in.max_window_len, n_frames = in.n_frames, max_frame_len = in.max_frame_len;
    const int *cu_frames = in.cu_frames, *input_ids = in.input_ids, *seq_lens = in.seq_lens, *feat_index = in.feat_index;
    const int* position_ids = in.position_ids;
    auto P_ = [&](size_t off) { return f.at(off); };
    auto F_ = [&](size_t off) { return f.at<float>(off); };
    const int L = n_patches, Dv = c.vit_hidden, Hv = c.vit_heads, hdv = c.vit_head_dim;
    const int unit = c.spatial_merge * c.spatial_merge, mlp_pad = qwen_mlp_pad(c.vit_mlp);
    const int D = c.hidden, M = pk ? pk->total_rows : B * S;

    // ---------------- vision tower ----------------
    {
        auto g = f.group(CAT_OTHER);
        const size_t n = (size_t)L * c.patch_dim;
        if (pixel_dtype == VQA_DTYPE_F32)
            TRY(f.launch(CAT_OTHER, 0, "pixel cast", cast_f32_bf16_kernel, (unsigned)((n / 4 + 255) / 256 + 1), 256, 0,
                         reinterpret_cast<const float*>(pixel_patches), P_(w.patches), n));
        else
            TRY(f.copy(P_(w.patches), pixel_patches, n * 2, "pixel copy"));
        // rotary table of the (already window-ordered) patch positions: [h freqs | w freqs] duplicated (:404-409, :487)
        TRY(qwen_rope_table(f, "vision rope table", vis_pos_hw, L, q.vis_axis, q.vis_inv_freq, hdv / 2, F_(w.vcos), F_(w.vsin), 0));
    }
    // patch embedding (Conv3d == GEMM), then re-order 2x2 groups into window order (:470-472)
    TRY(f.gemm(Gemm(P_(w.patches), q.patch_w, P_(w.vxn), L, Dv, c.patch_dim)));
    {
        auto g = f.group(CAT_OTHER);
        TRY(qwen_gather_rows(f, "window reorder", P_(w.vxn), P_(w.vx), window_index, L, unit, Dv));
        // the qkv GEMMs write head_dim of every 128-wide head slot; the attention kernel contracts q.k over all 128: zero the rest once
        if (hdv < 128) TRY(f.memset0(P_(w.vqkv), (size_t)L * 3 * Hv * 128 * 2, "vision qkv clear"));
    }
    const float vscale = 1.0f / sqrtf((float)hdv);
    for (int l = 0; l < c.vit_depth; ++l) {
        const QwenVisLayerW& Lw = q.vis[l];
        const bool full = (c.fullatt_mask >> l) & 1ull;
        TRY(f.rmsnorm(P_(w.vx), Lw.norm1, P_(w.vxn), L, Dv, c.rms_eps));
        Gemm qkv(P_(w.vxn), Lw.qkv_w, P_(w.vqkv), L, 3 * Hv * hdv, Dv);
        qkv.ldc = 3 * Hv * 128;
        if (hdv < 128) { qkv.c_group_in = hdv; qkv.c_group_out = 128; }
        TRY(f.gemm(qkv.with_bias(Lw.qkv_b), "vision qkv gemm"));
        TRY(qwen_rope(f, "vision rope", P_(w.vqkv), 3 * Hv * 128, 0, 2 * Hv, 128, hdv, F_(w.vcos), F_(w.vsin), L, 0));
        const int nseq = full ? n_frames : n_windows, mlen = full ? max_frame_len : max_window_len;
        static const bool no_pairs = getenv("VQA_ATTN128_NO_PAIRS") != nullptr;     // A/B switch
        TRY(f.attention(4.0 * (double)L * mlen * Hv * hdv, "vision attention", [&] {
            return launch_attn_tc128(P_(w.vqkv), 3 * Hv * 128, L, 0, Hv * 128, 2 * Hv * 128, P_(w.vattn), Hv * hdv, nseq, mlen, 0, Hv, 1,
                                     full ? cu_frames : cu_window, nullptr, vscale, false, st, nullptr,
                                     /*two windows per tile*/ !full && max_window_len <= 64 && !no_pairs, /*compact heads*/ hdv, hdv);
        }));
        TRY(f.gemm(Gemm(P_(w.vattn), Lw.proj_w, P_(w.vx), L, Dv, Hv * hdv).with_bias(Lw.proj_b).with_residual(P_(w.vx))));
        TRY(f.rmsnorm(P_(w.vx), Lw.norm2, P_(w.vxn), L, Dv, c.rms_eps));
        TRY(f.gemm(Gemm(P_(w.vxn), Lw.gu_w, P_(w.vff), L, 2 * mlp_pad, Dv).with_bias(Lw.gu_b).with_epilogue(EPI_GATED_SILU, mlp_pad)));
        TRY(f.gemm(Gemm(P_(w.vff), Lw.down_w, P_(w.vx), L, Dv, mlp_pad).with_bias(Lw.down_b).with_residual(P_(w.vx))));
    }
    // merger: RMSNorm -> [L/4, 4*Dv] -> Linear + GELU -> Linear; back to the original token order (:144-146, :512-513)
    TRY(f.rmsnorm(P_(w.vx), q.merger_ln, P_(w.vmerge_in), L, Dv, c.rms_eps));
    TRY(f.gemm(Gemm(P_(w.vmerge_in), q.fc1_w, P_(w.vfc1), L / unit, Dv * unit, Dv * unit).with_bias(q.fc1_b).with_epilogue(EPI_GELU_ERF)));
    TRY(f.gemm(Gemm(P_(w.vfc1), q.fc2_w, P_(w.vfeat), L / unit, c.out_hidden, Dv * unit).with_bias(q.fc2_b)));
    {
        auto g = f.group(CAT_OTHER);
        TRY(qwen_gather_rows(f, "merger reorder", P_(w.vfeat), P_(w.vfeat_orig), reverse_index, L / unit, 1, c.out_hidden));
        // ---------------- language model input ----------------
        // packed rows: one "sample" of M rows, all valid (its length is the last entry of cu_seqlens)
        TRY(qwen_embed(f, input_ids, feat_index, pk ? pk->cu_seqlens + pk->n_seq : seq_lens, q.embed, P_(w.vfeat_orig), P_(w.x), M, pk ? M : S, D));
        TRY(qwen_rope_table(f, "llm rope table", position_ids, M, q.text_axis, q.text_inv_freq, 64, F_(w.cos), F_(w.sin), 1));
    }
    const int Hq = c.heads, Hkv = c.kv_heads, qkv_cols = (Hq + 2 * Hkv) * 128;
    const float tscale = 1.0f / sqrtf(128.0f);
    for (int l = 0; l < c.layers; ++l) {
        const QwenLlmLayerW& Lw = q.llm[l];
        TRY(f.rmsnorm(P_(w.x), Lw.ln1, P_(w.xn), M, D, c.rms_eps));
        TRY(f.gemm(Gemm(P_(w.xn), Lw.qkv_w, P_(w.qkv), M, qkv_cols, D).with_bias(Lw.qkv_b)));
        // q heads and k heads are contiguous in the packed buffer -> one launch rotates Hq + Hkv heads
        TRY(qwen_rope(f, "llm rope", P_(w.qkv), qkv_cols, 0, Hq + Hkv, 128, 128, F_(w.cos), F_(w.sin), M, c.emulate_bf16_rounding));
        if (kv)
            TRY(kv_cache_write(f, P_(w.qkv), qkv_cols, Hq * 128, (Hq + Hkv) * 128, Hkv, S, M, seq_lens, nullptr, kv->kc + l * kv->layer_elems,
                               kv->vc + l * kv->layer_elems, kv->cap));
        TRY(f.attention(2.0 * B * (double)Hq * S * S * 128, pk ? "llm attention (packed)" : "llm attention", [&] {
            if (pk)
                return launch_attn_tc128(P_(w.qkv), qkv_cols, M, 0, Hq * 128, (Hq + Hkv) * 128, P_(w.attn), Hq * 128, pk->n_seq, pk->max_seq_len,
                                         0, Hq, Hq / Hkv, pk->cu_seqlens, nullptr, tscale, true, st, pk->kv_prefix);
            return launch_attn_tc128(P_(w.qkv), qkv_cols, M, 0, Hq * 128, (Hq + Hkv) * 128, P_(w.attn), Hq * 128, B, S, S, Hq, Hq / Hkv, nullptr,
                                     seq_lens, tscale, true, st);
        }));
        TRY(f.gemm(Gemm(P_(w.attn), Lw.o_w, P_(w.x), M, D, Hq * 128).with_residual(P_(w.x))));
        TRY(f.rmsnorm(P_(w.x), Lw.ln2, P_(w.xn), M, D, c.rms_eps));
        TRY(f.gemm(Gemm(P_(w.xn), Lw.gu_w, P_(w.ff), M, 2 * c.mlp, D).with_epilogue(EPI_GATED_SILU, c.mlp)));
        TRY(f.gemm(Gemm(P_(w.ff), Lw.down_w, P_(w.x), M, D, c.mlp).with_residual(P_(w.x))));
    }
    return VQA_OK;
}

// Last prompt position -> final norm (w.lastn); with a repetition penalty, also the bitmap of every prompt's ids (w.pen_bitmap).
static int qwen_last_position(Forward& f, QwenState& q, const QwenWorkspace& w, const vqa_qwen25vl_prompts& in, const vqa_qwen25vl_packed* pk,
                              float repetition_penalty) {
    const vqa_qwen25vl_config& c = q.cfg;
    const int B = in.batch, S = in.seq_len, D = c.hidden;
    const int *input_ids = in.input_ids, *seq_lens = in.seq_lens;
    auto P_ = [&](size_t off) { return f.at(off); };
    if (pk) TRY(f.launch(CAT_OTHER, 0, "last-row gather", gather_rows_by_index_kernel, B, 128, 0, P_(w.x), pk->pair_row, P_(w.last), D));
    else    TRY(f.launch(CAT_OTHER, 0, "last-row gather", gather_last_rows_kernel, B, 128, 0, P_(w.x), seq_lens, P_(w.last), S, D));
    TRY(f.rmsnorm(P_(w.last), q.final_norm, P_(w.lastn), B, D, c.rms_eps));
    uint32_t* bitmap = f.at<uint32_t>(w.pen_bitmap);
    if (repetition_penalty != 1.0f) {
        // HF applies RepetitionPenaltyLogitsProcessor over the prompt ids before the scores are returned (generation/utils.py:2762-2770,
        // logits_process.py): one bit per (sample, vocabulary id) that occurs in the sample's prompt.
        auto g = f.group(CAT_OTHER);
        TRY(f.memset0(bitmap, (size_t)B * token_bitmap_words(c.vocab) * 4, "penalty bitmap clear"));
        if (pk)
            TRY(qwen_token_bitmap_packed(f, input_ids, pk->cu_seqlens, pk->kv_prefix, pk->pair_seq, pk->max_prompt_len, B, c.vocab, bitmap));
        else
            TRY(qwen_token_bitmap(f, input_ids, seq_lens, B, S, c.vocab, bitmap));
    }
    return VQA_OK;
}

static int qwen_score(vqa_handle* h, QwenState& q, const vqa_qwen25vl_prompts& in, const vqa_qwen25vl_packed* pk, const int* answer_ids,
                      float temperature, float repetition_penalty, float* out_probs, float* out_logprobs, void* workspace, size_t workspace_bytes,
                      cudaStream_t st) {
    const vqa_qwen25vl_config& c = q.cfg;
    const int B = in.batch;
    const QwenWorkspace w = qwen_plan_rows(c, B, pk ? (size_t)pk->total_rows : (size_t)B * in.seq_len, in.n_patches);
    if (workspace_bytes < w.total) return fail(h, VQA_ERR_WORKSPACE, "workspace too small");
    Forward f(h, workspace, st);
    auto F_ = [&](size_t off) { return f.at<float>(off); };
    TRY(qwen_prefill(f, q, w, in, pk));
    TRY(qwen_last_position(f, q, w, in, pk, repetition_penalty));
    // ---------------- lm_head with fused log-softmax gather ----------------
    // T = 1 target per row: score = exp(logprob) = softmax(logits / T)[answer] (qwen2vl_model.py:160-167)
    const Gemm lm = Gemm(f.at(w.lastn), q.lm_head, nullptr, B, c.vocab, c.hidden).processed(temperature, f.at<uint32_t>(w.pen_bitmap),
                                                                                          repetition_penalty);
    return lmhead_score(f, lm, answer_ids, F_(w.lse_max), F_(w.lse_sum), F_(w.label_logit), out_probs, out_logprobs ? out_logprobs : F_(w.logprob),
                        B, 1);
}

// forward_with_trace support: top-k of the last-position distribution of the LAST scoring call (its final hidden states -- and, when a
// repetition penalty is in use, its prompt-token bitmap -- are still in the workspace). Materialises the [B, vocab] bf16 logits of that
// one position -- trace mode only.
static int qwen_topk(vqa_handle* h, QwenState& q, int B, size_t rows, int n_patches, int K, float temperature, float repetition_penalty, int* out_ids,
                     float* out_probs, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    const vqa_qwen25vl_config& c = q.cfg;
    const QwenWorkspace w = qwen_plan_rows(c, B, rows, n_patches);
    if (workspace_bytes < w.total) return fail(h, VQA_ERR_WORKSPACE, "workspace too small");
    Forward f(h, workspace, st);
    bf16* logits = f.at(w.trace_logits);
    TRY(f.gemm(Gemm(f.at(w.lastn), q.lm_head, logits, B, c.vocab, c.hidden), "lm_head"));
    // the bitmap was built by the scoring call with the same penalty
    return qwen_topk_softmax(f, logits, c.vocab, B, c.vocab, temperature, f.at<uint32_t>(w.pen_bitmap), repetition_penalty, K, out_ids, out_probs);
}

// ================================================================================================ greedy generation
// Workspace of a generation: the scoring plan of the padded prefill (its language-model buffers hold B rows during decode steps; the
// [B, vocab] logits of a step go to trace_logits), then the K/V cache (capacity seq_len + max_new_tokens per sequence), the decode
// attention partials, the split-K slices of the decode GEMMs, and the step state.
struct QwenGenWorkspace {
    QwenWorkspace w;
    size_t kcache, vcache, attn_o, attn_ml, splitk, next_ids, pos3, done, n_done, total;
    int cap, splits;
    size_t layer_elems;
};

static QwenGenWorkspace qwen_gen_plan(const vqa_qwen25vl_config& c, int B, int S, int n_patches, int max_new, int num_sms) {
    QwenGenWorkspace g;
    g.w = qwen_plan_rows(c, B, (size_t)B * S, n_patches);
    Plan pl;
    pl.off = g.w.total;
    g.cap = S + max_new;
    g.splits = decode_attn_splits(B, c.kv_heads, g.cap, num_sms);
    g.layer_elems = (size_t)B * c.kv_heads * g.cap * 128;
    g.kcache = pl.take((size_t)c.layers * g.layer_elems * 2);
    g.vcache = pl.take((size_t)c.layers * g.layer_elems * 2);
    g.attn_o = pl.take((size_t)B * c.heads * g.splits * 128 * 4);
    g.attn_ml = pl.take((size_t)B * c.heads * g.splits * 2 * 4);
    const int qkv_cols = (c.heads + 2 * c.kv_heads) * 128;
    g.splitk = pl.take((size_t)8 * B * std::max(qkv_cols, c.hidden) * 4);      // splitk_slices() cuts at most 8 slices
    g.next_ids = pl.take((size_t)B * 4);
    g.pos3 = pl.take((size_t)3 * B * 4);
    g.done = pl.take((size_t)B * 4);
    g.n_done = pl.take(4);
    g.total = pl.off;
    return g;
}

// lm_head on w.lastn into [B, vocab] bf16 logits, then (rollout scoring) the answer log-probabilities of this step, then the greedy token
// (smp NULL) or the sampled one of every unfinished sequence and its bookkeeping
static int qwen_select_token(Forward& f, QwenState& q, const QwenGenWorkspace& g, int B, const vqa_qwen25vl_generation& a,
                             const vqa_qwen25vl_sampling* smp) {
    const vqa_qwen25vl_config& c = q.cfg;
    const QwenWorkspace& w = g.w;
    bf16* logits = f.at(w.trace_logits);
    // The [B, vocab] bf16 logits are 0.3 MB per sequence against the 1.1 GB lm_head weight (7B) that the GEMM streams either way.
    TRY(f.gemm(Gemm(f.at(w.lastn), q.lm_head, logits, B, c.vocab, c.hidden), "lm_head"));
    uint32_t* bitmap = a.repetition_penalty != 1.0f ? f.at<uint32_t>(w.pen_bitmap) : nullptr;
    if (const vqa_qwen25vl_answer_score* s = a.score)
        TRY(answer_logprob(f, logits, B, c.vocab, bitmap, a.repetition_penalty, *s, a.max_new_tokens, a.out_lengths, f.at<int>(g.done)));
    if (smp)
        return sample_select(f, logits, B, c.vocab, bitmap, a.repetition_penalty, *smp, a.eos_ids, a.n_eos, a.max_new_tokens, a.first_position,
                             a.out_tokens, a.out_lengths, f.at<int>(g.done), f.at<int>(g.n_done), a.all_done, f.at<int>(g.next_ids),
                             f.at<int>(g.pos3));
    return greedy_select(f, logits, B, c.vocab, bitmap, a.repetition_penalty, a.eos_ids, a.n_eos, a.max_new_tokens, a.first_position, a.out_tokens,
                         a.out_lengths, f.at<int>(g.done), f.at<int>(g.n_done), a.all_done, f.at<int>(g.next_ids), f.at<int>(g.pos3));
}

// The prefill of vqa_qwen25vl_score over the padded rows, with every layer's K/V stored in the cache, then the first token (greedy when
// smp is NULL, else sampled).
static int qwen_generate_prefill(vqa_handle* h, QwenState& q, const vqa_qwen25vl_prompts& in, const vqa_qwen25vl_generation& a,
                                 const vqa_qwen25vl_sampling* smp, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    const QwenGenWorkspace g = qwen_gen_plan(q.cfg, in.batch, in.seq_len, in.n_patches, a.max_new_tokens, h->num_sms);
    if (workspace_bytes < g.total) return fail(h, VQA_ERR_WORKSPACE, "workspace too small");
    Forward f(h, workspace, st);
    TRY(generate_init(f, in.batch, a.max_new_tokens, a.out_tokens, a.out_lengths, f.at<int>(g.done), f.at<int>(g.n_done), a.all_done));
    const QwenKVCache kv{f.at(g.kcache), f.at(g.vcache), g.layer_elems, g.cap};
    TRY(qwen_prefill(f, q, g.w, in, nullptr, &kv));
    TRY(qwen_last_position(f, q, g.w, in, nullptr, a.repetition_penalty));
    return qwen_select_token(f, q, g, in.batch, a, smp);
}

// One decode step: every sequence feeds its last token (finished ones recompute their frozen last step, which writes nothing new).
// Decode GEMMs have M = B <= 128 rows and stream their weights. At 7B width qkv (N = 4608), o and down (N = 3584) make 36 / 28 / 28
// of the 128-wide N tiles that splitk_slices() counts, far fewer than 132 SMs, so their K range is split (2, 4 and 4 slices:
// tools/bench_generate.py measures the step with and without). gate_up (N = 2 x 18944) and the lm_head (N = 152064) already make
// 296 and 1188 tiles and have no split.
static int qwen_generate_step(vqa_handle* h, QwenState& q, int B, int S, int n_patches, const vqa_qwen25vl_generation& a,
                              const vqa_qwen25vl_sampling* smp, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    const vqa_qwen25vl_config& c = q.cfg;
    const QwenGenWorkspace g = qwen_gen_plan(c, B, S, n_patches, a.max_new_tokens, h->num_sms);
    if (workspace_bytes < g.total) return fail(h, VQA_ERR_WORKSPACE, "workspace too small");
    const QwenWorkspace& w = g.w;
    Forward f(h, workspace, st);
    auto P_ = [&](size_t off) { return f.at(off); };
    auto F_ = [&](size_t off) { return f.at<float>(off); };
    const int D = c.hidden, Hq = c.heads, Hkv = c.kv_heads, qkv_cols = (Hq + 2 * Hkv) * 128;
    float* skw = F_(g.splitk);
    auto skinny = [&](Gemm gm) {
        const int s = splitk_slices(gm.M, gm.N, gm.K, f.nsm);
        return s > 1 ? gm.split_k(s, skw) : gm;
    };
    {
        auto grp = f.group(CAT_OTHER);
        TRY(f.launch(CAT_OTHER, 0, "decode embed", gather_rows_by_index_kernel, B, 128, 0, q.embed, f.at<int>(g.next_ids), P_(w.x), D));
        TRY(qwen_rope_table(f, "decode rope table", f.at<int>(g.pos3), B, q.text_axis, q.text_inv_freq, 64, F_(w.cos), F_(w.sin), 1));
    }
    const float tscale = 1.0f / sqrtf(128.0f);
    for (int l = 0; l < c.layers; ++l) {
        const QwenLlmLayerW& Lw = q.llm[l];
        TRY(f.rmsnorm(P_(w.x), Lw.ln1, P_(w.xn), B, D, c.rms_eps));
        TRY(f.gemm(skinny(Gemm(P_(w.xn), Lw.qkv_w, P_(w.qkv), B, qkv_cols, D).with_bias(Lw.qkv_b)), "decode qkv gemm"));
        TRY(qwen_rope(f, "decode rope", P_(w.qkv), qkv_cols, 0, Hq + Hkv, 128, 128, F_(w.cos), F_(w.sin), B, c.emulate_bf16_rounding));
        bf16 *kc = f.at(g.kcache) + l * g.layer_elems, *vc = f.at(g.vcache) + l * g.layer_elems;
        TRY(kv_cache_write(f, P_(w.qkv), qkv_cols, Hq * 128, (Hq + Hkv) * 128, Hkv, 1, B, a.seq_lens, a.out_lengths, kc, vc, g.cap));
        TRY(decode_attention(f, P_(w.qkv), qkv_cols, kc, vc, g.cap, a.seq_lens, a.out_lengths, B, Hq, Hkv, tscale, g.splits, F_(g.attn_o),
                             F_(g.attn_ml), P_(w.attn), Hq * 128));
        TRY(f.gemm(skinny(Gemm(P_(w.attn), Lw.o_w, P_(w.x), B, D, Hq * 128).with_residual(P_(w.x))), "decode o gemm"));
        TRY(f.rmsnorm(P_(w.x), Lw.ln2, P_(w.xn), B, D, c.rms_eps));
        TRY(f.gemm(Gemm(P_(w.xn), Lw.gu_w, P_(w.ff), B, 2 * c.mlp, D).with_epilogue(EPI_GATED_SILU, c.mlp), "decode gate_up gemm"));
        TRY(f.gemm(skinny(Gemm(P_(w.ff), Lw.down_w, P_(w.x), B, D, c.mlp).with_residual(P_(w.x))), "decode down gemm"));
    }
    TRY(f.rmsnorm(P_(w.x), q.final_norm, P_(w.lastn), B, D, c.rms_eps));
    return qwen_select_token(f, q, g, B, a, smp);
}

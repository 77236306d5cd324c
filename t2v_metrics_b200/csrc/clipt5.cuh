// Host-side orchestration of the CLIP-FlanT5 VQAScore forward: CLIP ViT -> projector -> T5 encoder over the spliced sequence -> T5 decoder
// -> lm_head with the log-softmax gather of the labels. A fixed sequence of kernel launches on the caller's stream.
#pragma once
#include "host.cuh"
#include "attention.cuh"
#include "attention_sm90.cuh"
#include "qwen_kernels.cuh"   // cast_f32_bf16_kernel, gather_rows_by_index_kernel
#include "qwen_decode.cuh"    // generate_init, greedy_select
#include "t5_decode.cuh"

static int clipt5_finalize(vqa_handle* h) {
    const vqa_clipt5_config& c = h->cfg;
    bool ok = true;
    const int P = (c.image_size / c.patch_size) * (c.image_size / c.patch_size);
    const int Dv = c.vit_hidden, Dm = c.d_model, inner = c.n_heads * 64;
    h->patch_w = need(h, "vit.patch_embed.weight", Dv, h->kpad, ok);
    h->cls = need(h, "vit.class_embedding", Dv, 1, ok);
    h->pos = need(h, "vit.position_embedding", P + 1, Dv, ok);
    h->pre_ln_w = need(h, "vit.pre_ln.weight", Dv, 1, ok);
    h->pre_ln_b = need(h, "vit.pre_ln.bias", Dv, 1, ok);
    h->vit.resize(c.vit_layers_run);
    for (int i = 0; i < c.vit_layers_run; ++i) {
        const std::string p = "vit.layers." + std::to_string(i) + ".";
        VitLayerW& L = h->vit[i];
        L.ln1_w = need(h, p + "ln1.weight", Dv, 1, ok); L.ln1_b = need(h, p + "ln1.bias", Dv, 1, ok);
        L.qkv_w = need(h, p + "qkv.weight", 3 * Dv, Dv, ok); L.qkv_b = need(h, p + "qkv.bias", 3 * Dv, 1, ok);
        L.out_w = need(h, p + "out.weight", Dv, Dv, ok); L.out_b = need(h, p + "out.bias", Dv, 1, ok);
        L.ln2_w = need(h, p + "ln2.weight", Dv, 1, ok); L.ln2_b = need(h, p + "ln2.bias", Dv, 1, ok);
        L.fc1_w = need(h, p + "fc1.weight", c.vit_mlp, Dv, ok); L.fc1_b = need(h, p + "fc1.bias", c.vit_mlp, 1, ok);
        L.fc2_w = need(h, p + "fc2.weight", Dv, c.vit_mlp, ok); L.fc2_b = need(h, p + "fc2.bias", Dv, 1, ok);
    }
    h->proj0_w = need(h, "proj.0.weight", Dm, Dv, ok); h->proj0_b = need(h, "proj.0.bias", Dm, 1, ok);
    h->proj2_w = need(h, "proj.2.weight", Dm, Dm, ok); h->proj2_b = need(h, "proj.2.bias", Dm, 1, ok);
    h->shared = need(h, "t5.shared", c.vocab, Dm, ok);
    h->enc_rel = need(h, "t5.enc.rel_bias", c.rel_buckets, c.n_heads, ok);
    h->dec_rel = need(h, "t5.dec.rel_bias", c.rel_buckets, c.n_heads, ok);
    h->enc_final_ln = need(h, "t5.enc.final_ln", Dm, 1, ok);
    h->dec_final_ln = need(h, "t5.dec.final_ln", Dm, 1, ok);
    h->lm_head = need(h, "t5.lm_head", c.vocab, Dm, ok);
    h->enc.resize(c.enc_layers);
    for (int i = 0; i < c.enc_layers; ++i) {
        const std::string p = "t5.enc." + std::to_string(i) + ".";
        T5EncLayerW& L = h->enc[i];
        L.ln0 = need(h, p + "ln0", Dm, 1, ok); L.qkv = need(h, p + "qkv", 3 * inner, Dm, ok);
        L.o = need(h, p + "o", Dm, inner, ok); L.ln1 = need(h, p + "ln1", Dm, 1, ok);
        L.wi = need(h, p + "wi", 2 * c.d_ff, Dm, ok); L.wo = need(h, p + "wo", Dm, c.d_ff, ok);
        if (c.emulate_bf16_rounding & VQA_FLAG_FUSE_NORMS) {
            L.qkv_g = need(h, p + "qkv_g", 3 * inner, Dm, ok);
            L.wi_g = need(h, p + "wi_g", 2 * c.d_ff, Dm, ok);
        }
    }
    h->dec.resize(c.dec_layers);
    for (int i = 0; i < c.dec_layers; ++i) {
        const std::string p = "t5.dec." + std::to_string(i) + ".";
        T5DecLayerW& L = h->dec[i];
        L.ln0 = need(h, p + "ln0", Dm, 1, ok); L.qkv = need(h, p + "qkv", 3 * inner, Dm, ok);
        L.o = need(h, p + "o", Dm, inner, ok); L.ln1 = need(h, p + "ln1", Dm, 1, ok);
        L.cq = need(h, p + "cq", inner, Dm, ok); L.ckv = need(h, p + "ckv", 2 * inner, Dm, ok);
        L.co = need(h, p + "co", Dm, inner, ok); L.ln2 = need(h, p + "ln2", Dm, 1, ok);
        L.wi = need(h, p + "wi", 2 * c.d_ff, Dm, ok); L.wo = need(h, p + "wo", Dm, c.d_ff, ok);
        L.ckT = nullptr;
        if (c.cross_attention_mode == 0) L.ckT = need(h, p + "ckT", Dm, inner, ok);
    }
    return ok ? VQA_OK : VQA_ERR_MISSING_WEIGHT;
}

// ------------------------------------------------------------------------------------------------ workspace plan
struct ClipT5Workspace {
    // vision
    size_t patches, patch_out, hv, vn, vqkv, vattn, vmlp, proj1, proj2;
    // t5
    size_t x, xn, qkv, attn, ff, bias_table, seq_lens, ckv, ssq_a, ssq_b;
    size_t y, yn, dqkv, dattn, dq, dff, splitk, splitk_bytes;
    size_t xt, qt, csc, cctx;   // absorbed cross-attention: Xenc^T, q~ = Wk^T q, scores/probs, context sum p.h
    size_t lse_max, lse_sum, label_logit;
    size_t total;
};
static int ssq_stride(int d_model) { return (d_model / 32 + 3) / 4 * 4; }

// Buffers of the absorbed cross-attention (clipt5_absorbed_cross_attention), taken in this order from `pl`: the transposed encoder output
// xt [B, Dm, Sp], q~ [B * T * H, Dm], the scores / probabilities csc [B * T * H (+ 256 spare rows), Sp] and the context sums ctx [B * T * H, Dm].
struct CrossAttnBuffers { size_t xt, qt, csc, ctx; };
static CrossAttnBuffers take_cross_attn_buffers(Plan& pl, size_t B, size_t T, size_t S, size_t H, size_t Dm) {
    const size_t Sp = (S + 7) / 8 * 8, TH = T * H;
    CrossAttnBuffers b;
    b.xt = pl.take(B * Dm * Sp * 2);
    b.qt = pl.take(B * TH * Dm * 2);
    b.csc = pl.take((B * TH + 256) * Sp * 2);
    b.ctx = pl.take(B * TH * Dm * 2);
    return b;
}
static ClipT5Workspace plan_workspace(const vqa_handle* h, int B, int NI, int L, int T) {
    const vqa_clipt5_config& c = h->cfg;
    const int P = (c.image_size / c.patch_size) * (c.image_size / c.patch_size);
    const size_t Mv = (size_t)NI * (P + 1), Mp = (size_t)NI * P;
    const int S = L - 1 + P;
    const size_t M = (size_t)B * S, Md = (size_t)B * T;
    const size_t inner = (size_t)c.n_heads * 64;
    Plan pl;
    ClipT5Workspace w;
    w.patches = pl.take(Mp * h->kpad * 2);
    w.patch_out = pl.take(Mp * c.vit_hidden * 2);
    w.hv = pl.take(Mv * c.vit_hidden * 4);      // fp32: the vision tower's residual stream (see the vision loop)
    w.vn = pl.take(Mv * c.vit_hidden * 2);
    w.vqkv = pl.take(Mv * 3 * c.vit_hidden * 2);
    w.vattn = pl.take(Mv * c.vit_hidden * 2);
    w.vmlp = pl.take(Mv * c.vit_mlp * 2);
    w.proj1 = pl.take(Mv * c.d_model * 2);
    w.proj2 = pl.take(Mv * c.d_model * 2);
    w.x = pl.take(M * c.d_model * 2);
    w.xn = pl.take(M * c.d_model * 2);
    w.qkv = pl.take(M * 3 * inner * 2);
    w.attn = pl.take(M * inner * 2);
    w.ff = pl.take(M * c.d_ff * 2);
    // fused-norm mode: per-row partial sums of squares of the residual stream, two buffers (the stream is rewritten twice per layer);
    // worst case one partial per 32 output columns
    w.ssq_a = pl.take(M * (size_t)ssq_stride(c.d_model) * 4);
    w.ssq_b = pl.take(M * (size_t)ssq_stride(c.d_model) * 4);
    w.bias_table = pl.take((size_t)c.n_heads * (2 * S - 1) * 4);
    w.seq_lens = pl.take((size_t)B * 4);
    if (c.cross_attention_mode == 0) {
        w.ckv = 0;
        const CrossAttnBuffers xb = take_cross_attn_buffers(pl, B, T, S, c.n_heads, c.d_model);
        w.xt = xb.xt; w.qt = xb.qt; w.csc = xb.csc; w.cctx = xb.ctx;
    } else {
        w.ckv = pl.take(M * 2 * inner * 2);
        w.xt = w.qt = w.csc = w.cctx = 0;
    }
    w.y = pl.take(Md * c.d_model * 2);
    w.yn = pl.take(Md * c.d_model * 2);
    w.dqkv = pl.take(Md * 3 * inner * 2);
    w.dattn = pl.take(Md * inner * 2);
    w.dq = pl.take(Md * inner * 2);
    w.dff = pl.take(Md * c.d_ff * 2);
    {   // fp32 partial tiles of the decoder's split-K GEMMs (largest of the eligible shapes; 0 when none is)
        size_t sk = 0;
        const int shapes[4][2] = {{(int)(3 * inner), c.d_model}, {c.d_model, (int)inner}, {(int)inner, c.d_model}, {c.d_model, c.d_ff}};
        for (const auto& nk : shapes) {
            const int s = splitk_slices((int)Md, nk[0], nk[1], h->num_sms);
            if (s > 1) sk = std::max(sk, (size_t)s * Md * nk[0] * 4);
        }
        w.splitk = pl.take(sk);
        w.splitk_bytes = sk;
    }
    const size_t ntiles = (size_t)LMHEAD_PARTS * ((c.vocab + LMHEAD_BN - 1) / LMHEAD_BN);
    w.lse_max = pl.take(Md * ntiles * 4);
    w.lse_sum = pl.take(Md * ntiles * 4);
    w.label_logit = pl.take(Md * 4);
    w.total = pl.off;
    return w;
}

// Sum of squares of every row of x (bf16 [rows, D]) into slot 0 of its partial-sum row (the other slots are zero): seeds the fused
// RMSNorm chain for the encoder's input embeddings. One warp per row.
__global__ void __launch_bounds__(256) row_ssq_kernel(const bf16* __restrict__ x, float* __restrict__ ssq, int rows, int D, int stride) {
    pdl_launch_dependents();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * D);
    float ss = 0.f;
    for (int i = lane; i < D / 8; i += 32) {
        const uint4 v = xr[i];
        const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = unpack_bf16x2(u[e]);
            ss = fmaf(f.x, f.x, ss);
            ss = fmaf(f.y, f.y, ss);
        }
    }
    ss = warp_sum(ss);
    if (lane == 0) ssq[(size_t)row * stride] = ss;
}

// ------------------------------------------------------------------------------------------------ glue launches
// Every kernel a forward shares with a kernel-level entry point (vqa_b200.cu) is launched by one stage function taking the forward's
// Forward: here for CLIP-FlanT5, in qwen25vl.cuh for the Qwen glue, in qwen_decode.cuh for the decode loops and in host.cuh for the lm_head
// tail. The forwards and the entry points both call these, so the two cannot launch a kernel with different geometry.

// Pixels [n_images, 3, image_size, image_size] (fp32 or bf16) -> patch rows out [n_images * P, kpad] bf16.
static int clipt5_patchify(Forward& f, const void* pixels, int pixel_dtype, bf16* out, int n_images, int image_size, int patch, int kpad) {
    const int rows = n_images * (image_size / patch) * (image_size / patch);
    if (pixel_dtype == VQA_DTYPE_F32)
        return f.launch(CAT_OTHER, 0, "patchify", patchify_kernel<float>, rows, 128, 0, reinterpret_cast<const float*>(pixels), out, n_images,
                        image_size, image_size, patch, kpad);
    return f.launch(CAT_OTHER, 0, "patchify", patchify_kernel<bf16>, rows, 128, 0, reinterpret_cast<const bf16*>(pixels), out, n_images,
                    image_size, image_size, patch, kpad);
}

// Text embeddings and image features -> the encoder input x [B, S = L - 1 + P, D] and seq_lens [B]. Image i's features are rows
// [i * rows_per_image + row_offset, + P) of feats (row stride ldf).
static int clipt5_splice(Forward& f, const int* ids, const int* text_lens, const int* image_index, const bf16* shared, const bf16* feats, int ldf,
                         int row_offset, int rows_per_image, bf16* x, int* seq_lens, int B, int L, int P, int D, int image_token) {
    const int S = L - 1 + P;
    return f.launch(CAT_OTHER, 0, "splice", splice_embed_kernel, B * S, 128, 0, ids, text_lens, image_index, shared, feats, ldf, row_offset,
                    rows_per_image, x, seq_lens, B, L, S, P, D, image_token);
}

// The encoder's relative-position bias table [H, 2S - 1] fp32 from rel_emb [buckets, H] and the bucket LUT [2 * max_distance + 1].
static int clipt5_bias_table(Forward& f, const bf16* rel_emb, const int* lut, int max_distance, float* table, int H, int S) {
    return f.launch(CAT_OTHER, 0, "bias table", bias_table_from_lut_kernel, (H * (2 * S - 1) + 255) / 256, 256, 0, rel_emb, lut, max_distance,
                    table, H, S);
}

// Decoder input embeddings y [B * T, D] of shift_right(labels [B, T]); labels NULL with T = 1: the start token (generation prefill).
static int clipt5_decoder_embed(Forward& f, const int* labels, const bf16* shared, bf16* y, int B, int T, int D, int start_id, int pad_id) {
    return f.launch(CAT_OTHER, 0, "decoder embed", decoder_embed_kernel, B * T, 128, 0, labels, shared, y, T, D, start_id, pad_id);
}

// Sum of squares of the rows of x [rows, D] into slot 0 of ssq [rows, stride].
static int clipt5_row_ssq(Forward& f, const bf16* x, float* ssq, int rows, int D, int stride) {
    return f.launch(CAT_NORM, 0, "row ssq", row_ssq_kernel, (rows + 7) / 8, 256, 0, x, ssq, rows, D, stride);
}

// The CLIP embeddings and pre_layrnorm: patch rows [n_images * P, D] -> fp32 y [n_images * (P + 1), D].
static int clipt5_embed_ln(Forward& f, const bf16* patch, const bf16* cls, const bf16* pos, const bf16* gamma, const bf16* beta, float* y,
                           int n_images, int P, int D, float eps) {
    const int blocks = (n_images * (P + 1) + 7) / 8;
    if (D == 1024)
        return f.launch(CAT_NORM, 0, "clip_embed_ln", clip_embed_ln_kernel<1024>, blocks, 256, 0, patch, cls, pos, gamma, beta, y, n_images, P, eps);
    if (D == 256)
        return f.launch(CAT_NORM, 0, "clip_embed_ln", clip_embed_ln_kernel<256>, blocks, 256, 0, patch, cls, pos, gamma, beta, y, n_images, P, eps);
    return fail(f.h, VQA_ERR_UNSUPPORTED, "vit_hidden must be 1024 or 256");
}

// Head-dim-64 attention of the vision tower and the T5 encoder: packed qkv [B * S, 3 * H * 64] -> out [B * S, H * 64] (launch_attn_tc).
static int clipt5_attention_d64(Forward& f, const char* what, const bf16* qkv, bf16* out, int B, int S, int H, const int* seq_lens,
                                const float* bias_table, float scale, int bias_const_from, bool round_scores) {
    const int inner = H * 64;
    return f.attention(4.0 * B * (double)H * S * S * 64, what, [&] {
        return launch_attn_tc(qkv, 3 * inner, 0, inner, 2 * inner, out, inner, B, S, H, seq_lens, bias_table, scale, bias_const_from, round_scores,
                              f.st);
    });
}

// The scoring path's decoder self-attention over T target rows: packed qkv [B * T, 3 * H * 64] -> out [B * T, H * 64].
static int clipt5_decoder_self_attention(Forward& f, const bf16* qkv, bf16* out, const bf16* rel_emb, const int* lut, int max_distance, int B,
                                         int T, int H, int round_scores) {
    return f.launch(CAT_ATTENTION, 4.0 * B * (double)H * T * T * 64, "decoder self attention", t5_decoder_self_attn_kernel, (B * H * T + 3) / 4,
                    128, 4 * T * sizeof(float), qkv, out, rel_emb, lut, max_distance, B, T, H, round_scores);
}

// One cached decoder self-attention layer of a generation step: the step's K / V rows of qkv [B, 3 * H * 64] appended to kc / vc
// [B, H, cap, 64] (t5_kv_cache_append_kernel), then each row attends to its cache (t5_decode_self_attn_kernel) into out [B, H * 64].
constexpr int T5_DEC_ATTN_WARPS = 4;
static int clipt5_cached_self_attention(Forward& f, const bf16* qkv, bf16* kc, bf16* vc, int cap, const int* lengths, bf16* out,
                                        const bf16* rel_emb, const int* lut, int max_distance, int B, int H, int round_scores) {
    TRY(f.launch(CAT_OTHER, 0, "kv cache append", t5_kv_cache_append_kernel, (B * H * 8 + 255) / 256, 256, 0, qkv, B, H, lengths, kc, vc, cap));
    return f.launch(CAT_ATTENTION, 4.0 * B * (double)H * cap * 64, "decoder self attention (cached)", t5_decode_self_attn_kernel,
                    (B * H + T5_DEC_ATTN_WARPS - 1) / T5_DEC_ATTN_WARPS, 32 * T5_DEC_ATTN_WARPS, T5_DEC_ATTN_WARPS * cap * sizeof(float), qkv,
                    (const bf16*)kc, (const bf16*)vc, cap, lengths, out, rel_emb, lut, max_distance, B, H, round_scores);
}

// ------------------------------------------------------------------------------------------------ forward
// Encoder output x [B * S, Dm] -> xt [B, Dm, Sp] (Sp = S rounded up to 8, columns [S, Sp) zero): the K-major operand of GEMM (3) of the
// absorbed cross-attention.
static int clipt5_transpose_encoder(Forward& f, const bf16* x, bf16* xt, int B, int S, int Dm) {
    const int Sp = (S + 7) / 8 * 8;
    return f.launch(CAT_OTHER, 0, "encoder transpose", transpose_bsd_kernel, dim3((Sp + 31) / 32, (Dm + 31) / 32, B), dim3(32, 8), 0, x, xt, S,
                    Dm, Sp);
}

// The image and prompt inputs of one encoder pass (see vqa_clipt5_score)
struct ClipT5Prompts {
    const void* pixels; int pixel_dtype, n_images;
    const int *image_index, *input_ids, *text_lens;
    int B, L;
};

// Vision tower, projector, multimodal splice, T5 encoder and its final norm into w.xn (prompt lengths in w.seq_lens), and for the absorbed
// cross-attention the transposed encoder output in w.xt: everything a decoder pass reads of the prompts.
static int clipt5_encode(Forward& f, const ClipT5Workspace& w, const ClipT5Prompts& in) {
    vqa_handle* h = f.h;
    const vqa_clipt5_config& c = h->cfg;
    const void* pixels = in.pixels;
    const int pixel_dtype = in.pixel_dtype, n_images = in.n_images, B = in.B, L = in.L;
    const int *image_index = in.image_index, *input_ids = in.input_ids, *text_lens = in.text_lens;
    auto P_ = [&](size_t off) { return f.at(off); };
    const bool round_attn = (c.emulate_bf16_rounding & VQA_FLAG_ROUND_ATTN_SCORES) != 0;
    const bool fuse_norms = (c.emulate_bf16_rounding & VQA_FLAG_FUSE_NORMS) != 0;

    const int grid_w = c.image_size / c.patch_size;
    const int P = grid_w * grid_w;
    const int Dv = c.vit_hidden, Dm = c.d_model, H = c.n_heads, inner = H * 64, Hv = c.vit_heads;
    const int Mp = n_images * P, Mv = n_images * (P + 1);
    const int S = L - 1 + P;
    const int M = B * S;

    // Precision of the vision tower's residual stream: the reference runs CLIPVisionModel under torch.autocast(bf16). nn.LayerNorm is on
    // autocast's fp32 list, so pre_layrnorm hands the encoder an fp32 tensor, every `residual + hidden_states` (modeling_clip.py:371,
    // :376) promotes to fp32, and only the Linear inputs are cast to bf16. hidden_states[-2] is therefore an fp32 tensor, rounded to
    // bf16 once where the projector's first Linear consumes it. The engine keeps the same: hv is fp32, the out_proj / fc2 epilogues add
    // the bf16 Linear output into it unrounded, the LayerNorms read fp32 and write the bf16 GEMM operand.
    float* hv = f.at<float>(w.hv);

    // ---------------- vision tower (CLIP ViT, layers 0 .. vit_layers_run-1; hidden_states[-2]) ----------------
    TRY(clipt5_patchify(f, pixels, pixel_dtype, P_(w.patches), n_images, c.image_size, c.patch_size, h->kpad));
    TRY(f.gemm(Gemm(P_(w.patches), h->patch_w, P_(w.patch_out), Mp, Dv, h->kpad)));
    TRY(clipt5_embed_ln(f, P_(w.patch_out), h->cls, h->pos, h->pre_ln_w, h->pre_ln_b, hv, n_images, P, Dv, c.vit_ln_eps));
    for (int l = 0; l < c.vit_layers_run; ++l) {
        const VitLayerW& Lw = h->vit[l];
        TRY(f.layernorm_f32(hv, Lw.ln1_w, Lw.ln1_b, P_(w.vn), Mv, Dv, c.vit_ln_eps));
        TRY(f.gemm(Gemm(P_(w.vn), Lw.qkv_w, P_(w.vqkv), Mv, 3 * Dv, Dv).with_bias(Lw.qkv_b)));
        TRY(clipt5_attention_d64(f, "vit attention", P_(w.vqkv), P_(w.vattn), n_images, P + 1, Hv, nullptr, nullptr, 0.125f, 0, round_attn));
        TRY(f.gemm(Gemm(P_(w.vattn), Lw.out_w, hv, Mv, Dv, Dv).with_bias(Lw.out_b).accumulate_f32(), "gemm (fp32 residual)"));
        TRY(f.layernorm_f32(hv, Lw.ln2_w, Lw.ln2_b, P_(w.vn), Mv, Dv, c.vit_ln_eps));
        TRY(f.gemm(Gemm(P_(w.vn), Lw.fc1_w, P_(w.vmlp), Mv, c.vit_mlp, Dv).with_bias(Lw.fc1_b).with_epilogue(EPI_QUICK_GELU)));
        TRY(f.gemm(Gemm(P_(w.vmlp), Lw.fc2_w, hv, Mv, Dv, c.vit_mlp).with_bias(Lw.fc2_b).accumulate_f32(), "gemm (fp32 residual)"));
    }
    // hidden_states[-2] -> bf16 (`.to(images.dtype)` / the projector Linear's autocast cast): the single rounding of the tower's output
    const size_t n_hv = (size_t)Mv * Dv;
    TRY(f.launch(CAT_OTHER, 0, "vision output cast", cast_f32_bf16_kernel, (unsigned)((n_hv / 4 + 255) / 256 + 1), 256, 0, hv, P_(w.vn), n_hv));
    // mlp2x_gelu projector (Linear -> GELU(erf) -> Linear), applied to every row; the CLS rows are simply not spliced
    TRY(f.gemm(Gemm(P_(w.vn), h->proj0_w, P_(w.proj1), Mv, Dm, Dv).with_bias(h->proj0_b).with_epilogue(EPI_GELU_ERF)));
    TRY(f.gemm(Gemm(P_(w.proj1), h->proj2_w, P_(w.proj2), Mv, Dm, Dm).with_bias(h->proj2_b)));

    // ---------------- multimodal splice -> T5 encoder input ----------------
    int* seq_lens = f.at<int>(w.seq_lens);
    float* bias_table = f.at<float>(w.bias_table);
    {
        auto g = f.group(CAT_OTHER);
        // feature block of an image = P + 1 rows, first patch row = 1 (drop CLS: mm_vision_select_feature='patch')
        TRY(clipt5_splice(f, input_ids, text_lens, image_index, h->shared, P_(w.proj2), Dm, 1, P + 1, P_(w.x), seq_lens, B, L, P, Dm,
                          c.image_token_id));
        TRY(clipt5_bias_table(f, h->enc_rel, h->lut_bidir, c.rel_max_distance, bias_table, H, S));
    }

    // ---------------- T5 encoder ----------------
    // fuse_norms: the two T5LayerNorms of a layer never run as kernels. The GEMMs that write the residual stream (o, wo) leave per-row
    // partial sums of squares of what they stored; the GEMMs that read it (qkv, wi) take x itself with gamma folded into their weights and
    // scale their accumulator rows by rsqrt(mean(x^2) + eps) in the epilogue (gemm_sm90.cuh, GemmParams::ssq_*).
    NormFuse nf_cons, nf_prod;
    float* ssq_cur = f.at<float>(w.ssq_a);
    float* ssq_nxt = f.at<float>(w.ssq_b);
    if (fuse_norms) {
        const int parts = ssq_parts_for(pick_variant(M, Dm, EPI_STORE), Dm);
        const int stride = (parts + 3) / 4 * 4;
        if (stride > ssq_stride(Dm)) return fail(h, VQA_ERR_UNSUPPORTED, "fused norms: partial-sum stride exceeds the workspace plan");
        nf_cons.stride = nf_prod.stride = stride;
        nf_cons.inv_dim = 1.0f / (float)Dm;
        nf_cons.eps = c.t5_ln_eps;
        auto g = f.group(CAT_NORM);
        TRY(f.memset0(ssq_cur, (size_t)M * stride * 4, "ssq clear"));
        TRY(f.memset0(ssq_nxt, (size_t)M * stride * 4, "ssq clear"));
        TRY(clipt5_row_ssq(f, P_(w.x), ssq_cur, M, Dm, stride));
    }
    for (int l = 0; l < c.enc_layers; ++l) {
        const T5EncLayerW& Lw = h->enc[l];
        if (fuse_norms) {
            nf_cons.ssq_in = ssq_cur;
            TRY(f.gemm(Gemm(P_(w.x), Lw.qkv_g, P_(w.qkv), M, 3 * inner, Dm).with_norm(nf_cons)));
        } else {
            TRY(f.rmsnorm(P_(w.x), Lw.ln0, P_(w.xn), M, Dm, c.t5_ln_eps));
            TRY(f.gemm(Gemm(P_(w.xn), Lw.qkv, P_(w.qkv), M, 3 * inner, Dm)));
        }
        TRY(clipt5_attention_d64(f, "t5 encoder attention", P_(w.qkv), P_(w.attn), B, S, H, seq_lens, bias_table, 1.0f, c.rel_max_distance,
                                 round_attn));
        if (fuse_norms) {
            nf_prod.ssq_out = ssq_nxt;
            TRY(f.gemm(Gemm(P_(w.attn), Lw.o, P_(w.x), M, Dm, inner).with_residual(P_(w.x)).with_norm(nf_prod)));
            std::swap(ssq_cur, ssq_nxt);
            nf_cons.ssq_in = ssq_cur;
            TRY(f.gemm(Gemm(P_(w.x), Lw.wi_g, P_(w.ff), M, 2 * c.d_ff, Dm).with_epilogue(EPI_GATED_GELU, c.d_ff).with_norm(nf_cons)));
            nf_prod.ssq_out = ssq_nxt;
            TRY(f.gemm(Gemm(P_(w.ff), Lw.wo, P_(w.x), M, Dm, c.d_ff).with_residual(P_(w.x)).with_norm(nf_prod)));
            std::swap(ssq_cur, ssq_nxt);
        } else {
            TRY(f.gemm(Gemm(P_(w.attn), Lw.o, P_(w.x), M, Dm, inner).with_residual(P_(w.x))));
            TRY(f.rmsnorm(P_(w.x), Lw.ln1, P_(w.xn), M, Dm, c.t5_ln_eps));
            TRY(f.gemm(Gemm(P_(w.xn), Lw.wi, P_(w.ff), M, 2 * c.d_ff, Dm).with_epilogue(EPI_GATED_GELU, c.d_ff)));
            TRY(f.gemm(Gemm(P_(w.ff), Lw.wo, P_(w.x), M, Dm, c.d_ff).with_residual(P_(w.x))));
        }
    }
    TRY(f.rmsnorm(P_(w.x), h->enc_final_ln, P_(w.xn), M, Dm, c.t5_ln_eps));  // encoder output lives in xn from here on
    if (c.cross_attention_mode == 0) TRY(clipt5_transpose_encoder(f, P_(w.xn), P_(w.xt), B, S, Dm));
    return VQA_OK;
}

// Absorbed cross-attention of the B * T decoder rows q [B * T, H * 64] against the encoder output x [B * S, Dm] (and its transpose xt from
// clipt5_transpose_encoder) into out [B * T, H * 64] (exact in real arithmetic; 30x fewer FLOPs than projecting the S encoder rows because
// only T rows per pair attend):
//   q.(Wk x_s) = (Wk^T q).x_s          sum_s p_s (Wv x_s) = Wv (sum_s p_s x_s)
// The scoring pass, every generation step and vqa_op_t5_cross_attention run this sequence.
struct AbsorbedCrossAttn {
    const bf16 *q, *x, *xt;
    const int* seq_lens;          // [B] encoder rows each pair attends to (<= S)
    const bf16 *wkT, *wv;         // Wk^T [Dm, H * 64]; Wv [H * 64, Dm] (the V half of the layer's k|v weight)
    bf16 *qt, *csc, *ctx, *out;   // CrossAttnBuffers
    int B, T, S, H, Dm;
};
static int clipt5_absorbed_cross_attention(Forward& f, const AbsorbedCrossAttn& a) {
    const int B = a.B, S = a.S, Dm = a.Dm, H = a.H, inner = H * 64, Md = B * a.T, TH = a.T * H, Sp = (S + 7) / 8 * 8;
    // (1) q~[b,t,h,:] = Wk[h]^T q[b,t,h,:]   -- per head: [B*T, 64] x ckT[:, h*64:(h+1)*64]^T -> rows (b*T+t)*H + h
    Gemm g1(a.q, a.wkT, a.qt, Md, Dm, 64);
    g1.lda = inner; g1.ldw = inner; g1.ldc = H * Dm;
    TRY(f.gemm(g1.batched(BatchSpec{H, 0, 64, 0, 64, (long long)Dm, Md, inner, Dm, inner}, Dm >= 256 ? 2561 : 1281), "batched gemm"));
    // (2) scores[b,(t,h),s] = q~[b,(t,h),:] . x[b,s,:]   -- per pair: [T*H, d] x [S, d]^T
    Gemm g2(a.qt, a.x, a.csc, TH, Sp, Dm);
    TRY(f.gemm(g2.batched(BatchSpec{B, TH, 0, S, 0, (long long)TH * Sp, (long long)B * TH, Dm, (long long)B * S, Dm}, 1281), "batched gemm"));
    TRY(f.launch(CAT_ATTENTION, 0, "cross softmax", cross_softmax_kernel, (B * TH + 7) / 8, 256, 0, a.csc, a.seq_lens, TH, B * TH, S, Sp));
    // (3) ctx[b,(t,h),:] = sum_s p[b,(t,h),s] x[b,s,:]   -- per pair: [T*H, Sp] x (x[b]^T)[d, Sp]^T
    Gemm g3(a.csc, a.xt, a.ctx, TH, Dm, Sp);
    TRY(f.gemm(g3.batched(BatchSpec{B, TH, 0, Dm, 0, (long long)TH * Dm, (long long)B * TH, Sp, (long long)B * Dm, Sp}, Dm >= 256 ? 2561 : 1281),
               "batched gemm"));
    // (4) o[b,t,h,:] = Wv[h] ctx[b,t,h,:]   -- per head: [B*T, d] (cols h*d..) x Wv[h*64:(h+1)*64, :]^T -> cols h*64..
    Gemm g4(a.ctx, a.wv, a.out, Md, 64, Dm);
    g4.lda = H * Dm; g4.ldc = inner;
    return f.gemm(g4.batched(BatchSpec{H, 0, Dm, 64, 0, 64, Md, (long long)H * Dm, inner, Dm}, 641), "batched gemm");
}
static int clipt5_absorbed_cross_attention(Forward& f, const ClipT5Workspace& w, const T5DecLayerW& Lw, int B, int T, int S) {
    const vqa_clipt5_config& c = f.h->cfg;
    return clipt5_absorbed_cross_attention(f, AbsorbedCrossAttn{f.at(w.dq), f.at(w.xn), f.at(w.xt), f.at<int>(w.seq_lens), Lw.ckT,
                                                                Lw.ckv + (size_t)c.n_heads * 64 * c.d_model, f.at(w.qt), f.at(w.csc),
                                                                f.at(w.cctx), f.at(w.dattn), B, T, S, c.n_heads, c.d_model});
}

// Reference association (cross_attention_mode 1): K/V projection of all S encoder rows (modeling_t5.py:297-299) into kv [B * S, 2 * H * 64],
// then t5_cross_attn_kernel (T <= 8). round_scores: bf16 scores before the softmax.
static int clipt5_reference_cross_attention(Forward& f, const bf16* q, const bf16* x, const bf16* wkv, bf16* kv, bf16* out, const int* seq_lens,
                                            int B, int T, int S, int H, int Dm, int round_scores) {
    const int inner = H * 64;
    TRY(f.gemm(Gemm(x, wkv, kv, B * S, 2 * inner, Dm)));
    return f.launch(CAT_ATTENTION, 4.0 * B * (double)H * T * S * 64, "cross attention", t5_cross_attn_kernel<8>, B * H, 128, 0, q, (const bf16*)kv,
                    out, seq_lens, 2 * inner, B, T, S, H, round_scores);
}

// Decoder store-GEMMs: M = B*T rows against 4096-row weights -> split-K when that fills the SMs, else the plain path
static Gemm decoder_split_k(const Forward& f, const ClipT5Workspace& w, Gemm g) {
    const int sl = splitk_slices(g.M, g.N, g.K, f.nsm);
    if (sl > 1 && (size_t)sl * g.M * g.N * 4 <= w.splitk_bytes) g.split_k(sl, f.at<float>(w.splitk));
    return g;
}

// Arguments as vqa_clipt5_score, already validated.
static int clipt5_score(vqa_handle* h, const void* pixels, int pixel_dtype, int n_images, const int* image_index, const int* input_ids,
                        const int* text_lens, const int* labels, int B, int L, int T, float* out_scores, float* out_logprobs, void* workspace,
                        size_t workspace_bytes, cudaStream_t st) {
    const vqa_clipt5_config& c = h->cfg;
    const ClipT5Workspace w = plan_workspace(h, B, n_images, L, T);
    if (workspace_bytes < w.total) return fail(h, VQA_ERR_WORKSPACE, "workspace too small");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(h, VQA_ERR_INVALID_ARG, "workspace must be 256-byte aligned");
    Forward f(h, workspace, st);
    auto P_ = [&](size_t off) { return f.at(off); };
    const int rnd = c.emulate_bf16_rounding & VQA_FLAG_ROUND_DECODER;
    const int P = (c.image_size / c.patch_size) * (c.image_size / c.patch_size);
    const int Dm = c.d_model, H = c.n_heads, inner = H * 64;
    const int S = L - 1 + P;
    const int Md = B * T;
    TRY(clipt5_encode(f, w, ClipT5Prompts{pixels, pixel_dtype, n_images, image_index, input_ids, text_lens, B, L}));
    int* seq_lens = f.at<int>(w.seq_lens);

    // ---------------- T5 decoder (T target rows per pair) ----------------
    TRY(clipt5_decoder_embed(f, labels, h->shared, P_(w.y), B, T, Dm, c.decoder_start_id, c.pad_token_id));
    auto dec = [&](Gemm g) { return decoder_split_k(f, w, g); };
    for (int l = 0; l < c.dec_layers; ++l) {
        const T5DecLayerW& Lw = h->dec[l];
        // self-attention
        TRY(f.rmsnorm(P_(w.y), Lw.ln0, P_(w.yn), Md, Dm, c.t5_ln_eps));
        TRY(f.gemm(dec(Gemm(P_(w.yn), Lw.qkv, P_(w.dqkv), Md, 3 * inner, Dm))));
        TRY(clipt5_decoder_self_attention(f, P_(w.dqkv), P_(w.dattn), h->dec_rel, h->lut_unidir, c.rel_max_distance, B, T, H, rnd));
        TRY(f.gemm(dec(Gemm(P_(w.dattn), Lw.o, P_(w.y), Md, Dm, inner).with_residual(P_(w.y)))));
        TRY(f.rmsnorm(P_(w.y), Lw.ln1, P_(w.yn), Md, Dm, c.t5_ln_eps));
        TRY(f.gemm(dec(Gemm(P_(w.yn), Lw.cq, P_(w.dq), Md, inner, Dm))));
        if (c.cross_attention_mode != 0) {
            TRY(clipt5_reference_cross_attention(f, P_(w.dq), P_(w.xn), Lw.ckv, P_(w.ckv), P_(w.dattn), seq_lens, B, T, S, H, Dm, rnd));
        } else {
            TRY(clipt5_absorbed_cross_attention(f, w, Lw, B, T, S));
        }
        TRY(f.gemm(dec(Gemm(P_(w.dattn), Lw.co, P_(w.y), Md, Dm, inner).with_residual(P_(w.y)))));
        // gated FFN
        TRY(f.rmsnorm(P_(w.y), Lw.ln2, P_(w.yn), Md, Dm, c.t5_ln_eps));
        TRY(f.gemm(Gemm(P_(w.yn), Lw.wi, P_(w.dff), Md, 2 * c.d_ff, Dm).with_epilogue(EPI_GATED_GELU, c.d_ff)));
        TRY(f.gemm(dec(Gemm(P_(w.dff), Lw.wo, P_(w.y), Md, Dm, c.d_ff).with_residual(P_(w.y)))));
    }
    TRY(f.rmsnorm(P_(w.y), h->dec_final_ln, P_(w.yn), Md, Dm, c.t5_ln_eps));

    // ---------------- lm_head x hidden, fused log-sum-exp + label gather; logits never reach HBM ----------------
    return lmhead_score(f, Gemm(P_(w.yn), h->lm_head, nullptr, Md, c.vocab, Dm), labels, f.at<float>(w.lse_max), f.at<float>(w.lse_sum),
                        f.at<float>(w.label_logit), out_scores, out_logprobs, B, T);
}

// ================================================================================================ greedy generation
// Workspace of a generation: the scoring plan at T = 1 (its decoder buffers hold the B rows of a step, its split-K slices are sized for
// them, and the encoder output and prompt lengths stay in it for every step), then the self-attention K/V cache (capacity max_new_tokens
// per sequence: the start token and the first max_new_tokens - 1 generated tokens are the inputs), the [B, vocab] bf16 logits of a step,
// and the step state.
struct ClipT5GenWorkspace {
    ClipT5Workspace w;
    size_t kcache, vcache, logits, next_ids, done, n_done, total;
    size_t layer_elems;
    int cap;
};
static ClipT5GenWorkspace clipt5_gen_plan(const vqa_handle* h, int B, int n_images, int L, int max_new) {
    const vqa_clipt5_config& c = h->cfg;
    ClipT5GenWorkspace g;
    g.w = plan_workspace(h, B, n_images, L, 1);
    Plan pl;
    pl.off = g.w.total;
    g.cap = max_new;
    g.layer_elems = (size_t)B * c.n_heads * g.cap * 64;
    g.kcache = pl.take((size_t)c.dec_layers * g.layer_elems * 2);
    g.vcache = pl.take((size_t)c.dec_layers * g.layer_elems * 2);
    g.logits = pl.take((size_t)B * c.vocab * 2);
    g.next_ids = pl.take((size_t)B * 4);
    g.done = pl.take((size_t)B * 4);
    g.n_done = pl.take(4);
    g.total = pl.off;
    return g;
}

// Encoder sharing of a sampled prefill: slots [0, n_prompts) of xn [B, S, Dm], xt [B, Dm, Sp] and seq_lens [B] hold the encoded prompts;
// every slot b >= n_prompts becomes a copy of slot prompt_index[b] (clamped to [0, n_prompts), so no index reaches outside the slots).
// Reads only slots below n_prompts and writes only slots at or above it, so the copies are independent. blockIdx.y = b - n_prompts;
// each slot is xn_vecs + xt_vecs 16-byte vectors, the padding columns of xt included.
__global__ void __launch_bounds__(256) expand_prompts_kernel(const int* __restrict__ prompt_index, int n_prompts, uint4* xn, size_t xn_vecs,
                                                             uint4* xt, size_t xt_vecs, int* seq_lens) {
    pdl_launch_dependents();
    const int b = n_prompts + blockIdx.y;
    const int src = min(max(prompt_index[b], 0), n_prompts - 1);
    if (blockIdx.x == 0 && threadIdx.x == 0) seq_lens[b] = seq_lens[src];
    const size_t n = xn_vecs + xt_vecs, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (i < xn_vecs) {
            xn[b * xn_vecs + i] = xn[src * xn_vecs + i];
        } else {
            const size_t j = i - xn_vecs;
            xt[b * xt_vecs + j] = xt[src * xt_vecs + j];
        }
    }
}

// Expands the n_prompts encoded prompts of xn / xt / seq_lens to B slots (expand_prompts_kernel); none when n_prompts == B. Profiled as
// the bytes it moves: each further slot's xn and xt block read once and written once.
static int clipt5_expand_prompts(Forward& f, const int* prompt_index, int n_prompts, int B, int S, int Dm, bf16* xn, bf16* xt, int* seq_lens) {
    if (n_prompts >= B) return VQA_OK;
    const int Sp = (S + 7) / 8 * 8;
    const size_t xn_vecs = (size_t)S * Dm / 8, xt_vecs = (size_t)Dm * Sp / 8;
    const int slots = B - n_prompts;
    const double bytes = 2.0 * slots * (double)(xn_vecs + xt_vecs) * 16 + 8.0 * slots;
    const unsigned gx = (unsigned)std::min<size_t>((xn_vecs + xt_vecs + 2047) / 2048, 4096);
    return f.op(CAT_OTHER, 0.0, bytes, 1, "encoder expand", [&] {
        expand_prompts_kernel<<<dim3(gx, slots), 256, 0, f.st>>>(prompt_index, n_prompts, reinterpret_cast<uint4*>(xn), xn_vecs,
                                                                  reinterpret_cast<uint4*>(xt), xt_vecs, seq_lens);
        return cudaGetLastError();
    });
}

// Outputs and constants of a generation, the same for the prefill and every step
struct ClipT5GenArgs {
    const int* eos_ids; int n_eos;
    int max_new;
    int* tokens;             // [B, max_new], -1 after a sequence's last token
    int* lengths;            // [B] tokens generated so far
    int* all_done;           // 1 once every sequence has finished
};

// One decoder position per sequence: the start token (first) or the last selected token (next_ids), through every decoder layer with
// its self-attention K/V appended to the cache, then the final norm, the lm_head into [B, vocab] bf16 logits, and the greedy (smp NULL)
// or sampled token of every unfinished sequence. Finished sequences recompute their frozen last position, which changes nothing they output.
static int clipt5_decode_step(Forward& f, const ClipT5GenWorkspace& g, int B, int S, const ClipT5GenArgs& a, const vqa_qwen25vl_sampling* smp,
                              bool first) {
    vqa_handle* h = f.h;
    const vqa_clipt5_config& c = h->cfg;
    const ClipT5Workspace& w = g.w;
    auto P_ = [&](size_t off) { return f.at(off); };
    const int rnd = c.emulate_bf16_rounding & VQA_FLAG_ROUND_DECODER;
    const int Dm = c.d_model, H = c.n_heads, inner = H * 64;
    int* next_ids = f.at<int>(g.next_ids);
    if (first)    // decoder_embed_kernel at T = 1 embeds the start token and reads no labels
        TRY(clipt5_decoder_embed(f, nullptr, h->shared, P_(w.y), B, 1, Dm, c.decoder_start_id, c.pad_token_id));
    else
        TRY(f.launch(CAT_OTHER, 0, "decoder embed", gather_rows_by_index_kernel, B, 128, 0, h->shared, (const int*)next_ids, P_(w.y), Dm));
    auto dec = [&](Gemm gm) { return decoder_split_k(f, w, gm); };
    for (int l = 0; l < c.dec_layers; ++l) {
        const T5DecLayerW& Lw = h->dec[l];
        bf16 *kc = f.at(g.kcache) + l * g.layer_elems, *vc = f.at(g.vcache) + l * g.layer_elems;
        TRY(f.rmsnorm(P_(w.y), Lw.ln0, P_(w.yn), B, Dm, c.t5_ln_eps));
        TRY(f.gemm(dec(Gemm(P_(w.yn), Lw.qkv, P_(w.dqkv), B, 3 * inner, Dm))));
        TRY(clipt5_cached_self_attention(f, P_(w.dqkv), kc, vc, g.cap, a.lengths, P_(w.dattn), h->dec_rel, h->lut_unidir, c.rel_max_distance, B, H,
                                         rnd));
        TRY(f.gemm(dec(Gemm(P_(w.dattn), Lw.o, P_(w.y), B, Dm, inner).with_residual(P_(w.y)))));
        TRY(f.rmsnorm(P_(w.y), Lw.ln1, P_(w.yn), B, Dm, c.t5_ln_eps));
        TRY(f.gemm(dec(Gemm(P_(w.yn), Lw.cq, P_(w.dq), B, inner, Dm))));
        TRY(clipt5_absorbed_cross_attention(f, w, Lw, B, 1, S));
        TRY(f.gemm(dec(Gemm(P_(w.dattn), Lw.co, P_(w.y), B, Dm, inner).with_residual(P_(w.y)))));
        TRY(f.rmsnorm(P_(w.y), Lw.ln2, P_(w.yn), B, Dm, c.t5_ln_eps));
        TRY(f.gemm(Gemm(P_(w.yn), Lw.wi, P_(w.dff), B, 2 * c.d_ff, Dm).with_epilogue(EPI_GATED_GELU, c.d_ff)));
        TRY(f.gemm(dec(Gemm(P_(w.dff), Lw.wo, P_(w.y), B, Dm, c.d_ff).with_residual(P_(w.y)))));
    }
    TRY(f.rmsnorm(P_(w.y), h->dec_final_ln, P_(w.yn), B, Dm, c.t5_ln_eps));
    // The [B, vocab] bf16 logits are 64 KB per sequence against the 263 MB lm_head weight (xxl) that the GEMM streams either way.
    bf16* logits = f.at(g.logits);
    TRY(f.gemm(Gemm(P_(w.yn), h->lm_head, logits, B, c.vocab, Dm), "lm_head"));
    if (smp)    // no repetition penalty and no positions: the arguments greedy selection gets
        return sample_select(f, logits, B, c.vocab, nullptr, 1.0f, *smp, a.eos_ids, a.n_eos, a.max_new, nullptr, a.tokens, a.lengths,
                             f.at<int>(g.done), f.at<int>(g.n_done), a.all_done, next_ids, nullptr);
    return greedy_select(f, logits, B, c.vocab, nullptr, 1.0f, a.eos_ids, a.n_eos, a.max_new, nullptr, a.tokens, a.lengths, f.at<int>(g.done),
                         f.at<int>(g.n_done), a.all_done, next_ids, nullptr);
}

// Encoder pass of vqa_clipt5_score over the in.B prompts, copied to the `batch` sequence slots by prompt_index when in.B < batch
// (clipt5_expand_prompts), the generation state reset, then the first decoder position (the start token) and the first token.
static int clipt5_generate_prefill(vqa_handle* h, const ClipT5Prompts& in, int batch, const int* prompt_index, const ClipT5GenArgs& a,
                                   const vqa_qwen25vl_sampling* smp, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    const ClipT5GenWorkspace g = clipt5_gen_plan(h, batch, in.n_images, in.L, a.max_new);
    if (workspace_bytes < g.total) return fail(h, VQA_ERR_WORKSPACE, "workspace too small");
    Forward f(h, workspace, st);
    const int P = (h->cfg.image_size / h->cfg.patch_size) * (h->cfg.image_size / h->cfg.patch_size);
    const int S = in.L - 1 + P;
    TRY(clipt5_encode(f, g.w, in));
    TRY(clipt5_expand_prompts(f, prompt_index, in.B, batch, S, h->cfg.d_model, f.at(g.w.xn), f.at(g.w.xt), f.at<int>(g.w.seq_lens)));
    TRY(generate_init(f, batch, a.max_new, a.tokens, a.lengths, f.at<int>(g.done), f.at<int>(g.n_done), a.all_done));
    return clipt5_decode_step(f, g, batch, S, a, smp, true);
}

// One decode step: every sequence feeds its last selected token.
static int clipt5_generate_step(vqa_handle* h, int B, int n_images, int L, const ClipT5GenArgs& a, const vqa_qwen25vl_sampling* smp,
                                void* workspace, size_t workspace_bytes, cudaStream_t st) {
    const ClipT5GenWorkspace g = clipt5_gen_plan(h, B, n_images, L, a.max_new);
    if (workspace_bytes < g.total) return fail(h, VQA_ERR_WORKSPACE, "workspace too small");
    Forward f(h, workspace, st);
    const int P = (h->cfg.image_size / h->cfg.patch_size) * (h->cfg.image_size / h->cfg.patch_size);
    return clipt5_decode_step(f, g, B, L - 1 + P, a, smp, false);
}

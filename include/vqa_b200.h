/*
 * vqa_b200.h -- C ABI of libvqa_b200.so, the H100-native (sm_90a) VQAScore engine.
 *
 * This is the drop-in boundary for the scoring hot path of linzhiqiu/t2v_metrics: one call computes, for a batch of
 * (image, question) pairs, the score the reference's VQAScoreModel.forward() returns
 * (t2v_metrics/models/vqascore_models/vqa_model.py:10-18, called from t2v_metrics/score.py:104-106).
 * For CLIP-FlanT5 that is exp(-mean CE(logits, labels)) of T5ForConditionalGeneration on the spliced
 * [text | 576 CLIP patch features | text] sequence (v3.0 clip_t5_model.py; arithmetic in
 * transformers/models/t5/modeling_t5.py:992-1133 and transformers/models/clip/modeling_clip.py:647-696).
 *
 * Conventions
 *   - plain C types only; every pointer documented as HOST or DEVICE memory;
 *   - the caller owns all buffers (weights, inputs, outputs, workspace); the library never frees caller memory and
 *     keeps only borrowed device pointers to the bound weights;
 *   - all work is enqueued on the given CUDA stream (passed as void* = cudaStream_t); no internal device sync;
 *   - every function returns 0 on success or a negative vqa_status; vqa_last_error() gives the message;
 *   - a handle belongs to one device and one in-flight call; distinct handles are independent.
 */
#ifndef VQA_B200_H
#define VQA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VQA_B200_ABI_VERSION 3

typedef enum {
    VQA_OK = 0,
    VQA_ERR_INVALID_ARG = -1,
    VQA_ERR_MISSING_WEIGHT = -2,
    VQA_ERR_CUDA = -3,
    VQA_ERR_WORKSPACE = -4,
    VQA_ERR_UNSUPPORTED = -5
} vqa_status;

typedef enum { VQA_DTYPE_BF16 = 0, VQA_DTYPE_F32 = 1, VQA_DTYPE_I32 = 2 } vqa_dtype;

/* CLIP-FlanT5 architecture description (replaces the HF config objects the reference loads in
 * t2v_metrics/models/vqascore_models/mm_utils.py:182-241). */
typedef struct {
    /* CLIP ViT vision tower (transformers/models/clip/modeling_clip.py) */
    int32_t image_size;       /* 336 */
    int32_t patch_size;       /* 14 */
    int32_t vit_hidden;       /* 1024 */
    int32_t vit_heads;        /* 16 (head_dim must be 64) */
    int32_t vit_mlp;          /* 4096 */
    int32_t vit_layers_run;   /* encoder layers executed = select_layer -2 -> num_hidden_layers - 1 = 23 */
    float   vit_ln_eps;       /* 1e-5 */
    /* T5 encoder-decoder (transformers/models/t5/modeling_t5.py) */
    int32_t d_model;          /* 4096 (xxl) / 2048 (xl) */
    int32_t n_heads;          /* 64 / 32 (d_kv must be 64) */
    int32_t d_ff;             /* 10240 / 5120 */
    int32_t enc_layers;       /* 24 */
    int32_t dec_layers;       /* 24 */
    int32_t vocab;            /* 32128 */
    int32_t rel_buckets;      /* 32 */
    int32_t rel_max_distance; /* 128 */
    float   t5_ln_eps;        /* 1e-6 */
    int32_t image_token_id;   /* -200, t2v_metrics/constants.py:7 */
    int32_t pad_token_id;     /* 0 */
    int32_t decoder_start_id; /* 0 */
    int32_t emulate_bf16_rounding; /* bit flags. 1: the small decoder kernels round scores / bias adds to bf16 where the reference's eager path
                                      does. 2: the wgmma attention forms the reference's bf16 score tensors before the softmax (off: fp32
                                      scores). 4: fuse the encoder's T5LayerNorms into the GEMMs around them -- needs t5.enc.{i}.qkv_g / wi_g
                                      (= qkv . diag(ln0), wi . diag(ln1)); the o / wo epilogues emit row sums of squares, the qkv / wi
                                      epilogues apply rsqrt(mean(x^2) + eps) to their accumulator rows */
    int32_t cross_attention_mode;  /* 0: absorbed (q.(Wk x) = (Wk^T q).x, needs t5.dec.{i}.ckT); 1: project K/V of all
                                      encoder rows in every decoder layer, as modeling_t5.py:297-299 does */
} vqa_clipt5_config;

/* A named device tensor handed to vqa_bind_weights (borrowed pointer, bf16, row-major contiguous). */
typedef struct {
    const char* name;  /* HOST string, canonical engine name (see INTEGRATION.md for the HF -> engine mapping) */
    const void* data;  /* DEVICE pointer */
    int64_t shape[4];
    int32_t ndim;
    int32_t dtype;     /* vqa_dtype; weights must be VQA_DTYPE_BF16 */
} vqa_tensor;

/* Qwen2.5-VL architecture description (vision tower + language model; transformers/models/qwen2_5_vl/
 * configuration_qwen2_5_vl.py:51-64,106-125; 7B values in comments). The vision tower's 80-wide heads are laid out
 * zero-padded to 128 columns per head in the fused qkv / proj weights, and its MLP width is padded to a multiple of 128
 * (both done by the host when it fuses the checkpoint tensors, engine.convert_qwen_state_dict). */
typedef struct {
    int32_t vit_depth;        /* 32 */
    int32_t vit_hidden;       /* 1280 */
    int32_t vit_heads;        /* 16 */
    int32_t vit_head_dim;     /* 80 (real head width; stored padded to 128) */
    int32_t vit_mlp;          /* 3420 (stored padded to 3456) */
    int32_t patch_dim;        /* 3 * temporal_patch(2) * 14 * 14 = 1176 */
    int32_t spatial_merge;    /* 2 */
    int32_t out_hidden;       /* 3584 */
    uint64_t fullatt_mask;    /* bit l set: vision block l attends over whole frames (7,15,23,31), else 112-px windows */
    int32_t hidden;           /* 3584 */
    int32_t layers;           /* 28 */
    int32_t heads;            /* 28 (head_dim must be 128) */
    int32_t kv_heads;         /* 4 */
    int32_t mlp;              /* 18944 */
    int32_t vocab;            /* 152064 */
    float   rms_eps;          /* 1e-6 */
    int32_t emulate_bf16_rounding;
} vqa_qwen25vl_config;

typedef struct vqa_handle vqa_handle;

/* ABI / build info ("vqa_b200 abi=3 arch=sm_90a ..."). Never fails. */
const char* vqa_version(void);

/* Create an engine for a CLIP-FlanT5 model on CUDA device `device`. */
int vqa_create_clipt5(const vqa_clipt5_config* cfg, int device, vqa_handle** out);

/* Borrow device pointers of the model weights. May be called several times; names are matched exactly.
 * Replaces model_cls.from_pretrained(...).to(device, bf16) (mm_utils.py:201,228) -- loading stays in the host. */
int vqa_bind_weights(vqa_handle* h, const vqa_tensor* tensors, int32_t n);

/* Check that every weight the forward needs is bound with the right shape. */
int vqa_finalize_weights(vqa_handle* h);

/* Bytes of device workspace vqa_clipt5_score needs for up to `batch` pairs, `n_images` distinct images,
 * text length `text_len` (ids per row incl. the image slot) and `label_len` target tokens. */
size_t vqa_clipt5_workspace_bytes(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len,
                                  int32_t label_len);

/* Score `batch` (image, question) pairs.
 *   pixels      DEVICE [n_images, 3, image_size, image_size], dtype pixel_dtype (F32 or BF16): CLIPImageProcessor output
 *   image_index DEVICE int32 [batch] -> which image each pair uses, or NULL for identity (n_images == batch)
 *   input_ids   DEVICE int32 [batch, text_len], image slot = cfg.image_token_id, right-padded with pad_token_id
 *   text_lens   DEVICE int32 [batch] valid ids per row
 *   labels      DEVICE int32 [batch, label_len] < vocab, -100 = ignored (padding). Every negative label is ignored like -100: it adds
 *               nothing to the mean and the decoder input after it is pad_token_id
 *   out_scores  DEVICE float [batch] : exp(-mean CE)  (v3.0 CLIPT5Model.forward); NaN for a pair whose labels are all ignored, as the
 *               reference's CrossEntropyLoss(reduction='mean') gives over zero targets
 *   out_logprobs DEVICE float [batch, label_len] per-token log-probabilities (ignored positions are not written), or NULL
 *   workspace   DEVICE, >= vqa_clipt5_workspace_bytes(...)
 *   stream      cudaStream_t
 */
int vqa_clipt5_score(vqa_handle* h, const void* pixels, int32_t pixel_dtype, int32_t n_images,
                     const int32_t* image_index, const int32_t* input_ids, const int32_t* text_lens,
                     const int32_t* labels, int32_t batch, int32_t text_len, int32_t label_len, float* out_scores,
                     float* out_logprobs, void* workspace, size_t workspace_bytes, void* stream);

/* ---- CLIP-FlanT5 greedy generation (HF T5ForConditionalGeneration.generate(inputs_embeds=<spliced prompt>, do_sample=False, num_beams=1))
 * One prefill, then one decode step per further token, all on the caller's stream. The prefill runs the encoder pass of vqa_clipt5_score
 * (same inputs, no labels) and keeps its output in the workspace, then feeds the decoder start token and selects the first token. A step
 * feeds each prompt's last token through the decoder, appending every layer's self-attention K/V row to a cache inside the workspace
 * (capacity max_new_tokens per prompt), and selects the next one. Selection: arg-max of the bf16 lm_head logits cast to fp32, ties to the
 * lowest id; no logits processors. A prompt finishes after emitting one of eos_ids (which is kept in its output) or max_new_tokens tokens;
 * later steps leave it unchanged. Needs cross_attention_mode 0.
 *   eos_ids [n_eos]         DEVICE; n_eos may be 0
 *   out_tokens [batch, max_new_tokens]  generated ids, -1 after a prompt's last one; out_lengths [batch] tokens generated so far;
 *   all_done [1]            1 once every prompt has finished
 * Every step-dependent value lives in device memory: the step takes the same arguments every time, so one CUDA graph of it can be
 * replayed for every token. The prefill and the steps must use the same workspace, sizes and pointers. batch <= 128,
 * max_new_tokens <= 2048. */
size_t vqa_clipt5_generate_workspace_bytes(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, int32_t max_new_tokens);
int vqa_clipt5_generate_prefill(vqa_handle* h, const void* pixels, int32_t pixel_dtype, int32_t n_images, const int32_t* image_index,
                                const int32_t* input_ids, const int32_t* text_lens, int32_t batch, int32_t text_len, const int32_t* eos_ids,
                                int32_t n_eos, int32_t max_new_tokens, int32_t* out_tokens, int32_t* out_lengths, int32_t* all_done,
                                void* workspace, size_t workspace_bytes, void* stream);
int vqa_clipt5_generate_step(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, const int32_t* eos_ids, int32_t n_eos,
                             int32_t max_new_tokens, int32_t* out_tokens, int32_t* out_lengths, int32_t* all_done, void* workspace,
                             size_t workspace_bytes, void* stream);

/* ---- Qwen2.5-VL (replaces Qwen2VLModel.forward's per-sample generate(max_new_tokens=1, output_scores=True) +
 * softmax(scores / T)[answer_id], t2v_metrics/models/vqascore_models/qwen2vl_model.py:160-167,190-289) ---- */
int vqa_create_qwen25vl(const vqa_qwen25vl_config* cfg, int device, vqa_handle** out);

/* Rotary metadata (HOST arrays, copied): for frequency index i < n_half the rotation angle of a token is
 * position[axis[i]] * inv_freq[i]. Text: n_half = 64, axis = mrope sections (t,h,w) (modeling_qwen2_5_vl.py:650-662),
 * inv_freq = rope_theta^(-2i/128). Vision: n_half = head_dim/2 = 40, axis = [h]*20 + [w]*20, inv_freq = 10000^(-2i/40). */
int vqa_qwen25vl_set_rope(vqa_handle* h, const float* text_inv_freq, const int32_t* text_axis, int32_t text_half,
                          const float* vis_inv_freq, const int32_t* vis_axis, int32_t vis_half);

/* The inputs of one prefill: `batch` prompts and the images / videos they show. All index arrays are DEVICE int32 and are produced by
 * the host's mirror of the reference's index logic (rot_pos_emb :382-409, get_window_index :411-451, get_rope_index :1024-1133).
 * Packed rows (a vqa_qwen25vl_packed is given) ignore seq_lens and seq_len: input_ids / feat_index [total_rows] and position_ids
 * [3, total_rows] are then in packed row order.
 * The library reads this struct, and every struct below, only during the call it is passed to and keeps no pointer to it; a CUDA graph
 * captured from a call keeps the values the struct held at capture. */
typedef struct {
    const void* pixel_patches;     /* [n_patches, patch_dim], all images concatenated, processor (merge-block) order */
    int32_t pixel_dtype;           /* F32 or BF16 */
    int32_t n_patches;
    const int32_t* vis_pos_hw;     /* [2, n_patches]  (h, w) index of every patch, already in WINDOW order */
    const int32_t* window_index;   /* [n_patches / merge^2]  window order of the 2x2 patch groups */
    const int32_t* reverse_index;  /* argsort(window_index) */
    const int32_t* cu_window;      /* [n_windows + 1]  cumulative patch counts (window order) */
    int32_t n_windows;
    int32_t max_window_len;
    const int32_t* cu_frames;      /* [n_frames + 1]  cumulative patch counts (window order) */
    int32_t n_frames;
    int32_t max_frame_len;
    const int32_t* input_ids;      /* [batch, seq_len] right-padded */
    const int32_t* seq_lens;       /* [batch] */
    const int32_t* feat_index;     /* [batch, seq_len] row of the merged vision features for image-token positions, -1 elsewhere */
    const int32_t* position_ids;   /* [3, batch*seq_len] (t, h, w) mRoPE positions */
    int32_t batch;
    int32_t seq_len;
} vqa_qwen25vl_prompts;

/* KV-prefix sharing (SURVEY 8(f)1; reference score.py:104-106 repeats one image across N texts and qwen2vl_model.py:190 re-runs the whole
 * prompt per text). The language-model tokens are given as PACKED rows: sequences stored back to back (cu_seqlens [n_seq + 1]); the
 * [chat prefix + vision tokens] of an image is ONE sequence (kv_prefix = -1), each prompt's remaining tokens are a sequence of their own whose
 * kv_prefix names the shared one: its rows attend to all prefix rows, then causally to themselves. Causality makes this exact (a prefix
 * row never sees a suffix), and the prefix rows go through every layer once per image instead of once per prompt. */
typedef struct {
    int32_t total_rows;
    const int32_t* cu_seqlens;     /* [n_seq + 1] */
    const int32_t* kv_prefix;      /* [n_seq], -1 = none */
    int32_t n_seq;
    int32_t max_seq_len;           /* longest sequence */
    const int32_t* pair_row;       /* [batch] packed row of each prompt's last token */
    const int32_t* pair_seq;       /* [batch] the sequence holding it */
    int32_t max_prompt_len;        /* longest prefix + suffix (repetition-penalty bitmap) */
} vqa_qwen25vl_packed;

/* Bytes of device workspace of one scoring call: n_prompts prompts in `rows` language-model rows (padded rows: batch * seq_len; packed
 * rows: total_rows). */
size_t vqa_qwen25vl_workspace_bytes(vqa_handle* h, int32_t n_prompts, int64_t rows, int32_t n_patches);

/* Score prompts->batch prompts in one prefill, over padded rows (packed == NULL) or packed rows.
 *   answer_ids     DEVICE [batch] the answer's first token id
 *   repetition_penalty  1.0 = off; otherwise HF's RepetitionPenaltyLogitsProcessor over each sample's prompt ids is applied to the
 *                  fp32 logits before the temperature (generation/utils.py:2762-2770; the checkpoint's generation_config.json
 *                  decides it in the reference, SURVEY F8)
 *   out_probs      DEVICE [batch] softmax(processed last-position logits / temperature)[answer_id]; out_logprobs optional
 */
int vqa_qwen25vl_score(vqa_handle* h, const vqa_qwen25vl_prompts* prompts, const vqa_qwen25vl_packed* packed, const int32_t* answer_ids,
                       float temperature, float repetition_penalty, float* out_probs, float* out_logprobs, void* workspace,
                       size_t workspace_bytes, void* stream);

/* Trace output (reference forward_with_trace, qwen2vl_model.py:303-493, top-5 at :439-447): the k <= 8 most probable next tokens of every
 * prompt of the LAST scoring call on this handle (vqa_qwen25vl_score: total_rows = batch * seq_len over padded rows, packed->total_rows
 * over packed rows) with the same n_patches and the same workspace -- its final hidden states and, when repetition_penalty != 1, its prompt-token
 * bitmap are still there -- under the same processing as the score: bf16 logits -> fp32 -> repetition penalty -> 1/T -> softmax over the
 * whole vocabulary. out_ids / out_probs: DEVICE [batch, k], most probable first; out_ids[b][0] is the token generate(max_new_tokens=1,
 * do_sample=False) would emit. This call materialises [batch, vocab] bf16 logits of that one position in the workspace -- a debugging
 * aid; the scoring path never stores logits. */
int vqa_qwen25vl_topk(vqa_handle* h, int32_t batch, int64_t total_rows, int32_t n_patches, int32_t k, float temperature,
                      float repetition_penalty, int32_t* out_ids, float* out_probs, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Qwen2.5-VL greedy generation (reference Qwen2VLModel.generate, qwen2vl_model.py:495-563: generate(do_sample=False)) ----
 * One prefill, then one decode step per further token, all on the caller's stream. The prefill runs the vision tower and the padded-row
 * prefill of vqa_qwen25vl_score (same index arrays, no answer ids), stores every layer's post-rope K/V rows in a cache inside the workspace
 * (capacity seq_len + max_new_tokens per prompt), and selects the first token. A step feeds each prompt's last token through the
 * language model and selects the next one. Selection: bf16 lm_head logits -> fp32 -> HF's RepetitionPenaltyLogitsProcessor over the
 * prompt ids and the tokens generated so far (repetition_penalty 1.0 = off) -> arg-max, ties to the lowest id. A prompt finishes after
 * emitting one of eos_ids (which is kept in its output) or max_new_tokens tokens; later steps leave it unchanged.
 * Every step-dependent value lives in device memory: the step takes the same arguments every time, so one CUDA graph of it can be
 * replayed for every token. The prefill and the steps must use the same workspace, sizes and pointers. batch <= 128. */

/* ---- Qwen2.5-VL scoring over a greedy rollout (reference Qwen2VLModel.forward / forward_with_trace with max_new_tokens > 1,
 * qwen2vl_model.py:169-493: generate(do_sample=False, output_scores=True), then softmax(scores[s] / T)[answer id] at chosen steps) ----
 * A generation with an answer score launches one more kernel per token, between the lm_head and the selection: for every step s of every
 * unfinished prompt b, the log-softmax of the step's processed scores (bf16 logits -> fp32 -> repetition penalty over the prompt and the
 * tokens generated before s -> / temperature), over the whole vocabulary, at each of the prompt's answer ids. The temperature only
 * affects these probabilities; the tokens are those of the plain generation, bit for bit. Same workspace
 * (vqa_qwen25vl_generate_workspace_bytes) and the same rules for it. The outputs are caller-owned. */
typedef struct {
    const int32_t* answer_ids;     /* DEVICE [batch, n_max], prompt b's ids in its first answer_counts[b] entries (no cap on n_max) */
    const int32_t* answer_counts;  /* DEVICE [batch] */
    int32_t n_max;
    float temperature;
    int32_t top_k;                 /* 0 <= top_k <= 8 */
    float* out_logp;               /* [batch, max_new_tokens, n_max] fp32, [b, s, j] = log p(s, answer_ids[b, j]); entries of steps a
                                      prompt did not generate and of j >= answer_counts[b] are not written */
    int32_t* out_topk_ids;         /* [batch, max_new_tokens, top_k]: the step's top_k ids (ties to the lower id) and probabilities; */
    float* out_topk_probs;         /* may be NULL when top_k == 0 */
} vqa_qwen25vl_answer_score;

/* The outputs and constants of a generation, the same for the prefill and every step. All pointers DEVICE. */
typedef struct {
    const int32_t* seq_lens;       /* [batch] prompt lengths: the prefill's prompts->seq_lens, the same pointer */
    const int32_t* first_position; /* [batch] mRoPE position of the first generated token: the last prompt token's position + 1; token t
                                      sits at that + t on all three axes (what transformers' generate() feeds) */
    const int32_t* eos_ids;        /* [n_eos]; n_eos may be 0 */
    int32_t n_eos;
    int32_t max_new_tokens;
    float repetition_penalty;
    int32_t* out_tokens;           /* [batch, max_new_tokens] generated ids, -1 after a prompt's last one */
    int32_t* out_lengths;          /* [batch] tokens generated so far */
    int32_t* all_done;             /* [1] 1 once every prompt has finished */
    const vqa_qwen25vl_answer_score* score;   /* HOST; NULL = plain greedy generation, else a scored rollout */
} vqa_qwen25vl_generation;

size_t vqa_qwen25vl_generate_workspace_bytes(vqa_handle* h, int32_t batch, int32_t seq_len, int32_t n_patches, int32_t max_new_tokens);
int vqa_qwen25vl_generate_prefill(vqa_handle* h, const vqa_qwen25vl_prompts* prompts, const vqa_qwen25vl_generation* gen, void* workspace,
                                  size_t workspace_bytes, void* stream);
int vqa_qwen25vl_generate_step(vqa_handle* h, const vqa_qwen25vl_generation* gen, int32_t batch, int32_t seq_len, int32_t n_patches,
                               void* workspace, size_t workspace_bytes, void* stream);

/* ---- Qwen2.5-VL sampled generation (reference Qwen2VLModel.generate with do_sample and temperature > 0, qwen2vl_model.py:495-563:
 * generate(do_sample=True, temperature=T, top_p=p) with the checkpoint's top_k, default 50) ----
 * The same prefill and steps as the greedy generation, with the selection replaced: HF's sampling distribution, built as its processors
 * build it -- repetition penalty (as above), then scores / temperature (an fp32 division; none at 1.0), then top-k (every id whose score
 * is >= the k-th largest stays, ties included), then top-p (in ascending order of (score, id), the ids whose cumulative probability is
 * <= fp32(1 - top_p) go, the most probable always stays; lower ids of the group of equal scores at the cut go first) -- and one draw from
 * the softmax of the kept scores: Gumbel-max with the uniforms of Philox4x32-10 keyed by seeds[b] at counter (id / 4, t, 0, 0), lane
 * id % 4, where t is the index of the token. A prompt's tokens depend on its seed, prompt and sizes only, not on its batch position or
 * on whether the step is replayed from a CUDA graph. A score that overflows fp32 (or a NaN logit) saturates to +-FLT_MAX (NaN to
 * -FLT_MAX), where HF's softmax would be NaN; a top_p whose fp32(1 - top_p) rounds to 1 keeps only the most probable id, as HF does.
 * 1 - top_p is taken in double and rounded to fp32 once, as HF's TopPLogitsWarper compares its fp32 cumulative probabilities with
 * 1 - top_p of the caller's Python float (a float top_p, rounded before the subtraction, would move the threshold by up to 10 fp32 ulps).
 * Same workspace (vqa_qwen25vl_generate_workspace_bytes) and the same rules for it; gen->score must be NULL (a scored rollout is greedy). Refused with VQA_ERR_INVALID_ARG: a NULL seeds pointer, a temperature that is
 * not positive and finite, top_k < 0, top_p outside (0, 1]. */
typedef struct {
    const uint64_t* seeds;  /* DEVICE [batch]: prompt b's key; its draws depend on (seeds[b], step, id) only */
    float temperature;      /* > 0 and finite; 1.0 = no division */
    int32_t top_k;          /* >= 0; 0 = off */
    double top_p;           /* (0, 1]; 1.0 = off. A double, as the caller's Python float: the threshold is fp32(1 - top_p) of it, as HF's */
} vqa_qwen25vl_sampling;

int vqa_qwen25vl_generate_prefill_sampled(vqa_handle* h, const vqa_qwen25vl_prompts* prompts, const vqa_qwen25vl_generation* gen,
                                          const vqa_qwen25vl_sampling* sampling, void* workspace, size_t workspace_bytes, void* stream);
int vqa_qwen25vl_generate_step_sampled(vqa_handle* h, const vqa_qwen25vl_generation* gen, const vqa_qwen25vl_sampling* sampling, int32_t batch,
                                       int32_t seq_len, int32_t n_patches, void* workspace, size_t workspace_bytes, void* stream);

/* ---- CLIP-FlanT5 sampled generation (HF T5ForConditionalGeneration.generate(inputs_embeds=<spliced prompt>, do_sample=True,
 * temperature=T, top_k=k, top_p=p)) ----
 * The greedy generation's prefill and steps (vqa_clipt5_generate_*) with the selection replaced by the draw the Qwen2.5-VL sampled
 * generation makes: vqa_qwen25vl_sampling is shared by both models, with the same warpers (no repetition penalty here: FlanT5's generation
 * config has none), the same tie rules, saturation and Philox4x32-10 uniforms. Sequence b's draws depend on (seeds[b], step, id) only:
 * not on its slot, on the other sequences, or on whether the step is replayed from a CUDA graph.
 * Encoder sharing: the prefill encodes n_prompts <= batch prompts (input_ids [n_prompts, text_len], text_lens / image_index [n_prompts])
 * into sequence slots 0 .. n_prompts - 1, then copies prompt prompt_index[b] into every slot b >= n_prompts (the encoder output, its
 * transposed copy and the prompt length; one launch, none when n_prompts == batch), so n draws of one (image, prompt) pair run the
 * vision tower and the encoder once. prompt_index: DEVICE [batch], entries b < n_prompts unused, entries b >= n_prompts in
 * [0, n_prompts) (others are clamped into that range); NULL when n_prompts == batch. The steps do not depend on n_prompts.
 * Same workspace (vqa_clipt5_generate_workspace_bytes(batch, ...)) and the same rules for it. Refused with VQA_ERR_INVALID_ARG before any
 * launch: a NULL seeds pointer, a temperature that is not positive and finite, top_k < 0, top_p outside (0, 1], n_prompts outside
 * [1, batch], n_prompts < batch with a NULL prompt_index; cross_attention_mode 1 is refused as the greedy generation refuses it. */
int vqa_clipt5_generate_prefill_sampled(vqa_handle* h, const void* pixels, int32_t pixel_dtype, int32_t n_images, const int32_t* image_index,
                                        const int32_t* input_ids, const int32_t* text_lens, int32_t batch, int32_t text_len,
                                        const int32_t* eos_ids, int32_t n_eos, int32_t max_new_tokens, int32_t* out_tokens,
                                        int32_t* out_lengths, int32_t* all_done, int32_t n_prompts, const int32_t* prompt_index,
                                        const vqa_qwen25vl_sampling* sampling, void* workspace, size_t workspace_bytes, void* stream);
int vqa_clipt5_generate_step_sampled(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, const int32_t* eos_ids, int32_t n_eos,
                                     int32_t max_new_tokens, int32_t* out_tokens, int32_t* out_lengths, int32_t* all_done,
                                     const vqa_qwen25vl_sampling* sampling, void* workspace, size_t workspace_bytes, void* stream);

/* Number of kernels, memsets and copies the last forward call on this handle (vqa_clipt5_score, vqa_qwen25vl_score, vqa_qwen25vl_topk,
 * a generate prefill or step) enqueued (for bench.py's gpu_launches). */
int64_t vqa_last_launch_count(vqa_handle* h);

/* Optional device-side timing of the forward: with profiling on, every launch of a forward call (as above) is bracketed by CUDA
 * events on the caller's stream. After the caller synchronised the stream, vqa_profile_read returns, per category
 * {0 gemm, 1 attention, 2 norm, 3 other} (arrays of 4): device ms, algorithmic FLOPs (2MNK / 4*S*S*d), algorithmic bytes
 * (GEMM: A and W read once, C written once, residual read once) and scope counts of the LAST call. Used by bench.py for the
 * roofline object. */
int vqa_set_profile(vqa_handle* h, int32_t enable);
int vqa_profile_read(vqa_handle* h, float* ms, double* flops, double* bytes, int64_t* scopes);

/* Parity investigation aids: byte offsets, inside the caller-owned workspace of a call with the same sizes, of intermediate tensors
 * that the reference exposes too (encoder_last_hidden_state, decoder_hidden_states[-1], ...). Valid after the stream has passed
 * the scoring call. CLIP-FlanT5 (n >= 6): {encoder output, decoder output (both after the final T5LayerNorm), projector output,
 * encoder / decoder residual streams, last vision-tower hidden state (fp32)}. Qwen2.5-VL (n >= 4): {last-position hidden state after the
 * final norm, merged vision features, residual stream, last-position residual}; sizes as vqa_qwen25vl_workspace_bytes. */
int vqa_clipt5_debug_layout(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, int32_t label_len, size_t* offsets,
                            int32_t n);
int vqa_qwen25vl_debug_layout(vqa_handle* h, int32_t n_prompts, int64_t rows, int32_t n_patches, size_t* offsets, int32_t n);

/* Process-wide override of the GEMM tile order (tuning): group_rows > 0 = A rows per M group, chunk_rows > 0 = W rows per
 * L2-resident chunk, chunk_rows < 0 = one chunk; 0 = automatic. */
int vqa_set_gemm_schedule(int32_t group_rows, int32_t chunk_rows);

/* Tuning aid: number of clusters of `cluster_size` CTAs of the 256-wide GEMM kernel (one CTA per SM) the current device can hold at once
 * (cudaOccupancyMaxActiveClusters); negative vqa_status on error. */
int vqa_debug_max_active_clusters(int32_t cluster_size);

/* 1 when this process launches the GEMM and attention kernels with programmatic dependent launch (VQA_PDL=1, read once per process),
 * else 0. */
int vqa_debug_pdl_enabled(void);

/* Process-wide override of the image pre-processing tile plan (vqa_clip_preprocess, vqa_qwen_preprocess_video; tests and tuning): every
 * image gets tile_rows (1..32) output rows and min(tile_cols, out_w) output columns per CTA, i.e. ceil(out_w / tile_cols) column tiles,
 * and stages chunk_groups (1 or 2) groups of 4 canvas rows per pass. A plan call for an image whose forced plan does not fit
 * the kernel's shared memory fails with an error naming this override. All zero = the automatic plan (the default). */
int vqa_debug_set_preprocess_tiles(int32_t tile_rows, int32_t tile_cols, int32_t chunk_groups);

/* Host-only: the tile plan of each item of a pre-processing call, as the planner (with any override above) makes it. layout 0 = CLIP
 * (heights, widths, n_items, out_size, pad_to_square as vqa_clip_preprocess_workspace_bytes), 1 = Qwen patch rows (n_frames, heights,
 * widths, is_video, n_items, patch, temporal_patch, merge, min_pixels, max_pixels as vqa_qwen_preprocess_video_plan; n_frames and
 * is_video NULL = still images). geometry HOST [n_items][5] = (tile_rows, tile_cols, col_tiles, chunk_groups, band_groups). */
int vqa_debug_preprocess_geometry(int32_t layout, const int32_t* n_frames, const int32_t* heights, const int32_t* widths,
                                  const int32_t* is_video, int32_t n_items, int32_t out_size, int32_t pad_to_square, int32_t patch,
                                  int32_t temporal_patch, int32_t merge, int64_t min_pixels, int64_t max_pixels, int32_t* geometry);

/* Process-wide override of the output rows per CTA of the antialiased video-file resize (vqa_qwen_preprocess_video_aa; tests): any
 * tile_rows in 1..32. A plan call whose forced band of input rows does not fit the kernel's shared memory fails with an error naming
 * this override. 0 = the automatic plan (the default). */
int vqa_debug_set_preprocess_aa_rows(int32_t tile_rows);

/* Host-only: the launch geometry of vqa_qwen_preprocess_video_aa for these windows (arguments as vqa_qwen_preprocess_video_aa_plan),
 * with any override above. geometry HOST [3] = (tile_rows, band_rows, tiles_x): output rows per CTA, input rows of the tallest band,
 * 64-column tiles per row tile. */
int vqa_debug_preprocess_aa_geometry(int32_t in_h, int32_t in_w, int32_t out_h, int32_t out_w, const int32_t* first_h, int32_t htaps,
                                     const int32_t* first_v, int32_t vtaps, int32_t patch, int32_t merge, int32_t* geometry);

const char* vqa_last_error(vqa_handle* h);
void vqa_destroy(vqa_handle* h);

/* ---- image pre-processing on the device (SURVEY 8(f)2) ----
 * Replaces expand2square (t2v_metrics/models/vqascore_models/mm_utils.py:128-139) + the CLIP image processor of the v3.0 wrapper
 * (PIL BICUBIC resize of the shortest edge to out_size, centre crop, /255, (x - mean) / std): bit-identical to Pillow's integer
 * resampling (Resample.c) and to the fp32 normalisation of oracle/clipt5_oracle.py:clip_preprocess.
 *   src        DEVICE, the decoded images as packed HWC uint8 RGB, image i at byte offsets[i], heights[i] x widths[i] x 3
 *   offsets / heights / widths   HOST arrays [n_images]
 *   pad_to_square  1 = image_aspect_ratio 'pad' (centre on a max(h, w) square of `background`), 0 = plain resize + centre crop
 *   out        DEVICE [n_images, 3, out_size, out_size], out_dtype VQA_DTYPE_F32 or VQA_DTYPE_BF16
 *   workspace  DEVICE, >= vqa_clip_preprocess_workspace_bytes(...) (0 = bad arguments, see vqa_last_error(NULL))
 *   host_staging  optional HOST buffer of the same size, ideally pinned: the geometry + tap tables are written there and copied
 *              with ONE asynchronous cudaMemcpyAsync; the caller must leave it untouched until `stream` has passed this call.
 *              NULL: the tables are copied from the library's pageable memory (the runtime stages that copy synchronously). */
size_t vqa_clip_preprocess_workspace_bytes(const int32_t* heights, const int32_t* widths, int32_t n_images, int32_t out_size,
                                           int32_t pad_to_square);
int vqa_clip_preprocess(const void* src, const int64_t* offsets, const int32_t* heights, const int32_t* widths, int32_t n_images,
                        int32_t out_size, int32_t pad_to_square, const uint8_t* background, const float* mean, const float* stdv,
                        void* out, int32_t out_dtype, void* workspace, size_t workspace_bytes, void* host_staging, void* stream);

/* Qwen2.5-VL still images and decoded video frame stacks in one launch. Every frame gets the still-image pre-processing: smart_resize
 * (qwen_vl_utils / image_processing_qwen2_vl.py:62-87) + PIL-exact bicubic resize + /255 + normalise + 14x14 patch rows in 2x2 merge-block
 * order (image_processing_qwen2_vl.py:191-220); qwen_vl_utils fetch_video on a list of frames runs fetch_image on each. A stack then
 * goes through Qwen2VLVideoProcessor._preprocess with do_resize=False (video_processing_qwen2_vl.py:228-275): frames 2k and 2k+1 fill
 * temporal slots 0 and 1 of temporal group k's patch rows, and an odd last frame fills both (the processor's padding with copies of the
 * last frame; no second read of the source).
 *   n_frames / heights / widths / is_video   HOST arrays [n_items]; all frames of an item share its size. is_video[i] == 0: a still
 *              image (n_frames[i] must be 1), its frame written to every temporal slot, grid (1, gh, gw); else a video of
 *              ceil(n_frames / temporal_patch) temporal groups. A 1-frame video has the pixels of a still but is a video grid.
 *   frame_offsets  HOST [sum n_frames]: byte offset in `src` of every frame (HWC uint8 RGB), item by item.
 * vqa_qwen_preprocess_video_plan is host-only: grid_thw [n_items][3], total_patches = rows of `out`, workspace_bytes = device scratch.
 * out: DEVICE [total_patches, 3*temporal_patch*patch^2], item i's rows after those of items < i. At most 65535 frames per call. */
int vqa_qwen_preprocess_video_plan(const int32_t* n_frames, const int32_t* heights, const int32_t* widths, const int32_t* is_video,
                                   int32_t n_items, int32_t patch, int32_t temporal_patch, int32_t merge, int64_t min_pixels,
                                   int64_t max_pixels, int32_t* grid_thw, int64_t* total_patches, size_t* workspace_bytes);
int vqa_qwen_preprocess_video(const void* src, const int64_t* frame_offsets, const int32_t* n_frames, const int32_t* heights,
                              const int32_t* widths, const int32_t* is_video, int32_t n_items, int32_t patch, int32_t temporal_patch,
                              int32_t merge, int64_t min_pixels, int64_t max_pixels, const float* mean, const float* stdv, void* out,
                              int32_t out_dtype, void* workspace, size_t workspace_bytes, void* host_staging, void* stream);

/* Qwen2.5-VL frames sampled from a video FILE: qwen_vl_utils fetch_video resizes them as one tensor with torchvision
 * resize(BICUBIC, antialias=True) (torch's _upsample_bicubic2d_aa in fp32: the horizontal pass, then the vertical one, each output the
 * fused multiply-add of its taps in order; then clamp, round half to even, uint8), and the processor runs with do_resize=False. Here both
 * passes run on the device with torch's own fp32 weights, and the uint8 result goes to the same patch rows as vqa_qwen_preprocess_video
 * writes for a frame stack. One video is sent in slices of frames: each call takes frames [frame0, frame0 + n_frames) of a video of
 * total_frames frames and writes their temporal slots.
 *   first_h / first_v   HOST [out_w] / [out_h]: first input column / row of each output's window; windows inside the frame, rows
 *                       non-decreasing in the output row.
 *   weights_h / weights_v  HOST fp32 [out_w][htaps] / [out_h][vtaps]: the taps, zero-padded where a window is shorter.
 *   src      DEVICE uint8 [n_frames, in_h, in_w, 3] RGB.
 *   out      DEVICE [total_patches, 3*temporal_patch*patch^2]: the video's patch rows (same layout as vqa_qwen_preprocess_video's).
 * vqa_qwen_preprocess_video_aa_plan is host-only: total_patches = rows of the whole video, workspace_bytes = device scratch per call. */
int vqa_qwen_preprocess_video_aa_plan(int32_t in_h, int32_t in_w, int32_t out_h, int32_t out_w, const int32_t* first_h, int32_t htaps,
                                      const int32_t* first_v, int32_t vtaps, int32_t patch, int32_t temporal_patch, int32_t merge,
                                      int32_t total_frames, int64_t* total_patches, size_t* workspace_bytes);
int vqa_qwen_preprocess_video_aa(const void* src, int32_t n_frames, int32_t frame0, int32_t total_frames, int32_t in_h, int32_t in_w,
                                 int32_t out_h, int32_t out_w, const int32_t* first_h, const float* weights_h, int32_t htaps,
                                 const int32_t* first_v, const float* weights_v, int32_t vtaps, int32_t patch, int32_t temporal_patch,
                                 int32_t merge, const float* mean, const float* stdv, void* out, int32_t out_dtype, void* workspace,
                                 size_t workspace_bytes, void* host_staging, void* stream);

/* Host-only helper (no GPU needed): the 22-bit fixed-point bicubic tap table of one resize axis (in_size -> out_size, output
 * pixels [first, first + count)), exactly as vqa_clip_preprocess builds it after Pillow's precompute_coeffs /
 * normalize_coeffs_8bpc. bounds [count][2] = (first source index, taps used); kk [count][ksize]; returns ksize (0 = bad
 * arguments). Either output pointer may be NULL. */
int32_t vqa_resample_table(int32_t in_size, int32_t out_size, int32_t first, int32_t count, int32_t* bounds, int32_t* kk);

/* ---- kernel-level entry points (used by tests/ and bench.py to exercise single kernels through the same ABI) ----
 * Each one checks its arguments, then launches through the same stage function (grid, block, shared memory, arguments) as the forwards, so
 * a test of an entry point covers the launch the forwards make. */

/* C[M,N] = epilogue(A[M,K] . W[N,K]^T); all DEVICE bf16 row-major. epilogue: 0 store, 1 quick_gelu, 2 gelu(erf),
 * 3 gated gelu_new, 5 relu, 6 gated silu (C = bf16(bf16(silu(bf16(gate + b_gate))) * bf16(up + b_up)), the Qwen2.5-VL MLPs). The gated
 * epilogues 3 and 6 read W = [gate; up] with the up block `gate_up_offset` rows below the gate block (gate_up_offset + N/2 <= w_rows;
 * the bias is laid out the same way) and write C [M, N/2]; N/2 must be a multiple of 8.
 * bias [N] / residual [M, ldr] may be NULL. variant: 0 auto, else (BLOCK_N * 10 + rows / 128): 2561, 1281, 641, 321 are 128-row tiles
 * with BLOCK_N = 256 / 128 / 64 / 32. The two-CTA codes 2562 and 1282 of earlier hardware are still accepted and are aliases of 2561 and
 * 1281 (sm_90a has no CTA-pair MMA). Any other value is rejected. */
int vqa_op_gemm_bf16(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C, int32_t ldc,
                     int32_t M, int32_t N, int32_t K, const void* bias, const void* residual, int32_t ldr,
                     int32_t epilogue, int32_t gate_up_offset, int32_t variant, void* stream);

/* vqa_op_gemm_bf16 with the fused-RMSNorm hooks the encoder uses when emulate_bf16_rounding & 4 (T5LayerNorm, modeling_t5.py:55-68, folded
 * into the GEMMs around it). ssq_in DEVICE float [M, stride] or NULL: partial sums of squares of the rows of A; the epilogue multiplies
 * accumulator row m by rsqrt(sum_i ssq_in[m][i] / norm_dim + eps) before the Linear's bf16 rounding (W must carry the norm's gain:
 * W . diag(gamma)). ssq_out DEVICE float [M, stride] or NULL (epilogue 0 only): receives the partial sums of squares of the bf16 rows this
 * launch stores, slots [0, *parts_out); the caller zeroes the buffer first. stride % 4 == 0. No bias. */
int vqa_op_gemm_bf16_normfuse(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C, int32_t ldc, int32_t M, int32_t N,
                              int32_t K, const void* residual, int32_t ldr, int32_t epilogue, int32_t gate_up_offset, const float* ssq_in,
                              float* ssq_out, int32_t stride, int32_t norm_dim, float eps, int32_t* parts_out, void* stream);

/* The lm_head of vqa_qwen25vl_score with its fused log-softmax gather: with x_n = bf16(h[m].W[n]) in fp32, penalised where bit n of row m
 * of pen_bitmap [M, ceil(N / 32)] is set (x < 0 ? x * repetition_penalty : x / repetition_penalty; pen_bitmap NULL or penalty 1: none) and
 * divided by the temperature, logprob[m] = x_label[m] - logsumexp_n x_n. Logits are never stored; labels in [0, N). All DEVICE; K, ldh, ldw
 * multiples of 8 and >= K, H / W 16-byte aligned, temperature and penalty > 0. scratch DEVICE float: lse_max and lse_sum (M x 2 ceil(N / 128)
 * partials each), the label logits [M] and the scores [M]; *scratch_needed (HOST, optional) receives its size in bytes, also when a smaller
 * scratch_bytes returns VQA_ERR_WORKSPACE. */
int vqa_op_lmhead_logprob(const void* H, int32_t ldh, const void* W, int32_t ldw, int32_t M, int32_t N, int32_t K, const int32_t* labels,
                          float temperature, const uint32_t* pen_bitmap, float repetition_penalty, float* logprob, float* scratch,
                          size_t scratch_bytes, size_t* scratch_needed, void* stream);

/* The per-step kernel of a scored rollout (vqa_qwen25vl_generation.score) on caller-given bf16 logits [batch, V]: for every b with
 * done[b] == 0, row lengths[b] of out_logp [batch, max_new, n_max] (and of out_topk_ids / out_topk_probs [batch, max_new, top_k] when top_k > 0), under the penalty
 * bitmap pen_bitmap [batch, ceil(V / 32)] (NULL = none) and the temperature. All pointers DEVICE. */
int vqa_op_answer_logprob(const void* logits, int32_t batch, int32_t V, const uint32_t* pen_bitmap, float repetition_penalty, float temperature,
                          const int32_t* answer_ids, const int32_t* answer_counts, int32_t n_max, int32_t max_new, const int32_t* lengths,
                          const int32_t* done, int32_t top_k, float* out_logp, int32_t* out_topk_ids, float* out_topk_probs, void* stream);

/* The Qwen2.5-VL K/V cache write: the K and V heads (kv_heads x 128 columns at k_col0 / v_col0) of the packed rows qkv [B * S, ld] go to
 * kc / vc [B, kv_heads, cap, 128]. gen_len == NULL (prefill): row s of sequence b goes to slot s when s < seq_lens[b], padded rows are not
 * written (S <= cap). gen_len given (decode, S == 1): the row of sequence b goes to slot seq_lens[b] + gen_len[b] - 1. All DEVICE; ld,
 * k_col0, v_col0 multiples of 8, pointers 16-byte aligned. */
int vqa_op_kv_cache_write(const void* qkv, int32_t ld, int32_t k_col0, int32_t v_col0, int32_t kv_heads, int32_t B, int32_t S,
                          const int32_t* seq_lens, const int32_t* gen_len, void* kc, void* vc, int32_t cap, void* stream);

/* The decode-step attention of vqa_qwen25vl_generate_step (head_dim 128, flash-decoding): query row b (q heads at q + b * ldq + h * 128)
 * attends to cache slots [0, seq_lens[b] + gen_len[b]) of kc / vc [B, kv_heads, cap, 128], KV head h / (q_heads / kv_heads);
 * out[b * ldo + h * 128 + d] bf16. q_heads / kv_heads in {1, 2, 4, 5, 7, 8} (else VQA_ERR_UNSUPPORTED). The keys are cut into `splits`
 * ranges of ceil(cap / splits) slots (splits == 0: the generation's rule, returned in *splits_out; splits <= cap), merged by a second kernel;
 * workspace DEVICE >= B * q_heads * splits * 130 floats. ldq / ldo multiples of 4, q and caches 8-byte aligned. */
int vqa_op_decode_attention_d128(const void* q, int32_t ldq, const void* kc, const void* vc, int32_t cap, const int32_t* seq_lens,
                                 const int32_t* gen_len, int32_t B, int32_t q_heads, int32_t kv_heads, float scale, int32_t splits,
                                 void* workspace, size_t workspace_bytes, int32_t* splits_out, void* out, int32_t ldo, void* stream);

/* The token selection of the greedy generations on caller-owned state (all DEVICE): for every b with done[b] == 0, the arg-max (ties to the
 * lowest id) of the bf16 logits [B, V] cast to fp32, under HF's repetition penalty on the ids set in pen_bitmap [B, ceil(V / 32)] (NULL = no
 * penalty); the token goes to tokens[b, lengths[b]] and next_ids[b], its bit is set, lengths[b] advances, and with first_pos [B] / pos3 [3, B]
 * (both NULL or both given) pos3[:, b] = first_pos[b] + index of the token. A sequence finishes on one of eos_ids [n_eos] or at max_new
 * tokens: done[b] = 1, ++n_done, and the one that finishes the last of the B raises *all_done. */
int vqa_op_greedy_select(const void* logits, int32_t B, int32_t V, uint32_t* pen_bitmap, float repetition_penalty, const int32_t* eos_ids,
                         int32_t n_eos, int32_t max_new, const int32_t* first_pos, int32_t* tokens, int32_t* lengths, int32_t* done,
                         int32_t* n_done, int32_t* all_done, int32_t* next_ids, int32_t* pos3, void* stream);

/* The token selection of the sampled generation (vqa_qwen25vl_generate_*_sampled) on caller-owned state: vqa_op_greedy_select with the
 * arg-max replaced by a draw under `sampling` (HOST struct; its seeds DEVICE [B]); the draw of row b uses step t = lengths[b].
 * kept: NULL, or DEVICE [B, ceil(V / 32)] that receives the bitmap of the ids each unfinished row kept after top-k and top-p (a debugging
 * and test aid; the generation passes NULL). */
int vqa_op_sample_select(const void* logits, int32_t B, int32_t V, uint32_t* pen_bitmap, float repetition_penalty, const int32_t* eos_ids,
                         int32_t n_eos, int32_t max_new, const int32_t* first_pos, int32_t* tokens, int32_t* lengths, int32_t* done,
                         int32_t* n_done, int32_t* all_done, int32_t* next_ids, int32_t* pos3, const vqa_qwen25vl_sampling* sampling,
                         uint32_t* kept, void* stream);

/* The per-id terms vqa_op_sample_select decides on (a test aid), computed by the same device functions as its kernel, for every row b < B
 * (finished or not) at step t = lengths[b], with the same logits, penalty bitmap, penalty and sampling struct (top_k and top_p unused but
 * checked). All pointers DEVICE; every output [B, V] except row_max [B]:
 *   score     fp32 processed score (penalty, / temperature, -0 as +0, saturated)      row_max  the row's maximum score
 *   expv      fp32 expf(score - row_max)          mass     uint64 its mass in 2^-40 units, as the top-p cut sums it
 *   bits      uint32 Philox4x32-10 lane id % 4 of key seeds[b], counter (id / 4, t, 0, 0)
 *   gumbel_e  fp32 -log(u) of those bits          perturbed  fp32 (score - row_max) - log(gumbel_e), the draw's arg-max value */
int vqa_debug_sample_terms(const void* logits, int32_t B, int32_t V, const uint32_t* pen_bitmap, float repetition_penalty, const int32_t* lengths,
                           const vqa_qwen25vl_sampling* sampling, float* score, float* row_max, float* expv, uint64_t* mass, uint32_t* bits,
                           float* gumbel_e, float* perturbed, void* stream);

/* The encoder sharing of vqa_clipt5_generate_prefill_sampled on caller-owned buffers (tests): slots b >= n_prompts of xn bf16 [batch, S,
 * d_model], xt bf16 [batch, d_model, Sp] (Sp = S rounded up to 8) and seq_lens int32 [batch] become copies of slot prompt_index[b]
 * (clamped into [0, n_prompts)). All pointers DEVICE; xn and xt 16-byte aligned; d_model a multiple of 8; prompt_index may be NULL when
 * n_prompts == batch (nothing is launched). */
int vqa_op_clipt5_expand_prompts(void* xn, void* xt, int32_t* seq_lens, const int32_t* prompt_index, int32_t n_prompts, int32_t batch,
                                 int32_t S, int32_t d_model, void* stream);

/* Host-only (no GPU needed): T5's relative-position buckets (T5Attention._relative_position_bucket) of rel = -max_distance .. max_distance,
 * out[rel + max_distance], HOST int32 [2 * max_distance + 1] -- the table vqa_create_clipt5 builds for the encoder (bidirectional = 1) and
 * the decoder (0). */
int vqa_t5_bucket_lut(int32_t bidirectional, int32_t num_buckets, int32_t max_distance, int32_t* out);

/* The CLIP-FlanT5 scoring path's decoder self-attention (head_dim 64, causal, unidirectional buckets, no scale) over T <= 256 target rows:
 * packed qkv [B * T, 3 * H * 64] -> out [B * T, H * 64]. rel_emb [num_buckets, H] bf16, bucket_lut DEVICE int32 [2 * max_distance + 1]
 * (vqa_t5_bucket_lut). round_scores != 0: bf16 scores before and after the bias add, as the reference's eager attention forms them. */
int vqa_op_t5_decoder_self_attn(const void* qkv, void* out, const void* rel_emb, const int32_t* bucket_lut, int32_t max_distance, int32_t B,
                                int32_t T, int32_t H, int32_t round_scores, void* stream);

/* One cached decoder self-attention layer of vqa_clipt5_generate_step: the step's row qkv [B, 3 * H * 64] of sequence b sits at position
 * t = min(lengths[b], cap - 1); its K / V go to slot t of kc / vc [B, H, cap, 64] (cap <= 2048), then it attends to slots 0..t.
 * out [B, H * 64]; rel_emb / bucket_lut / round_scores as vqa_op_t5_decoder_self_attn. qkv and caches 16-byte aligned. */
int vqa_op_t5_decode_self_attn(const void* qkv, void* kc, void* vc, int32_t cap, const int32_t* lengths, void* out, const void* rel_emb,
                               const int32_t* bucket_lut, int32_t max_distance, int32_t B, int32_t H, int32_t round_scores, void* stream);

/* Bidirectional attention, head_dim 64, packed qkv [B*S, 3*H*64] -> out [B*S, H*64].
 * bias_table: DEVICE float [H, 2S-1] (index key - query + S - 1) or NULL; seq_lens DEVICE int32 [B] or NULL.
 * bias_const_from > 0: the caller guarantees bias_table[h][.] is constant for |key - query| >= bias_const_from on each side (T5's
 * relative_attention_max_distance, modeling_t5.py:189-234), which lets far key tiles fold the bias into one FFMA; 0: no assumption.
 * round_scores != 0: reproduce the bf16 tensors the reference's eager attention forms before its fp32 softmax (q.k^T as bf16, then the
 * bf16 `scores += position_bias`, modeling_t5.py:308-331); 0: scores and bias stay fp32.
 * B, S, H >= 1 with 3 * H * 64, B * S and H * B * ceil(S / 128) inside int32; qkv / out 16-byte aligned, bias_table / seq_lens 4-byte
 * aligned; with a bias table S <= 16496 (its row must fit in shared memory); else VQA_ERR_INVALID_ARG before anything launches. */
int vqa_op_attention_d64(const void* qkv, void* out, int32_t B, int32_t S, int32_t H, const int32_t* seq_lens,
                         const float* bias_table, float scale, int32_t bias_const_from, int32_t round_scores, void* stream);

/* T5LayerNorm / Qwen RMSNorm on [rows, D] bf16: y = gamma * bf16(x * rsqrt(mean(x^2) + eps)), fp32 statistics. D a multiple of 8 up to
 * 8192, rows >= 1; x, gamma and y 16-byte aligned; else VQA_ERR_INVALID_ARG before anything launches. */
int vqa_op_norm(const void* x, const void* gamma, void* y, int32_t rows, int32_t D, float eps, void* stream);

/* head_dim-128 attention on a packed buffer [rows, ld]: q heads at q_col0 + h*128, k/v heads at k_col0/v_col0 + (h/kv_group)*128,
 * out[row * ldo + h * 128 + d]. cu_seqlens [n_seq+1] (variable-length sequences) or NULL with fixed stride S and optional seq_lens [n_seq]:
 * then all S rows of every sequence are written, zeros past seq_lens[b], so S >= 1, n_seq * S <= rows and max_len >= S. q_heads a multiple
 * of kv_group; ld, ldo, the column offsets multiples of 8 with every head inside its row; qkv / out 16-byte aligned; else
 * VQA_ERR_INVALID_ARG before anything launches. */
int vqa_op_attention_d128(const void* qkv, int32_t ld, int64_t rows, int32_t q_col0, int32_t k_col0, int32_t v_col0, void* out,
                          int32_t ldo, int32_t n_seq, int32_t max_len, int32_t S, int32_t q_heads, int32_t kv_group,
                          const int32_t* cu_seqlens, const int32_t* seq_lens, float scale, int32_t causal, void* stream);

/* vqa_op_attention_d128 in variable-length mode with its extras: kv_prefix [n_seq] (or NULL): sequence b also attends to all rows of sequence
 * kv_prefix[b] >= 0, placed in front of its own keys; pair_sequences: two consecutive sequences (each <= 64 rows) share one 128-row tile under a
 * block-diagonal mask (non-causal, no kv_prefix, max_len <= 64); output head h is written at column h * o_head_stride, first d_out (multiple
 * of 8, <= 128 and <= o_head_stride) head dims only. The other checks are those of vqa_op_attention_d128. */
int vqa_op_attention_d128_ex(const void* qkv, int32_t ld, int64_t rows, int32_t q_col0, int32_t k_col0, int32_t v_col0, void* out, int32_t ldo,
                             int32_t n_seq, int32_t max_len, int32_t q_heads, int32_t kv_group, const int32_t* cu_seqlens, const int32_t* kv_prefix,
                             float scale, int32_t causal, int32_t pair_sequences, int32_t o_head_stride, int32_t d_out, void* stream);

/* Skinny GEMM (M <= 128): K cut into `splits` slices that run as one launch, fp32 partial tiles in `workspace` (splits * M * N floats), then one
 * reduction kernel: C = [residual +] bf16(A W^T + bias). splits == 0: the library picks (returned in *splits_out, may be 1). */
int vqa_op_gemm_bf16_splitk(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C, int32_t ldc, int32_t M, int32_t N,
                            int32_t K, const void* bias, const void* residual, int32_t ldr, int32_t splits, void* workspace,
                            size_t workspace_bytes, int32_t* splits_out, void* stream);

/* vqa_op_gemm_bf16 with the plain store epilogue, output columns written in groups: logical column c -> (c / group_in) * group_out + c % group_in. */
int vqa_op_gemm_bf16_grouped(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C, int32_t ldc, int32_t M, int32_t N,
                             int32_t K, const void* bias, int32_t group_in, int32_t group_out, int32_t variant, void* stream);

/* The CLIP tower's residual GEMMs (out_proj, fc2 under autocast): fp32 C[M, ldc] += bf16(A . W^T + bias) in place, the Linear's output rounded
 * to bf16 once and added to the fp32 stream unrounded. A / W bf16 as vqa_op_gemm_bf16 (lda, ldw, N, K multiples of 8, lda / ldw >= K);
 * C DEVICE float, ldc a multiple of 4 and >= N; bias [N] bf16 or NULL; variant as vqa_op_gemm_bf16. */
int vqa_op_gemm_bf16_f32acc(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, float* C, int32_t ldc, int32_t M, int32_t N,
                            int32_t K, const void* bias, int32_t variant, void* stream);

/* `nb` GEMMs of one shape in one launch, plain store epilogue: batch b computes C[b * c_stride + m * ldc + n] = bf16(sum_k A[m + b * a_row_off,
 * k + b * a_k_off] . W[n + b * w_row_off, k + b * w_k_off]) for m < M, n < N, k < K. A is read as an [a_rows, a_cols] matrix (row stride lda)
 * and W as [w_rows, w_cols] (ldw); rows past those extents read as zero, so a batch's last A or W rows may run past them (the absorbed
 * cross-attention's score GEMM reads Sp - S rows past the encoder output in its last batch). Accepted when every batch's first row lies
 * inside its operand's rows ((nb - 1) * a_row_off < a_rows, (nb - 1) * w_row_off < w_rows) and its K columns inside its columns
 * ((nb - 1) * a_k_off + K <= a_cols, likewise W); K a multiple of 64, or a_cols == K or w_cols == K (the k blocks are 64 columns wide
 * and are clipped only at the extents: with a K tail, the columns past K of the operand whose extent ends at K read as zero, and the other
 * operand's columns there, inside its extent, must be finite); lda, ldw, ldc, N, K, c_stride multiples of 8, a_cols <= lda, w_cols <= ldw, ldc >= N,
 * offsets >= 0, A / W / C 16-byte aligned; else VQA_ERR_INVALID_ARG. variant as vqa_op_gemm_bf16. */
int vqa_op_gemm_bf16_batched(const void* A, int32_t lda, const void* W, int32_t ldw, void* C, int32_t ldc, int32_t M, int32_t N, int32_t K,
                             int32_t nb, int32_t a_row_off, int32_t a_k_off, int32_t w_row_off, int32_t w_k_off, int64_t c_stride,
                             int64_t a_rows, int64_t a_cols, int64_t w_rows, int64_t w_cols, int32_t variant, void* stream);

/* One CLIP-FlanT5 decoder layer's cross-attention (head_dim 64, no scale, zero bias, encoder padding mask) as vqa_clipt5_score runs it:
 * decoder queries q [B * T, H * 64] against the encoder output x [B * S, d_model], pair b attending to its first seq_lens[b] rows
 * (1 <= seq_lens[b] <= S), into out [B * T, H * 64]. wkT = Wk^T [d_model, H * 64], wkv = [Wk; Wv] [2 * H * 64, d_model]. All DEVICE,
 * 16-byte aligned.
 *   mode 0 (cross_attention_mode 0, the absorbed association; round_scores unused, wkv's V half only): the encoder transpose, then
 *     q~ = Wk^T q, bf16 scores q~ . x, their masked fp32 softmax as bf16 P, ctx = P . x, out = Wv ctx. Workspace layout, each buffer
 *     starting at the next multiple of 256 bytes: xt [B, d_model, Sp] (Sp = S rounded up to 8; columns [S, Sp) zero) | q~ [B * T * H,
 *     d_model] (row (b * T + t) * H + h) | csc [B * T * H + 256, Sp] (row as q~: P, zero for keys >= seq_lens[b]) | ctx [B * T * H, d_model].
 *   mode 1 (the reference association, T <= 8 else VQA_ERR_UNSUPPORTED; wkT unused): kv = x . wkv^T [B * S, 2 * H * 64] in the workspace,
 *     then the flash-style kernel; round_scores != 0 rounds the scores to bf16 before the softmax.
 * workspace DEVICE, 256-byte aligned; *workspace_needed (HOST, optional) receives the bytes the call needs, also when it returns
 * VQA_ERR_WORKSPACE. */
int vqa_op_t5_cross_attention(const void* q, const void* x, const int32_t* seq_lens, const void* wkT, const void* wkv, void* out, int32_t B,
                              int32_t T, int32_t S, int32_t H, int32_t d_model, int32_t mode, int32_t round_scores, void* workspace,
                              size_t workspace_bytes, size_t* workspace_needed, void* stream);

/* nn.LayerNorm of the CLIP tower's fp32 residual stream (fp32 statistics): x DEVICE float [rows, D] -> y bf16 [rows, D]; gamma / beta bf16 [D].
 * D in {256, 512, 768, 1024} (else VQA_ERR_UNSUPPORTED); pointers 16-byte aligned. */
int vqa_op_layernorm_f32(const float* x, const void* gamma, const void* beta, void* y, int32_t rows, int32_t D, float eps, void* stream);

/* CLIP embeddings + pre_layrnorm: row t of image i is e = bf16(cls + pos[0]) for t = 0, bf16(patch[i * P + t - 1] + pos[t]) otherwise (the
 * reference adds in bf16), then LayerNorm(e) with fp32 statistics into y DEVICE float [n_images * (P + 1), D]. patch bf16 [n_images * P, D],
 * cls [D], pos [P + 1, D], gamma / beta [D]. D in {256, 1024} (else VQA_ERR_UNSUPPORTED); pointers 16-byte aligned. */
int vqa_op_clip_embed_ln(const void* patch, const void* cls, const void* pos, const void* gamma, const void* beta, float* y, int32_t n_images,
                         int32_t P, int32_t D, float eps, void* stream);

/* The CLIP-FlanT5 scoring path's glue kernels, launched as vqa_clipt5_score / vqa_clipt5_generate_* launch them. All pointers DEVICE. */

/* Patch gather for the patch-embedding GEMM: pixels [n_images, 3, image_size, image_size] (pixel_dtype F32 or BF16) -> out bf16
 * [n_images * P, kpad], P = (image_size / patch)^2, row i * P + py * (image_size / patch) + px, column c * patch^2 + ky * patch + kx holding
 * bf16(pixel); columns [3 * patch^2, kpad) are +0. kpad a multiple of 8 and >= 3 * patch^2; pixels aligned to their element size, out 16-byte
 * aligned. */
int vqa_op_patchify(const void* pixels, int32_t pixel_dtype, int32_t n_images, int32_t image_size, int32_t patch, int32_t kpad, void* out,
                    void* stream);

/* Multimodal splice into the encoder input out bf16 [B, S, D], S = L - 1 + P, and seq_lens int32 [B]. Row b's first text_lens[b] (1..L)
 * ids of ids int32 [B, L] are embedded with shared_emb bf16 [vocab, D] (ids in [0, vocab)), except that the first id equal to image_token
 * is replaced by the P feature rows of image image_index[b] (NULL: image b), rows [img * feat_rows_per_image + feat_row_offset, + P) of
 * feats bf16 (row stride ldf). seq_lens[b] = text_lens[b] - 1 + P with an image slot, text_lens[b] without; rows past it are +0. D and ldf
 * multiples of 8, ldf >= D, feat_row_offset + P <= feat_rows_per_image; shared_emb / feats / out 16-byte aligned. */
int vqa_op_splice_embed(const int32_t* ids, const int32_t* text_lens, const int32_t* image_index, const void* shared_emb, const void* feats,
                        int32_t ldf, int32_t feat_row_offset, int32_t feat_rows_per_image, void* out, int32_t* seq_lens, int32_t B, int32_t L,
                        int32_t P, int32_t D, int32_t image_token, void* stream);

/* Decoder input embeddings out bf16 [B * T, D] of shift_right(labels): row (b, 0) is shared_emb[start_id], row (b, t > 0) is
 * shared_emb[labels[b, t - 1]], or shared_emb[pad_id] for a negative label. labels int32 [B, T] (< vocab), or NULL with T = 1 (the
 * generation prefill's start token). D a multiple of 8; shared_emb / out 16-byte aligned. */
int vqa_op_decoder_embed(const int32_t* labels, const void* shared_emb, void* out, int32_t B, int32_t T, int32_t D, int32_t start_id,
                         int32_t pad_id, void* stream);

/* The T5 encoder's relative-position bias table: table float [H, 2S - 1], table[h, r] = rel_emb[bucket_lut[clamp(r - (S - 1), +-max_distance)
 * + max_distance], h] with rel_emb bf16 [num_buckets, H] and bucket_lut int32 [2 * max_distance + 1] (vqa_t5_bucket_lut). Past
 * |r - (S - 1)| >= max_distance every entry of a head and side equals the one at +-max_distance, which the encoder attention relies on
 * (bias_const_from = max_distance). */
int vqa_op_t5_bias_table(const void* rel_emb, const int32_t* bucket_lut, int32_t max_distance, float* table, int32_t H, int32_t S,
                         void* stream);

/* The tail of vqa_clipt5_score: the lm_head of H bf16 [B * T, ldh] against W bf16 [N, ldw] with its fused log-softmax gather of labels int32
 * [B, T] (< N; negative = ignored), then scores[b] = exp(mean of logprobs[b, t] over the labels of row b) (NaN when all are ignored) and,
 * unless logprobs is NULL, logprobs float [B * T] = bf16 logit of the label - logsumexp of the bf16 logits (ignored positions not written).
 * K, ldh, ldw multiples of 8 and >= K; H / W 16-byte aligned. scratch DEVICE float: the layout of vqa_op_lmhead_logprob at M = B * T (the
 * scores slot unused); *scratch_needed (HOST, optional) receives its size in bytes, also when a smaller scratch_bytes returns
 * VQA_ERR_WORKSPACE. */
int vqa_op_lmhead_score(const void* H, int32_t ldh, const void* W, int32_t ldw, int32_t B, int32_t T, int32_t N, int32_t K, const int32_t* labels,
                        float* scores, float* logprobs, float* scratch, size_t scratch_bytes, size_t* scratch_needed, void* stream);

/* Sum of squares of every row of x bf16 [rows, D] (fp32) into ssq float [rows, stride] at column 0, the seed of the fused-RMSNorm chain
 * (see vqa_op_gemm_bf16_normfuse); columns 1.. are not written. D a multiple of 8; x 16-byte aligned. */
int vqa_op_row_ssq(const void* x, float* ssq, int32_t rows, int32_t D, int32_t stride, void* stream);

/* The Qwen2.5-VL scoring path's glue kernels, launched as vqa_qwen25vl_score launches them. All pointers DEVICE. */

/* Rotary embedding (M-RoPE): the tables cos_t / sin_t [rows, 2 * half] float get, for i < half, angle = positions[axis_of_dim[i] * rows + row]
 * * inv_freq[i] (positions int32 [n_axes, rows], axis_of_dim int32 / inv_freq float [half]) and cos / sin(angle) at columns i and i + half;
 * then the n_heads heads of x bf16 [rows, ld] at columns col0 + h * head_stride are rotated in place over their first head_dim = 2 * half dims:
 * x' = x * cos + rotate_half(x) * sin. text_mode != 0: the tables are rounded to bf16 and every product is rounded to bf16 before the sum
 * (the language model); 0: fp32 throughout (the vision tower). head_dim a multiple of 16 and <= head_stride; ld, col0, head_stride multiples
 * of 8 with every head inside ld; x and the tables 16-byte aligned. */
int vqa_op_qwen_rope(const int32_t* positions, int32_t rows, const int32_t* axis_of_dim, const float* inv_freq, int32_t half, float* cos_t,
                     float* sin_t, void* x, int32_t ld, int32_t col0, int32_t n_heads, int32_t head_stride, int32_t head_dim, int32_t text_mode,
                     void* stream);

/* Row re-order: dst row r = src row index[r / group] * group + r % group for r < rows (rows a multiple of group), D bf16 columns (a multiple
 * of 8) per row: the vision tower's window order (group 4 = spatial_merge^2) and its inverse on the merged features (group 1). src / dst
 * 16-byte aligned. */
int vqa_op_gather_rows(const void* src, void* dst, const int32_t* index, int32_t rows, int32_t group, int32_t D, void* stream);

/* Embedding splice: row r = b * S + s of out [rows, D] (rows a multiple of S) is feats[feat_index[r]] when feat_index[r] >= 0, else
 * embed[ids[r]], for s < seq_lens[b]; zero past it (ids and feat_index are not read there). Padded rows: seq_lens [rows / S]; packed rows as
 * vqa_qwen25vl_score with a vqa_qwen25vl_packed: seq_lens = cu_seqlens + n_seq and S = rows. D a multiple of 8; embed / feats / out 16-byte aligned. */
int vqa_op_qwen_embed(const int32_t* ids, const int32_t* feat_index, const int32_t* seq_lens, const void* embed, const void* feats, void* out,
                      int32_t rows, int32_t S, int32_t D, void* stream);

/* Repetition-penalty bitmap: bit id of row b of bitmap uint32 [B, ceil(vocab / 32)] is OR-ed in for every prompt id of pair b with
 * 0 <= id < vocab (the caller zeroes the bitmap first). cu_seqlens NULL: padded prompts, ids [B, S], row b's first seq_lens[b] ids.
 * Otherwise packed rows: pair b's prompt is all of sequence kv_prefix[pair_seq[b]] (kv_prefix NULL or the entry < 0: none) followed by
 * sequence pair_seq[b], at most max_prompt_len ids in all. */
int vqa_op_token_bitmap(const int32_t* ids, const int32_t* seq_lens, int32_t B, int32_t S, const int32_t* cu_seqlens, const int32_t* kv_prefix,
                        const int32_t* pair_seq, int32_t max_prompt_len, int32_t vocab, uint32_t* bitmap, void* stream);

/* The trace output of vqa_qwen25vl_topk on caller bf16 logits [B, ldl] (ldl >= V): the K (1..8) most probable ids of each row, ties to the
 * lower id, into out_ids int32 / out_probs float [B, K], under the penalty bitmap pen_bitmap [B, ceil(V / 32)] (NULL or penalty 1: none)
 * and softmax(x / temperature) over all V. */
int vqa_op_topk_softmax(const void* logits, int64_t ldl, int32_t B, int32_t V, float temperature, const uint32_t* pen_bitmap,
                        float repetition_penalty, int32_t K, int32_t* out_ids, float* out_probs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VQA_B200_H */

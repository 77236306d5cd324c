// libvqa_b200.so -- C ABI of the VQAScore engine on one H100 (sm_90a). The model forwards (clipt5.cuh, qwen25vl.cuh) are fixed
// sequences of kernel launches on the caller's stream; no torch, no cuBLAS.
#include "clipt5.cuh"
#include "qwen25vl.cuh"
#include "preprocess.cuh"

// ------------------------------------------------------------------------------------------------ C ABI: lifecycle
extern "C" const char* vqa_version(void) {
    return "vqa_b200 abi=3 arch=sm_90a kernels=wgmma-gemm,flash-d64,t5-norm,lmhead-lse";
}

// Host mirror of T5Attention._relative_position_bucket (modeling_t5.py:189-234), fp32 like torch.
static int host_rel_bucket(int rel, bool bidirectional, int num_buckets, int max_distance) {
    int bucket = 0;
    if (bidirectional) {
        num_buckets /= 2;
        if (rel > 0) bucket += num_buckets;
        rel = abs(rel);
    } else {
        rel = -std::min(rel, 0);
    }
    const int max_exact = num_buckets / 2;
    if (rel < max_exact) return bucket + rel;
    float v = logf((float)rel / (float)max_exact) / (float)log((double)max_distance / (double)max_exact) *
              (float)(num_buckets - max_exact);
    int large = max_exact + (int)v;
    large = std::min(large, num_buckets - 1);
    return bucket + large;
}

// Host-only: the bucket of every clamped relative position rel in [-max_distance, max_distance], out[rel + max_distance] -- the table
// the attention kernels index (buckets saturate at |rel| = max_distance, so the clamp loses nothing).
extern "C" int vqa_t5_bucket_lut(int32_t bidirectional, int32_t num_buckets, int32_t max_distance, int32_t* out) {
    const int max_exact = bidirectional ? num_buckets / 4 : num_buckets / 2;
    if (!out || num_buckets < 4 || max_distance <= max_exact || max_distance > (1 << 20))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "bad bucket table request (num_buckets >= 4, exact range < max_distance <= 2^20)");
    for (int r = -max_distance; r <= max_distance; ++r) out[r + max_distance] = host_rel_bucket(r, bidirectional != 0, num_buckets, max_distance);
    return VQA_OK;
}

extern "C" int vqa_create_clipt5(const vqa_clipt5_config* cfg, int device, vqa_handle** out) {
    if (!cfg || !out) return fail(nullptr, VQA_ERR_INVALID_ARG, "null argument");
    if (cfg->vit_hidden % cfg->vit_heads || cfg->vit_hidden / cfg->vit_heads != 64)
        return fail(nullptr, VQA_ERR_UNSUPPORTED, "vision head_dim must be 64");
    if (cfg->image_size % cfg->patch_size) return fail(nullptr, VQA_ERR_INVALID_ARG, "image_size % patch_size != 0");
    if (cfg->d_model % 8 || cfg->d_ff % 64 || cfg->vit_hidden % 256)
        return fail(nullptr, VQA_ERR_UNSUPPORTED, "d_model % 8, d_ff % 64, vit_hidden % 256 must be 0");
    vqa_handle* h = new vqa_handle();
    h->cfg = *cfg;
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        g_global_err = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
        delete h;
        return VQA_ERR_CUDA;
    }
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess || prop.major != 9 || prop.minor != 0) {
        g_global_err = "vqa_b200 requires an sm_90 (H100) device";
        delete h;
        return VQA_ERR_UNSUPPORTED;
    }
    h->num_sms = prop.multiProcessorCount;
    const int kreal = 3 * cfg->patch_size * cfg->patch_size;
    h->kpad = (kreal + 63) / 64 * 64;
    // bucket LUTs
    const int md = cfg->rel_max_distance;
    std::vector<int> lb(2 * md + 1), lu(2 * md + 1);
    if (vqa_t5_bucket_lut(1, cfg->rel_buckets, md, lb.data()) != VQA_OK || vqa_t5_bucket_lut(0, cfg->rel_buckets, md, lu.data()) != VQA_OK) {
        delete h;
        return VQA_ERR_INVALID_ARG;
    }
    if (cudaMalloc(&h->lut_bidir, lb.size() * 4) != cudaSuccess || cudaMalloc(&h->lut_unidir, lu.size() * 4) != cudaSuccess ||
        cudaMemcpy(h->lut_bidir, lb.data(), lb.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(h->lut_unidir, lu.data(), lu.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
        g_global_err = "LUT allocation failed";
        delete h;
        return VQA_ERR_CUDA;
    }
    *out = h;
    return VQA_OK;
}

extern "C" int vqa_bind_weights(vqa_handle* h, const vqa_tensor* tensors, int32_t n) {
    if (!h || (!tensors && n > 0)) return fail(h, VQA_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n; ++i) {
        const vqa_tensor& t = tensors[i];
        if (!t.name || !t.data) return fail(h, VQA_ERR_INVALID_ARG, "tensor with null name/data");
        if (t.dtype != VQA_DTYPE_BF16) return fail(h, VQA_ERR_UNSUPPORTED, std::string(t.name) + ": weights must be bf16");
        if ((reinterpret_cast<uintptr_t>(t.data) & 15) != 0)
            return fail(h, VQA_ERR_INVALID_ARG, std::string(t.name) + ": pointer not 16-byte aligned");
        BoundTensor b;
        b.data = t.data; b.ndim = t.ndim;
        for (int d = 0; d < 4; ++d) b.shape[d] = (d < t.ndim) ? t.shape[d] : 1;
        h->tensors[t.name] = b;
    }
    h->finalized = false;
    return VQA_OK;
}

extern "C" int vqa_finalize_weights(vqa_handle* h) {
    if (!h) return VQA_ERR_INVALID_ARG;
    const int rc = h->kind == 1 ? qwen_finalize(h, *h->qwen) : clipt5_finalize(h);
    h->finalized = (rc == VQA_OK);
    return rc;
}

extern "C" size_t vqa_clipt5_workspace_bytes(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len,
                                             int32_t label_len) {
    if (!h || batch <= 0 || n_images <= 0 || text_len <= 0 || label_len <= 0) return 0;
    return plan_workspace(h, batch, n_images, text_len, label_len).total;
}

// ------------------------------------------------------------------------------------------------ forward
extern "C" int vqa_clipt5_score(vqa_handle* h, const void* pixels, int32_t pixel_dtype, int32_t n_images,
                                const int32_t* image_index, const int32_t* input_ids, const int32_t* text_lens,
                                const int32_t* labels, int32_t B, int32_t L, int32_t T, float* out_scores,
                                float* out_logprobs, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) return VQA_ERR_INVALID_ARG;
    if (h->kind != 0) return fail(h, VQA_ERR_INVALID_ARG, "not a CLIP-FlanT5 handle");
    if (!h->finalized) return fail(h, VQA_ERR_MISSING_WEIGHT, "vqa_finalize_weights has not succeeded");
    if (!pixels || !input_ids || !text_lens || !labels || !out_scores || !workspace)
        return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
    if (B <= 0 || L <= 0 || T <= 0 || n_images <= 0) return fail(h, VQA_ERR_INVALID_ARG, "non-positive size");
    if (T > 256) return fail(h, VQA_ERR_UNSUPPORTED, "label_len > 256 not supported by the decoder kernels");
    if (T > 8 && h->cfg.cross_attention_mode != 0)
        return fail(h, VQA_ERR_UNSUPPORTED, "label_len > 8 needs the absorbed cross-attention (cross_attention_mode = 0)");
    if (!image_index && n_images != B) return fail(h, VQA_ERR_INVALID_ARG, "image_index == NULL requires n_images == batch");
    if (pixel_dtype != VQA_DTYPE_F32 && pixel_dtype != VQA_DTYPE_BF16)
        return fail(h, VQA_ERR_INVALID_ARG, "pixel_dtype must be F32 or BF16");
    return clipt5_score(h, pixels, pixel_dtype, n_images, image_index, input_ids, text_lens, labels, B, L, T, out_scores, out_logprobs,
                        workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ CLIP-FlanT5 greedy generation
static int clipt5_gen_check(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, const ClipT5GenArgs& a, const void* workspace) {
    if (!h || h->kind != 0) return fail(h, VQA_ERR_INVALID_ARG, "not a CLIP-FlanT5 handle");
    if (!h->finalized) return fail(h, VQA_ERR_MISSING_WEIGHT, "vqa_finalize_weights has not succeeded");
    if ((a.n_eos > 0 && !a.eos_ids) || !a.tokens || !a.lengths || !a.all_done || !workspace) return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
    if (batch <= 0 || batch > 128 || n_images <= 0 || text_len <= 0 || a.max_new <= 0 || a.max_new > 2048 || a.n_eos < 0)
        return fail(h, VQA_ERR_INVALID_ARG, "bad size (1 <= batch <= 128, 1 <= max_new_tokens <= 2048)");
    if (h->cfg.cross_attention_mode != 0)
        return fail(h, VQA_ERR_UNSUPPORTED, "generation needs the absorbed cross-attention (cross_attention_mode = 0)");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(h, VQA_ERR_INVALID_ARG, "workspace must be 256-byte aligned");
    return VQA_OK;
}

extern "C" size_t vqa_clipt5_generate_workspace_bytes(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, int32_t max_new_tokens) {
    if (!h || h->kind != 0 || batch <= 0 || n_images <= 0 || text_len <= 0 || max_new_tokens <= 0) return 0;
    return clipt5_gen_plan(h, batch, n_images, text_len, max_new_tokens).total;
}

// A sampled generation's parameters (both models); the reference's scored forward is always greedy, so no answer score goes with them.
static int sampling_check(vqa_handle* h, const vqa_qwen25vl_sampling* s, const vqa_qwen25vl_answer_score* score) {
    if (!s || !s->seeds) return fail(h, VQA_ERR_INVALID_ARG, "sampling: null sampling struct or seeds");
    if (score) return fail(h, VQA_ERR_INVALID_ARG, "sampling: a scored rollout is greedy (gen->score must be NULL)");
    if (!(s->temperature > 0.f) || !std::isfinite(s->temperature) || s->top_k < 0 || !(s->top_p > 0.0) || !(s->top_p <= 1.0))
        return fail(h, VQA_ERR_INVALID_ARG, "sampling: bad parameters (temperature > 0 and finite, top_k >= 0, 0 < top_p <= 1)");
    return VQA_OK;
}

// The prefill and step of both CLIP-FlanT5 generations: smp NULL = greedy (n_prompts == batch, no prompt_index), else sampled.
static int clipt5_gen_prefill_entry(vqa_handle* h, const void* pixels, int32_t pixel_dtype, int32_t n_images, const int32_t* image_index,
                                    const int32_t* input_ids, const int32_t* text_lens, int32_t batch, int32_t text_len, const ClipT5GenArgs& a,
                                    int32_t n_prompts, const int32_t* prompt_index, const vqa_qwen25vl_sampling* smp, void* workspace,
                                    size_t workspace_bytes, void* stream) {
    if (int rc = clipt5_gen_check(h, batch, n_images, text_len, a, workspace)) return rc;
    if (!pixels || !input_ids || !text_lens) return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
    if (n_prompts < 1 || n_prompts > batch) return fail(h, VQA_ERR_INVALID_ARG, "1 <= n_prompts <= batch");
    if (n_prompts < batch && !prompt_index) return fail(h, VQA_ERR_INVALID_ARG, "prompt_index == NULL requires n_prompts == batch");
    if (!image_index && n_images != n_prompts) return fail(h, VQA_ERR_INVALID_ARG, "image_index == NULL requires n_images == n_prompts");
    if (pixel_dtype != VQA_DTYPE_F32 && pixel_dtype != VQA_DTYPE_BF16) return fail(h, VQA_ERR_INVALID_ARG, "pixel_dtype must be F32 or BF16");
    const ClipT5Prompts in{pixels, pixel_dtype, n_images, image_index, input_ids, text_lens, n_prompts, text_len};
    return clipt5_generate_prefill(h, in, batch, prompt_index, a, smp, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

static int clipt5_gen_step_entry(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, const ClipT5GenArgs& a,
                                 const vqa_qwen25vl_sampling* smp, void* workspace, size_t workspace_bytes, void* stream) {
    if (int rc = clipt5_gen_check(h, batch, n_images, text_len, a, workspace)) return rc;
    return clipt5_generate_step(h, batch, n_images, text_len, a, smp, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vqa_clipt5_generate_prefill(vqa_handle* h, const void* pixels, int32_t pixel_dtype, int32_t n_images, const int32_t* image_index,
                                           const int32_t* input_ids, const int32_t* text_lens, int32_t batch, int32_t text_len,
                                           const int32_t* eos_ids, int32_t n_eos, int32_t max_new_tokens, int32_t* out_tokens,
                                           int32_t* out_lengths, int32_t* all_done, void* workspace, size_t workspace_bytes, void* stream) {
    const ClipT5GenArgs a{eos_ids, n_eos, max_new_tokens, out_tokens, out_lengths, all_done};
    return clipt5_gen_prefill_entry(h, pixels, pixel_dtype, n_images, image_index, input_ids, text_lens, batch, text_len, a, batch, nullptr,
                                    nullptr, workspace, workspace_bytes, stream);
}

extern "C" int vqa_clipt5_generate_step(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, const int32_t* eos_ids, int32_t n_eos,
                                        int32_t max_new_tokens, int32_t* out_tokens, int32_t* out_lengths, int32_t* all_done, void* workspace,
                                        size_t workspace_bytes, void* stream) {
    const ClipT5GenArgs a{eos_ids, n_eos, max_new_tokens, out_tokens, out_lengths, all_done};
    return clipt5_gen_step_entry(h, batch, n_images, text_len, a, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int vqa_clipt5_generate_prefill_sampled(vqa_handle* h, const void* pixels, int32_t pixel_dtype, int32_t n_images,
                                                   const int32_t* image_index, const int32_t* input_ids, const int32_t* text_lens, int32_t batch,
                                                   int32_t text_len, const int32_t* eos_ids, int32_t n_eos, int32_t max_new_tokens,
                                                   int32_t* out_tokens, int32_t* out_lengths, int32_t* all_done, int32_t n_prompts,
                                                   const int32_t* prompt_index, const vqa_qwen25vl_sampling* sampling, void* workspace,
                                                   size_t workspace_bytes, void* stream) {
    if (int rc = sampling_check(h, sampling, nullptr)) return rc;
    const ClipT5GenArgs a{eos_ids, n_eos, max_new_tokens, out_tokens, out_lengths, all_done};
    return clipt5_gen_prefill_entry(h, pixels, pixel_dtype, n_images, image_index, input_ids, text_lens, batch, text_len, a, n_prompts,
                                    prompt_index, sampling, workspace, workspace_bytes, stream);
}

extern "C" int vqa_clipt5_generate_step_sampled(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, const int32_t* eos_ids,
                                                int32_t n_eos, int32_t max_new_tokens, int32_t* out_tokens, int32_t* out_lengths, int32_t* all_done,
                                                const vqa_qwen25vl_sampling* sampling, void* workspace, size_t workspace_bytes, void* stream) {
    if (int rc = sampling_check(h, sampling, nullptr)) return rc;
    const ClipT5GenArgs a{eos_ids, n_eos, max_new_tokens, out_tokens, out_lengths, all_done};
    return clipt5_gen_step_entry(h, batch, n_images, text_len, a, sampling, workspace, workspace_bytes, stream);
}

// Byte offsets inside the caller's workspace of the tensors a parity investigation wants to look at after a call has completed.
extern "C" int vqa_clipt5_debug_layout(vqa_handle* h, int32_t batch, int32_t n_images, int32_t text_len, int32_t label_len,
                                       size_t* offsets, int32_t n) {
    if (!h || h->kind != 0 || !offsets || n < 6 || batch <= 0 || n_images <= 0 || text_len <= 0 || label_len <= 0)
        return fail(h, VQA_ERR_INVALID_ARG, "bad debug layout argument");
    const ClipT5Workspace w = plan_workspace(h, batch, n_images, text_len, label_len);
    offsets[0] = w.xn;      // encoder output after the final T5LayerNorm  [B*S, d_model] bf16
    offsets[1] = w.yn;      // decoder output after the final T5LayerNorm  [B*T, d_model] bf16
    offsets[2] = w.proj2;   // projector output                            [NI*(P+1), d_model] bf16 (row 0 of each image = CLS)
    offsets[3] = w.x;       // encoder residual stream before the final norm
    offsets[4] = w.y;       // decoder residual stream before the final norm
    offsets[5] = w.hv;      // vision tower hidden states of the last executed layer [NI*(P+1), vit_hidden] FP32
    return VQA_OK;
}

extern "C" int vqa_qwen25vl_debug_layout(vqa_handle* h, int32_t n_prompts, int64_t rows, int32_t n_patches, size_t* offsets, int32_t n) {
    if (!h || h->kind != 1 || !offsets || n < 4 || n_prompts <= 0 || rows <= 0 || n_patches <= 0)
        return fail(h, VQA_ERR_INVALID_ARG, "bad debug layout argument");
    const QwenWorkspace w = qwen_plan_rows(h->qwen->cfg, n_prompts, (size_t)rows, n_patches);
    offsets[0] = w.lastn;       // last-position hidden state after the final RMSNorm [B, hidden] bf16
    offsets[1] = w.vfeat_orig;  // merged vision features in processor order         [n_patches / merge^2, out_hidden] bf16
    offsets[2] = w.x;           // language-model residual stream                     [B*S, hidden] bf16
    offsets[3] = w.last;        // last-position residual before the final norm       [B, hidden] bf16
    return VQA_OK;
}

// Process-wide override of the GEMM tile order (tuning / A-B measurements): group_rows > 0 = A rows per M group, chunk_rows > 0 = W rows
// per L2-resident chunk, chunk_rows < 0 = no chunking; 0 = automatic choice (gemm_sm90.cuh launch_gemm_t).
extern "C" int vqa_set_gemm_schedule(int32_t group_rows, int32_t chunk_rows) {
    g_gemm_group_rows_override = group_rows;
    g_gemm_chunk_rows_override = chunk_rows;
    return VQA_OK;
}

// 1 when this process launches the GEMM and attention kernels with programmatic dependent launch (VQA_PDL=1, read once), else 0.
extern "C" int vqa_debug_pdl_enabled(void) { return pdl_enabled() ? 1 : 0; }

// How many clusters of `cluster_size` CTAs of the 256-wide GEMM kernel (one CTA per SM: ~200 KB of shared memory) the current
// device can hold at once (cudaOccupancyMaxActiveClusters). 132 SMs do not always divide into GPC-local clusters of 4 or 8: this is the
// number a cluster-multicast variant of the GEMM has to be sized against. Returns the count, or a negative vqa_status.
extern "C" int vqa_debug_max_active_clusters(int32_t cluster_size) {
    if (cluster_size < 1 || cluster_size > 16) return VQA_ERR_INVALID_ARG;
    using Cfg = GemmConfig<256>;
    auto kernel = gemm_bf16_sm90_kernel<256, EPI_STORE, true>;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess) return VQA_ERR_CUDA;
    if (cluster_size > 8 && cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) return VQA_ERR_CUDA;
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(sms / cluster_size * cluster_size));
    cfg.blockDim = dim3(Cfg::NUM_THREADS);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeClusterDimension;
    attrs[0].val.clusterDim.x = (unsigned)cluster_size;
    attrs[0].val.clusterDim.y = 1;
    attrs[0].val.clusterDim.z = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) { cudaGetLastError(); return VQA_ERR_CUDA; }
    return n;
}

extern "C" int vqa_set_profile(vqa_handle* h, int32_t enable) {
    if (!h) return VQA_ERR_INVALID_ARG;
    h->profile = enable != 0;
    return VQA_OK;
}

// After the stream has been synchronised by the caller: device milliseconds, algorithmic FLOPs and launch-scope counts of
// the last vqa_clipt5_score call per category {0 gemm, 1 attention, 2 norm, 3 other}.
extern "C" int vqa_profile_read(vqa_handle* h, float* ms, double* flops, double* bytes, int64_t* scopes) {
    if (!h || !ms || !flops || !bytes || !scopes) return VQA_ERR_INVALID_ARG;
    for (int i = 0; i < CAT_COUNT; ++i) { ms[i] = 0.f; flops[i] = 0.0; bytes[i] = 0.0; scopes[i] = 0; }
    for (const auto& r : h->prof) {
        float t = 0.f;
        cudaError_t e = cudaEventElapsedTime(&t, h->ev_pool[r.ev0], h->ev_pool[r.ev1]);
        if (e != cudaSuccess) return fail(h, VQA_ERR_CUDA, std::string("cudaEventElapsedTime: ") + cudaGetErrorString(e));
        ms[r.cat] += t;
        flops[r.cat] += r.flops;
        bytes[r.cat] += r.bytes;
        scopes[r.cat] += 1;
    }
    return VQA_OK;
}

extern "C" int64_t vqa_last_launch_count(vqa_handle* h) { return h ? h->launches : 0; }
extern "C" const char* vqa_last_error(vqa_handle* h) { return h ? h->err.c_str() : g_global_err.c_str(); }
extern "C" void vqa_destroy(vqa_handle* h) {
    if (!h) return;
    if (h->lut_bidir) cudaFree(h->lut_bidir);
    if (h->lut_unidir) cudaFree(h->lut_unidir);
    for (cudaEvent_t e : h->ev_pool) cudaEventDestroy(e);
    if (h->qwen) {
        QwenState* q = h->qwen;
        if (q->text_axis) cudaFree(q->text_axis);
        if (q->vis_axis) cudaFree(q->vis_axis);
        if (q->text_inv_freq) cudaFree(q->text_inv_freq);
        if (q->vis_inv_freq) cudaFree(q->vis_inv_freq);
        delete q;
    }
    delete h;
}

// ------------------------------------------------------------------------------------------------ Qwen2.5-VL ABI
extern "C" int vqa_create_qwen25vl(const vqa_qwen25vl_config* cfg, int device, vqa_handle** out) {
    if (!cfg || !out) return fail(nullptr, VQA_ERR_INVALID_ARG, "null argument");
    if (cfg->heads % cfg->kv_heads) return fail(nullptr, VQA_ERR_INVALID_ARG, "heads % kv_heads != 0");
    if (cfg->vit_head_dim > 128 || cfg->vit_head_dim % 16 || cfg->vit_hidden != cfg->vit_heads * cfg->vit_head_dim)
        return fail(nullptr, VQA_ERR_UNSUPPORTED, "vision head_dim must be a multiple of 16, <= 128, and hidden = heads * head_dim");
    if (cfg->hidden % 8 || cfg->mlp % 128 || cfg->vit_hidden % 8 || cfg->patch_dim % 8)
        return fail(nullptr, VQA_ERR_UNSUPPORTED, "hidden % 8, mlp % 128, vit_hidden % 8, patch_dim % 8 must be 0");
    if (cfg->vit_depth > 64) return fail(nullptr, VQA_ERR_UNSUPPORTED, "vit_depth > 64");
    cudaError_t e = cudaSetDevice(device);
    cudaDeviceProp prop;
    if (e == cudaSuccess) e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess || prop.major != 9 || prop.minor != 0) return fail(nullptr, VQA_ERR_UNSUPPORTED, "vqa_b200 requires an sm_90 (H100) device");
    vqa_handle* h = new vqa_handle();
    h->kind = 1;
    h->num_sms = prop.multiProcessorCount;
    h->qwen = new QwenState();
    h->qwen->cfg = *cfg;
    *out = h;
    return VQA_OK;
}

extern "C" int vqa_qwen25vl_set_rope(vqa_handle* h, const float* text_inv_freq, const int32_t* text_axis, int32_t text_half,
                                     const float* vis_inv_freq, const int32_t* vis_axis, int32_t vis_half) {
    if (!h || h->kind != 1 || !text_inv_freq || !text_axis || !vis_inv_freq || !vis_axis)
        return fail(h, VQA_ERR_INVALID_ARG, "bad rope argument");
    QwenState& q = *h->qwen;
    if (text_half != 64 || vis_half != q.cfg.vit_head_dim / 2) return fail(h, VQA_ERR_INVALID_ARG, "rope table sizes do not match the config");
    auto up = [&](const void* src, size_t bytes, void** dst) -> bool {
        if (*dst) cudaFree(*dst);
        return cudaMalloc(dst, bytes) == cudaSuccess && cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice) == cudaSuccess;
    };
    if (!up(text_inv_freq, 64 * 4, (void**)&q.text_inv_freq) || !up(text_axis, 64 * 4, (void**)&q.text_axis) ||
        !up(vis_inv_freq, vis_half * 4, (void**)&q.vis_inv_freq) || !up(vis_axis, vis_half * 4, (void**)&q.vis_axis))
        return fail(h, VQA_ERR_CUDA, "rope table upload failed");
    q.rope_set = true;
    return VQA_OK;
}

// The ctypes mirrors in _lib.py are laid out by hand; tests/test_abi.py checks them against these numbers.
static_assert(sizeof(vqa_qwen25vl_prompts) == 112 && offsetof(vqa_qwen25vl_prompts, seq_len) == 108, "vqa_qwen25vl_prompts layout");
static_assert(sizeof(vqa_qwen25vl_packed) == 56 && offsetof(vqa_qwen25vl_packed, max_prompt_len) == 48, "vqa_qwen25vl_packed layout");
static_assert(sizeof(vqa_qwen25vl_answer_score) == 56 && offsetof(vqa_qwen25vl_answer_score, out_topk_probs) == 48,
              "vqa_qwen25vl_answer_score layout");
static_assert(sizeof(vqa_qwen25vl_generation) == 72 && offsetof(vqa_qwen25vl_generation, score) == 64, "vqa_qwen25vl_generation layout");
static_assert(sizeof(vqa_qwen25vl_sampling) == 24 && offsetof(vqa_qwen25vl_sampling, temperature) == 8 &&
              offsetof(vqa_qwen25vl_sampling, top_k) == 12 && offsetof(vqa_qwen25vl_sampling, top_p) == 16, "vqa_qwen25vl_sampling layout");

static int qwen_handle_check(vqa_handle* h) {
    if (!h || h->kind != 1) return fail(h, VQA_ERR_INVALID_ARG, "not a Qwen2.5-VL handle");
    if (!h->finalized) return fail(h, VQA_ERR_MISSING_WEIGHT, "vqa_finalize_weights has not succeeded");
    return VQA_OK;
}

// The inputs of a prefill; packed rows read neither seq_lens nor seq_len. After qwen_handle_check.
static int qwen_prompts_check(vqa_handle* h, const vqa_qwen25vl_prompts* p, bool packed) {
    if (!p || !p->pixel_patches || !p->vis_pos_hw || !p->window_index || !p->reverse_index || !p->cu_window || !p->cu_frames || !p->input_ids ||
        (!packed && !p->seq_lens) || !p->feat_index || !p->position_ids)
        return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
    const int unit = h->qwen->cfg.spatial_merge * h->qwen->cfg.spatial_merge;
    if (p->batch <= 0 || (!packed && p->seq_len <= 0) || p->n_patches <= 0 || p->n_patches % unit || p->n_windows <= 0 || p->n_frames <= 0)
        return fail(h, VQA_ERR_INVALID_ARG, "bad prompt / vision sizes");
    if (p->pixel_dtype != VQA_DTYPE_F32 && p->pixel_dtype != VQA_DTYPE_BF16) return fail(h, VQA_ERR_INVALID_ARG, "pixel_dtype must be F32 or BF16");
    return VQA_OK;
}

extern "C" size_t vqa_qwen25vl_workspace_bytes(vqa_handle* h, int32_t n_prompts, int64_t rows, int32_t n_patches) {
    if (!h || h->kind != 1 || n_prompts <= 0 || rows <= 0 || n_patches <= 0) return 0;
    return qwen_plan_rows(h->qwen->cfg, n_prompts, (size_t)rows, n_patches).total;
}

extern "C" int vqa_qwen25vl_score(vqa_handle* h, const vqa_qwen25vl_prompts* prompts, const vqa_qwen25vl_packed* packed, const int32_t* answer_ids,
                                  float temperature, float repetition_penalty, float* out_probs, float* out_logprobs, void* workspace,
                                  size_t workspace_bytes, void* stream) {
    if (int rc = qwen_handle_check(h)) return rc;
    if (int rc = qwen_prompts_check(h, prompts, packed != nullptr)) return rc;
    if (!answer_ids || !out_probs || !workspace) return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
    if (!(temperature > 0.f) || !(repetition_penalty > 0.f)) return fail(h, VQA_ERR_INVALID_ARG, "bad temperature / repetition penalty");
    if (packed) {
        if (!packed->cu_seqlens || !packed->kv_prefix || !packed->pair_row || !packed->pair_seq)
            return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
        if (packed->total_rows <= 0 || packed->n_seq <= 0 || packed->max_seq_len <= 0 || packed->max_prompt_len <= 0)
            return fail(h, VQA_ERR_INVALID_ARG, "bad packed sizes");
    }
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(h, VQA_ERR_INVALID_ARG, "workspace must be 256-byte aligned");
    return qwen_score(h, *h->qwen, *prompts, packed, answer_ids, temperature, repetition_penalty, out_probs, out_logprobs, workspace,
                      workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vqa_qwen25vl_topk(vqa_handle* h, int32_t batch, int64_t total_rows, int32_t n_patches, int32_t k, float temperature,
                                 float repetition_penalty, int32_t* out_ids, float* out_probs, void* workspace, size_t workspace_bytes, void* stream) {
    if (int rc = qwen_handle_check(h)) return rc;
    if (!out_ids || !out_probs || !workspace || batch <= 0 || total_rows <= 0 || n_patches <= 0 || k <= 0 || k > TOPK_MAX || !(temperature > 0.f) ||
        !(repetition_penalty > 0.f))
        return fail(h, VQA_ERR_INVALID_ARG, "bad top-k argument (1 <= k <= 8)");
    return qwen_topk(h, *h->qwen, batch, (size_t)total_rows, n_patches, k, temperature, repetition_penalty, out_ids, out_probs, workspace,
                     workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ Qwen2.5-VL greedy generation
static int qwen_rollout_check(vqa_handle* h, const vqa_qwen25vl_answer_score& s) {
    if (!s.answer_ids || !s.answer_counts || !s.out_logp || (s.top_k > 0 && (!s.out_topk_ids || !s.out_topk_probs)))
        return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
    if (s.n_max <= 0 || !(s.temperature > 0.f) || s.top_k < 0 || s.top_k > ANSWER_TOPK_MAX)
        return fail(h, VQA_ERR_INVALID_ARG, "bad answer size / temperature / top_k (n_max >= 1, temperature > 0, 0 <= top_k <= 8)");
    return VQA_OK;
}

static int qwen_gen_check(vqa_handle* h, const vqa_qwen25vl_generation* a, int32_t batch, int32_t seq_len, int32_t n_patches, const void* workspace) {
    if (!a) return fail(h, VQA_ERR_INVALID_ARG, "null generation");
    if (a->score)
        if (int rc = qwen_rollout_check(h, *a->score)) return rc;
    if (int rc = qwen_handle_check(h)) return rc;
    if (!a->seq_lens || !a->first_position || (a->n_eos > 0 && !a->eos_ids) || !a->out_tokens || !a->out_lengths || !a->all_done || !workspace)
        return fail(h, VQA_ERR_INVALID_ARG, "null device pointer");
    if (batch <= 0 || batch > 128 || seq_len <= 0 || n_patches <= 0 || a->max_new_tokens <= 0 || a->n_eos < 0 || !(a->repetition_penalty > 0.f))
        return fail(h, VQA_ERR_INVALID_ARG, "bad size / repetition penalty (1 <= batch <= 128, max_new_tokens >= 1)");
    if (!decode_attn_group_supported(h->qwen->cfg.heads / h->qwen->cfg.kv_heads))
        return fail(h, VQA_ERR_UNSUPPORTED, "decode attention supports 1, 2, 4, 5, 7 or 8 query heads per KV head");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(h, VQA_ERR_INVALID_ARG, "workspace must be 256-byte aligned");
    return VQA_OK;
}

extern "C" size_t vqa_qwen25vl_generate_workspace_bytes(vqa_handle* h, int32_t batch, int32_t seq_len, int32_t n_patches, int32_t max_new_tokens) {
    if (!h || h->kind != 1 || batch <= 0 || seq_len <= 0 || n_patches <= 0 || max_new_tokens <= 0) return 0;
    return qwen_gen_plan(h->qwen->cfg, batch, seq_len, n_patches, max_new_tokens, h->num_sms).total;
}

// The prefill and step of both generations: smp NULL = greedy, else sampled (checked by the _sampled entry points).
static int qwen_gen_prefill_entry(vqa_handle* h, const vqa_qwen25vl_prompts* prompts, const vqa_qwen25vl_generation* gen,
                                  const vqa_qwen25vl_sampling* smp, void* workspace, size_t workspace_bytes, void* stream) {
    if (!prompts) return fail(h, VQA_ERR_INVALID_ARG, "null prompts");
    if (int rc = qwen_gen_check(h, gen, prompts->batch, prompts->seq_len, prompts->n_patches, workspace)) return rc;
    if (int rc = qwen_prompts_check(h, prompts, false)) return rc;
    // the steps read the prompt lengths from gen->seq_lens: the prefill must have used the same ones
    if (gen->seq_lens != prompts->seq_lens) return fail(h, VQA_ERR_INVALID_ARG, "gen->seq_lens and prompts->seq_lens must be the same pointer");
    return qwen_generate_prefill(h, *h->qwen, *prompts, *gen, smp, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

static int qwen_gen_step_entry(vqa_handle* h, const vqa_qwen25vl_generation* gen, const vqa_qwen25vl_sampling* smp, int32_t batch,
                               int32_t seq_len, int32_t n_patches, void* workspace, size_t workspace_bytes, void* stream) {
    if (int rc = qwen_gen_check(h, gen, batch, seq_len, n_patches, workspace)) return rc;
    return qwen_generate_step(h, *h->qwen, batch, seq_len, n_patches, *gen, smp, workspace, workspace_bytes,
                              reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vqa_qwen25vl_generate_prefill(vqa_handle* h, const vqa_qwen25vl_prompts* prompts, const vqa_qwen25vl_generation* gen,
                                             void* workspace, size_t workspace_bytes, void* stream) {
    return qwen_gen_prefill_entry(h, prompts, gen, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int vqa_qwen25vl_generate_step(vqa_handle* h, const vqa_qwen25vl_generation* gen, int32_t batch, int32_t seq_len, int32_t n_patches,
                                          void* workspace, size_t workspace_bytes, void* stream) {
    return qwen_gen_step_entry(h, gen, nullptr, batch, seq_len, n_patches, workspace, workspace_bytes, stream);
}

extern "C" int vqa_qwen25vl_generate_prefill_sampled(vqa_handle* h, const vqa_qwen25vl_prompts* prompts, const vqa_qwen25vl_generation* gen,
                                                     const vqa_qwen25vl_sampling* sampling, void* workspace, size_t workspace_bytes,
                                                     void* stream) {
    if (int rc = sampling_check(h, sampling, gen ? gen->score : nullptr)) return rc;
    return qwen_gen_prefill_entry(h, prompts, gen, sampling, workspace, workspace_bytes, stream);
}

extern "C" int vqa_qwen25vl_generate_step_sampled(vqa_handle* h, const vqa_qwen25vl_generation* gen, const vqa_qwen25vl_sampling* sampling,
                                                  int32_t batch, int32_t seq_len, int32_t n_patches, void* workspace, size_t workspace_bytes,
                                                  void* stream) {
    if (int rc = sampling_check(h, sampling, gen ? gen->score : nullptr)) return rc;
    return qwen_gen_step_entry(h, gen, sampling, batch, seq_len, n_patches, workspace, workspace_bytes, stream);
}

// ------------------------------------------------------------------------------------------------ kernel-level ABI
static int device_sms() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    return sms;
}

// Every entry point below checks its arguments, then runs the stage function a forward runs (or f.gemm / f.attention / f.rmsnorm) through
// a Forward on the caller's stream and, when given, the caller's workspace. Its handle only counts the launches and keeps the error text.
template <typename Body>
static int glue_launch(void* stream, Body&& body, void* workspace = nullptr) {
    vqa_handle launcher;
    launcher.num_sms = device_sms();
    Forward f(&launcher, workspace, (cudaStream_t)stream);
    const int rc = body(f);
    return rc == VQA_OK ? VQA_OK : fail(nullptr, rc, launcher.err);
}

// a GEMM with the ABI's explicit layout
static Gemm abi_gemm(const void* A, int lda, const void* W, int ldw, int w_rows, void* C, int ldc, int M, int N, int K) {
    Gemm g((const bf16*)A, (const bf16*)W, C, M, N, K);
    g.lda = lda; g.ldw = ldw; g.w_rows = w_rows; g.ldc = ldc;
    return g;
}

static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// A gated epilogue stores its N / 2 output columns 8 at a time and reads the up block `gate_up_offset` rows below the gate block.
static int check_gated(int epilogue, int N, int w_rows, int gate_up_offset) {
    if (!epi_is_gated(epilogue)) return VQA_OK;
    if ((N / 2) % 8) return fail(nullptr, VQA_ERR_INVALID_ARG, "gated gemm: N / 2 must be a multiple of 8");
    if (gate_up_offset < 0 || (long long)gate_up_offset + N / 2 > w_rows)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "gated gemm: the up block [gate_up_offset, gate_up_offset + N / 2) must lie inside w_rows");
    return VQA_OK;
}

extern "C" int vqa_op_gemm_bf16(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C,
                                int32_t ldc, int32_t M, int32_t N, int32_t K, const void* bias, const void* residual,
                                int32_t ldr, int32_t epilogue, int32_t gate_up_offset, int32_t variant, void* stream) {
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad gemm argument");
    if (lda % 8 || ldw % 8 || ldc % 8 || N % 8 || K % 8) return fail(nullptr, VQA_ERR_INVALID_ARG, "gemm: ld/N/K must be multiples of 8");
    if (int rc = check_gated(epilogue, N, w_rows, gate_up_offset)) return rc;
    Gemm g = abi_gemm(A, lda, W, ldw, w_rows, C, ldc, M, N, K);
    g.bias = (const bf16*)bias; g.residual = residual; g.ldr = ldr; g.epi = epilogue; g.gate_up_offset = gate_up_offset; g.variant = variant;
    return glue_launch(stream, [&](Forward& f) { return f.gemm(g); });
}

// vqa_op_gemm_bf16 (plain store epilogue) whose output columns are written in groups: logical column c lands at (c / group_in) * group_out + c % group_in
// (heads narrower than the attention kernel's 128-wide slots are produced at their native width; the caller zeroes the slot padding).
extern "C" int vqa_op_gemm_bf16_grouped(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C, int32_t ldc, int32_t M,
                                        int32_t N, int32_t K, const void* bias, int32_t group_in, int32_t group_out, int32_t variant, void* stream) {
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0 || group_in <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad gemm argument");
    if (lda % 8 || ldw % 8 || ldc % 8 || N % 8 || K % 8) return fail(nullptr, VQA_ERR_INVALID_ARG, "gemm: ld/N/K must be multiples of 8");
    Gemm g = abi_gemm(A, lda, W, ldw, w_rows, C, ldc, M, N, K);
    g.bias = (const bf16*)bias; g.c_group_in = group_in; g.c_group_out = group_out; g.variant = variant;
    return glue_launch(stream, [&](Forward& f) { return f.gemm(g); });
}

// Skinny GEMM (M <= 128) with the K range cut into slices that run as one launch, partial tiles in `workspace` (fp32, splits * M * N floats; the
// slice count the library would pick is returned in *splits_out when splits == 0): C = [residual +] bf16(A W^T + bias).
extern "C" int vqa_op_gemm_bf16_splitk(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C, int32_t ldc, int32_t M, int32_t N,
                                       int32_t K, const void* bias, const void* residual, int32_t ldr, int32_t splits, void* workspace,
                                       size_t workspace_bytes, int32_t* splits_out, void* stream) {
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad gemm argument");
    if (lda % 8 || ldw % 8 || ldc % 8 || N % 8 || K % 8) return fail(nullptr, VQA_ERR_INVALID_ARG, "gemm: ld/N/K must be multiples of 8");
    if (splits == 0) splits = splitk_slices(M, N, K, device_sms());
    if (splits_out) *splits_out = splits;
    if (splits < 1 || K % (splits * 64)) return fail(nullptr, VQA_ERR_INVALID_ARG, "split-K: K must be a multiple of splits * 64");
    if (!workspace || workspace_bytes < (size_t)splits * M * N * 4) return fail(nullptr, VQA_ERR_WORKSPACE, "split-K workspace too small");
    Gemm g = abi_gemm(A, lda, W, ldw, w_rows, C, ldc, M, N, K);
    g.bias = (const bf16*)bias; g.residual = residual; g.ldr = ldr;
    return glue_launch(stream, [&](Forward& f) { return f.gemm(g.split_k(splits, (float*)workspace)); });
}

// vqa_op_gemm_bf16 with the fused-RMSNorm hooks (GemmParams::ssq_*): ssq_in [M, stride] partial sums of squares of the rows of A (the
// epilogue scales accumulator row m by rsqrt(sum / norm_dim + eps)), ssq_out [M, stride] receives this GEMM's partial sums of squares of the
// rows it stores (epilogue 0 only); either may be NULL. *parts_out (HOST, optional) = number of slots of ssq_out this launch writes.
extern "C" int vqa_op_gemm_bf16_normfuse(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, void* C, int32_t ldc, int32_t M,
                                         int32_t N, int32_t K, const void* residual, int32_t ldr, int32_t epilogue, int32_t gate_up_offset,
                                         const float* ssq_in, float* ssq_out, int32_t stride, int32_t norm_dim, float eps, int32_t* parts_out,
                                         void* stream) {
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0 || stride <= 0 || stride % 4 || norm_dim <= 0)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "bad gemm argument");
    if (lda % 8 || ldw % 8 || ldc % 8 || N % 8 || K % 8) return fail(nullptr, VQA_ERR_INVALID_ARG, "gemm: ld/N/K must be multiples of 8");
    if (int rc = check_gated(epilogue, N, w_rows, gate_up_offset)) return rc;
    const int variant = pick_variant(M, N, epilogue);
    const int parts = ssq_parts_for(variant, epi_is_gated(epilogue) ? N / 2 : N);
    if (parts_out) *parts_out = parts;
    if (ssq_out && parts > stride) return fail(nullptr, VQA_ERR_INVALID_ARG, "ssq stride smaller than the partial sums this launch writes");
    Gemm g = abi_gemm(A, lda, W, ldw, w_rows, C, ldc, M, N, K);
    g.residual = residual; g.ldr = ldr; g.epi = epilogue; g.gate_up_offset = gate_up_offset; g.variant = variant;
    g.nf.ssq_in = ssq_in; g.nf.ssq_out = ssq_out; g.nf.stride = stride; g.nf.inv_dim = 1.0f / (float)norm_dim; g.nf.eps = eps;
    return glue_launch(stream, [&](Forward& f) { return f.gemm(g); });
}

// Scratch of vqa_op_lmhead_logprob, in floats: lse_max | lse_sum ([M, LMHEAD_PARTS * n tiles] each) | label_logit [M] | scores [M].
static size_t lmhead_scratch_floats(int M, int N) {
    const size_t parts = (size_t)LMHEAD_PARTS * ((N + LMHEAD_BN - 1) / LMHEAD_BN);
    return 2 * (size_t)M * parts + 2 * (size_t)M;
}

extern "C" int vqa_op_lmhead_logprob(const void* Hs, int32_t ldh, const void* W, int32_t ldw, int32_t M, int32_t N, int32_t K,
                                     const int32_t* labels, float temperature, const uint32_t* pen_bitmap, float repetition_penalty,
                                     float* logprob, float* scratch, size_t scratch_bytes, size_t* scratch_needed, void* stream) {
    if (!Hs || !W || !labels || !logprob) return fail(nullptr, VQA_ERR_INVALID_ARG, "lmhead logprob: null pointer");
    if (M <= 0 || N <= 0 || K <= 0 || K % 8 || ldh % 8 || ldw % 8 || ldh < K || ldw < K)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "lmhead logprob: bad size (K, ldh, ldw multiples of 8, ldh / ldw >= K)");
    if (!(temperature > 0.f) || !(repetition_penalty > 0.f))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "lmhead logprob: temperature and repetition penalty must be > 0");
    if (!aligned(Hs, 16) || !aligned(W, 16) || !aligned(pen_bitmap, 4))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "lmhead logprob: H / W 16-byte aligned, pen_bitmap 4-byte aligned");
    const size_t need = lmhead_scratch_floats(M, N);
    if (scratch_needed) *scratch_needed = need * sizeof(float);
    if (!scratch || !aligned(scratch, 4) || scratch_bytes < need * sizeof(float))
        return fail(nullptr, VQA_ERR_WORKSPACE, "lmhead logprob: scratch smaller than lmhead_scratch_floats(M, N) floats");
    const size_t parts = (size_t)M * LMHEAD_PARTS * ((N + LMHEAD_BN - 1) / LMHEAD_BN);
    // one target per row; the scores exp(logprob) land in the scratch's last M floats and are not returned
    return glue_launch(stream, [&](Forward& f) {
        return lmhead_score(f, abi_gemm(Hs, ldh, W, ldw, N, nullptr, 0, M, N, K).processed(temperature, pen_bitmap, repetition_penalty), labels,
                            scratch, scratch + parts, scratch + 2 * parts, scratch + 2 * parts + M, logprob, M, 1);
    });
}

extern "C" int vqa_op_answer_logprob(const void* logits, int32_t batch, int32_t V, const uint32_t* pen_bitmap, float repetition_penalty,
                                     float temperature, const int32_t* answer_ids, const int32_t* answer_counts, int32_t n_max, int32_t max_new,
                                     const int32_t* lengths, const int32_t* done, int32_t top_k, float* out_logp, int32_t* out_topk_ids,
                                     float* out_topk_probs, void* stream) {
    if (!logits || !lengths || !done || batch <= 0 || V <= 0 || max_new <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad answer logprob argument");
    const vqa_qwen25vl_answer_score s{answer_ids, answer_counts, n_max, temperature, top_k, out_logp, out_topk_ids, out_topk_probs};
    if (int rc = qwen_rollout_check(nullptr, s)) return rc;
    return glue_launch(stream, [&](Forward& f) {
        return answer_logprob(f, (const bf16*)logits, batch, V, pen_bitmap, repetition_penalty, s, max_new, lengths, done);
    });
}

extern "C" int vqa_op_kv_cache_write(const void* qkv, int32_t ld, int32_t k_col0, int32_t v_col0, int32_t kv_heads, int32_t B, int32_t S,
                                     const int32_t* seq_lens, const int32_t* gen_len, void* kc, void* vc, int32_t cap, void* stream) {
    if (!qkv || !seq_lens || !kc || !vc) return fail(nullptr, VQA_ERR_INVALID_ARG, "kv cache write: null pointer");
    if (kv_heads <= 0 || B <= 0 || S <= 0 || cap <= 0 || S > cap || (gen_len && S != 1) || k_col0 < 0 || v_col0 < 0 ||
        ld < std::max(k_col0, v_col0) + kv_heads * 128)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "kv cache write: bad size (S <= cap, S == 1 in decode mode, heads inside ld)");
    if (ld % 8 || k_col0 % 8 || v_col0 % 8 || !aligned(qkv, 16) || !aligned(kc, 16) || !aligned(vc, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "kv cache write: ld, column offsets and pointers must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        return kv_cache_write(f, (const bf16*)qkv, ld, k_col0, v_col0, kv_heads, S, (long long)B * S, seq_lens, gen_len, (bf16*)kc, (bf16*)vc, cap);
    });
}

extern "C" int vqa_op_decode_attention_d128(const void* q, int32_t ldq, const void* kc, const void* vc, int32_t cap, const int32_t* seq_lens,
                                            const int32_t* gen_len, int32_t B, int32_t q_heads, int32_t kv_heads, float scale, int32_t splits,
                                            void* workspace, size_t workspace_bytes, int32_t* splits_out, void* out, int32_t ldo, void* stream) {
    if (!q || !kc || !vc || !seq_lens || !gen_len || !out) return fail(nullptr, VQA_ERR_INVALID_ARG, "decode attention: null pointer");
    if (B <= 0 || q_heads <= 0 || kv_heads <= 0 || cap <= 0 || splits < 0 || q_heads % kv_heads)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "decode attention: bad size (q_heads a multiple of kv_heads)");
    const int G = q_heads / kv_heads;
    if (!decode_attn_group_supported(G))
        return fail(nullptr, VQA_ERR_UNSUPPORTED, "decode attention supports 1, 2, 4, 5, 7 or 8 query heads per KV head");
    if (ldq < q_heads * 128 || ldo < q_heads * 128 || ldq % 4 || ldo % 4 || !aligned(q, 8) || !aligned(kc, 8) || !aligned(vc, 8) ||
        !aligned(out, 2))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "decode attention: ldq / ldo must cover the q heads and be multiples of 4, q / caches 8-byte aligned");
    if (splits == 0) splits = decode_attn_splits(B, kv_heads, cap, device_sms());
    if (splits_out) *splits_out = splits;
    if (splits > cap) return fail(nullptr, VQA_ERR_INVALID_ARG, "decode attention: more splits than cache slots");
    const size_t rows = (size_t)B * q_heads * splits;
    if (!workspace || !aligned(workspace, 4) || workspace_bytes < rows * 130 * 4)
        return fail(nullptr, VQA_ERR_WORKSPACE, "decode attention: workspace smaller than B * q_heads * splits * 130 floats");
    float* part_o = static_cast<float*>(workspace);
    return glue_launch(stream, [&](Forward& f) {
        return decode_attention(f, (const bf16*)q, ldq, (const bf16*)kc, (const bf16*)vc, cap, seq_lens, gen_len, B, q_heads, kv_heads, scale, splits,
                                part_o, part_o + rows * 128, (bf16*)out, ldo);
    });
}

extern "C" int vqa_op_greedy_select(const void* logits, int32_t B, int32_t V, uint32_t* pen_bitmap, float repetition_penalty, const int32_t* eos_ids,
                                    int32_t n_eos, int32_t max_new, const int32_t* first_pos, int32_t* tokens, int32_t* lengths, int32_t* done,
                                    int32_t* n_done, int32_t* all_done, int32_t* next_ids, int32_t* pos3, void* stream) {
    if (!logits || !tokens || !lengths || !done || !n_done || !all_done || !next_ids || (n_eos > 0 && !eos_ids) || (!first_pos != !pos3))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "greedy select: null pointer (first_pos and pos3 are given together or not at all)");
    if (B <= 0 || V <= 0 || max_new <= 0 || n_eos < 0 || !(repetition_penalty > 0.f))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "greedy select: bad size / repetition penalty");
    return glue_launch(stream, [&](Forward& f) {
        return greedy_select(f, (const bf16*)logits, B, V, pen_bitmap, repetition_penalty, eos_ids, n_eos, max_new, first_pos, tokens, lengths, done,
                             n_done, all_done, next_ids, pos3);
    });
}

extern "C" int vqa_op_sample_select(const void* logits, int32_t B, int32_t V, uint32_t* pen_bitmap, float repetition_penalty, const int32_t* eos_ids,
                                    int32_t n_eos, int32_t max_new, const int32_t* first_pos, int32_t* tokens, int32_t* lengths, int32_t* done,
                                    int32_t* n_done, int32_t* all_done, int32_t* next_ids, int32_t* pos3, const vqa_qwen25vl_sampling* sampling,
                                    uint32_t* kept, void* stream) {
    if (!logits || !tokens || !lengths || !done || !n_done || !all_done || !next_ids || (n_eos > 0 && !eos_ids) || (!first_pos != !pos3))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "sample select: null pointer (first_pos and pos3 are given together or not at all)");
    if (B <= 0 || V <= 0 || max_new <= 0 || n_eos < 0 || !(repetition_penalty > 0.f))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "sample select: bad size / repetition penalty");
    if (int rc = sampling_check(nullptr, sampling, nullptr)) return rc;
    return glue_launch(stream, [&](Forward& f) {
        return sample_select(f, (const bf16*)logits, B, V, pen_bitmap, repetition_penalty, *sampling, eos_ids, n_eos, max_new, first_pos, tokens,
                             lengths, done, n_done, all_done, next_ids, pos3, kept);
    });
}

extern "C" int vqa_debug_sample_terms(const void* logits, int32_t B, int32_t V, const uint32_t* pen_bitmap, float repetition_penalty,
                                      const int32_t* lengths, const vqa_qwen25vl_sampling* sampling, float* score, float* row_max, float* expv,
                                      uint64_t* mass, uint32_t* bits, float* gumbel_e, float* perturbed, void* stream) {
    if (!logits || !lengths || !score || !row_max || !expv || !mass || !bits || !gumbel_e || !perturbed)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "sample terms: null pointer");
    if (B <= 0 || V <= 0 || !(repetition_penalty > 0.f)) return fail(nullptr, VQA_ERR_INVALID_ARG, "sample terms: bad size / repetition penalty");
    if (int rc = sampling_check(nullptr, sampling, nullptr)) return rc;
    return glue_launch(stream, [&](Forward& f) {
        return sample_terms(f, (const bf16*)logits, B, V, pen_bitmap, repetition_penalty, *sampling, lengths, score, row_max, expv,
                            (unsigned long long*)mass, bits, gumbel_e, perturbed);
    });
}

extern "C" int vqa_op_clipt5_expand_prompts(void* xn, void* xt, int32_t* seq_lens, const int32_t* prompt_index, int32_t n_prompts, int32_t batch,
                                            int32_t S, int32_t d_model, void* stream) {
    if (!xn || !xt || !seq_lens || (n_prompts < batch && !prompt_index)) return fail(nullptr, VQA_ERR_INVALID_ARG, "expand prompts: null pointer");
    if (n_prompts < 1 || n_prompts > batch || S <= 0 || d_model <= 0 || d_model % 8)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "expand prompts: bad size (1 <= n_prompts <= batch, d_model a multiple of 8)");
    if (!aligned(xn, 16) || !aligned(xt, 16)) return fail(nullptr, VQA_ERR_INVALID_ARG, "expand prompts: xn and xt must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        return clipt5_expand_prompts(f, prompt_index, n_prompts, batch, S, d_model, (bf16*)xn, (bf16*)xt, seq_lens);
    });
}

static int check_t5_self_attn(const void* qkv, const void* out, const void* rel_emb, const int32_t* bucket_lut, int max_distance, int B, int H) {
    if (!qkv || !out || !rel_emb || !bucket_lut) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 self attention: null pointer");
    if (B <= 0 || H <= 0 || max_distance <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 self attention: bad size");
    if (!aligned(qkv, 4) || !aligned(out, 4)) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 self attention: qkv / out must be 4-byte aligned");
    return VQA_OK;
}

extern "C" int vqa_op_t5_decoder_self_attn(const void* qkv, void* out, const void* rel_emb, const int32_t* bucket_lut, int32_t max_distance, int32_t B,
                                           int32_t T, int32_t H, int32_t round_scores, void* stream) {
    if (int rc = check_t5_self_attn(qkv, out, rel_emb, bucket_lut, max_distance, B, H)) return rc;
    if (T <= 0 || T > 256) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 decoder self attention: 1 <= T <= 256");
    return glue_launch(stream, [&](Forward& f) {
        return clipt5_decoder_self_attention(f, (const bf16*)qkv, (bf16*)out, (const bf16*)rel_emb, bucket_lut, max_distance, B, T, H, round_scores);
    });
}

extern "C" int vqa_op_t5_decode_self_attn(const void* qkv, void* kc, void* vc, int32_t cap, const int32_t* lengths, void* out, const void* rel_emb,
                                          const int32_t* bucket_lut, int32_t max_distance, int32_t B, int32_t H, int32_t round_scores, void* stream) {
    if (int rc = check_t5_self_attn(qkv, out, rel_emb, bucket_lut, max_distance, B, H)) return rc;
    if (!kc || !vc || !lengths) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 decode self attention: null pointer");
    if (cap <= 0 || cap > 2048) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 decode self attention: 1 <= cap <= 2048");
    if (!aligned(qkv, 16) || !aligned(kc, 16) || !aligned(vc, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 decode self attention: qkv and caches must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        return clipt5_cached_self_attention(f, (const bf16*)qkv, (bf16*)kc, (bf16*)vc, cap, lengths, (bf16*)out, (const bf16*)rel_emb, bucket_lut,
                                            max_distance, B, H, round_scores);
    });
}

// What attn64_ws_kernel trusts of its arguments: int32 row / column / work-item arithmetic, 16-byte aligned TMA rows and output rows, 4-byte
// aligned lengths and bias entries, and a padded bias row that fits in shared memory next to the 2-stage K/V ring.
static int check_attn_d64(const void* qkv, const void* out, int B, int S, int H, const int32_t* seq_lens, const float* bias_table) {
    if (!qkv || !out) return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d64: null pointer");
    if (B < 1 || S < 1 || H < 1) return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d64: B, S and H must be >= 1");
    if (3LL * H * 64 > INT32_MAX || (long long)B * S > INT32_MAX || (long long)H * B * ((S + 127LL) / 128) > INT32_MAX)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d64: 3 * H * 64, B * S and H * B * ceil(S / 128) must fit in int32");
    if (!aligned(qkv, 16) || !aligned(out, 16) || !aligned(bias_table, 4) || !aligned(seq_lens, 4))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d64: qkv / out 16-byte aligned, bias_table / seq_lens 4-byte aligned");
    if (bias_table && S > attn64_max_bias_len(2))
        return fail(nullptr, VQA_ERR_INVALID_ARG,
                    "attention d64: with a bias table S must be <= " + std::to_string(attn64_max_bias_len(2)) + " (its row must fit in shared memory)");
    return VQA_OK;
}

extern "C" int vqa_op_attention_d64(const void* qkv, void* out, int32_t B, int32_t S, int32_t H, const int32_t* seq_lens,
                                    const float* bias_table, float scale, int32_t bias_const_from, int32_t round_scores, void* stream) {
    if (int rc = check_attn_d64(qkv, out, B, S, H, seq_lens, bias_table)) return rc;
    return glue_launch(stream, [&](Forward& f) {
        return clipt5_attention_d64(f, "attention", (const bf16*)qkv, (bf16*)out, B, S, H, seq_lens, bias_table, scale, bias_const_from,
                                    round_scores != 0);
    });
}

// What attn_wgmma_kernel trusts of its arguments: every q / k / v head inside the row of `ld` columns, 16-byte aligned TMA columns and
// output rows, every output head inside the row of `ldo` columns.
static int check_attn_d128(const void* qkv, int ld, long long rows, int q_col0, int k_col0, int v_col0, const void* out, int ldo, int n_seq,
                           int max_len, int q_heads, int kv_group, int o_head_stride, int d_out) {
    if (!qkv || !out) return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: null pointer");
    if (rows <= 0 || n_seq <= 0 || max_len <= 0 || q_heads <= 0 || kv_group <= 0 || q_heads % kv_group)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: bad size (q_heads a multiple of kv_group)");
    if (ld % 8 || ldo % 8 || q_col0 % 8 || k_col0 % 8 || v_col0 % 8 || q_col0 < 0 || k_col0 < 0 || v_col0 < 0 || !aligned(qkv, 16) ||
        !aligned(out, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: ld, ldo and column offsets multiples of 8, qkv / out 16-byte aligned");
    const long long kv_cols = (long long)(q_heads / kv_group) * 128;
    if ((long long)q_col0 + (long long)q_heads * 128 > ld || k_col0 + kv_cols > ld || v_col0 + kv_cols > ld)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: q / k / v heads must lie inside ld");
    if (d_out < 8 || d_out > 128 || d_out % 8 || o_head_stride % 8 || o_head_stride < d_out ||
        (long long)(q_heads - 1) * o_head_stride + d_out > ldo)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: 8 <= d_out <= 128 and o_head_stride multiples of 8, output heads inside ldo");
    return VQA_OK;
}

extern "C" int vqa_op_attention_d128(const void* qkv, int32_t ld, int64_t rows, int32_t q_col0, int32_t k_col0, int32_t v_col0,
                                     void* out, int32_t ldo, int32_t n_seq, int32_t max_len, int32_t S, int32_t q_heads, int32_t kv_group,
                                     const int32_t* cu_seqlens, const int32_t* seq_lens, float scale, int32_t causal, void* stream) {
    if (int rc = check_attn_d128(qkv, ld, rows, q_col0, k_col0, v_col0, out, ldo, n_seq, max_len, q_heads, kv_group, 128, 128)) return rc;
    // fixed stride: the kernel writes all S rows of every sequence (zeros past seq_lens[b]), so they must lie inside `rows` and the grid,
    // which covers max_len rows per sequence, must reach them
    if (!cu_seqlens && (S < 1 || (long long)n_seq * S > rows || max_len < S))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: fixed stride needs S >= 1, n_seq * S <= rows and max_len >= S");
    return glue_launch(stream, [&](Forward& f) {
        return f.attention(0, "attention d128", [&] {
            return launch_attn_tc128((const bf16*)qkv, ld, rows, q_col0, k_col0, v_col0, (bf16*)out, ldo, n_seq, max_len, S, q_heads, kv_group,
                                     cu_seqlens, seq_lens, scale, causal != 0, f.st);
        });
    });
}

// The same kernel with its variable-length extras: a shared key/value prefix per sequence, two short sequences per 128-row tile, compact output heads.
extern "C" int vqa_op_attention_d128_ex(const void* qkv, int32_t ld, int64_t rows, int32_t q_col0, int32_t k_col0, int32_t v_col0,
                                        void* out, int32_t ldo, int32_t n_seq, int32_t max_len, int32_t q_heads, int32_t kv_group,
                                        const int32_t* cu_seqlens, const int32_t* kv_prefix, float scale, int32_t causal,
                                        int32_t pair_sequences, int32_t o_head_stride, int32_t d_out, void* stream) {
    if (!cu_seqlens) return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: null cu_seqlens");
    if (int rc = check_attn_d128(qkv, ld, rows, q_col0, k_col0, v_col0, out, ldo, n_seq, max_len, q_heads, kv_group, o_head_stride, d_out))
        return rc;
    if (pair_sequences && (max_len > 64 || causal || kv_prefix))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "attention d128: pair_sequences takes sequences of <= 64 rows, non-causal, without kv_prefix");
    return glue_launch(stream, [&](Forward& f) {
        return f.attention(0, "attention d128", [&] {
            return launch_attn_tc128((const bf16*)qkv, ld, rows, q_col0, k_col0, v_col0, (bf16*)out, ldo, n_seq, max_len, 0, q_heads, kv_group,
                                     cu_seqlens, nullptr, scale, causal != 0, f.st, kv_prefix, pair_sequences != 0, o_head_stride, d_out);
        });
    });
}

extern "C" int vqa_op_norm(const void* x, const void* gamma, void* y, int32_t rows, int32_t D, float eps, void* stream) {
    if (!x || !gamma || !y) return fail(nullptr, VQA_ERR_INVALID_ARG, "norm: null pointer");
    if (rows <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "norm: rows must be >= 1");
    if (D <= 0 || D % 8 || D > 8192) return fail(nullptr, VQA_ERR_INVALID_ARG, "norm: D must be a multiple of 8 up to 8192");
    if (!aligned(x, 16) || !aligned(gamma, 16) || !aligned(y, 16)) return fail(nullptr, VQA_ERR_INVALID_ARG, "norm: x / gamma / y must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) { return f.rmsnorm((const bf16*)x, (const bf16*)gamma, (bf16*)y, rows, D, eps); });
}

// ------------------------------------------------------------------------------------------------ kernel-level ABI: the CLIP-FlanT5 scoring path
static bool gemm_variant_known(int v) { return v == 0 || v == 2561 || v == 2562 || v == 1281 || v == 1282 || v == 641 || v == 321; }

// The CLIP tower's residual GEMMs (out_proj, fc2): fp32 C[M, ldc] += bf16(A W^T + bias), in place.
extern "C" int vqa_op_gemm_bf16_f32acc(const void* A, int32_t lda, const void* W, int32_t ldw, int32_t w_rows, float* C, int32_t ldc, int32_t M,
                                       int32_t N, int32_t K, const void* bias, int32_t variant, void* stream) {
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0 || w_rows <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "fp32-accumulate gemm: bad argument");
    if (lda % 8 || ldw % 8 || N % 8 || K % 8 || ldc % 4 || lda < K || ldw < K || ldc < N)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "fp32-accumulate gemm: lda / ldw / N / K multiples of 8 and >= K, ldc a multiple of 4 and >= N");
    if (!aligned(A, 16) || !aligned(W, 16) || !aligned(C, 16) || !aligned(bias, 8))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "fp32-accumulate gemm: A / W / C 16-byte aligned, bias 8-byte aligned");
    if (!gemm_variant_known(variant)) return fail(nullptr, VQA_ERR_INVALID_ARG, "fp32-accumulate gemm: unknown tile variant");
    Gemm g = abi_gemm(A, lda, W, ldw, w_rows, C, ldc, M, N, K);
    g.bias = (const bf16*)bias; g.variant = variant;
    return glue_launch(stream, [&](Forward& f) { return f.gemm(g.accumulate_f32()); });
}

// `nb` GEMMs of one shape in one launch (BatchSpec), plain store epilogue. See include/vqa_b200.h for the acceptance rule.
extern "C" int vqa_op_gemm_bf16_batched(const void* A, int32_t lda, const void* W, int32_t ldw, void* C, int32_t ldc, int32_t M, int32_t N, int32_t K,
                                        int32_t nb, int32_t a_row_off, int32_t a_k_off, int32_t w_row_off, int32_t w_k_off, int64_t c_stride,
                                        int64_t a_rows, int64_t a_cols, int64_t w_rows, int64_t w_cols, int32_t variant, void* stream) {
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0 || nb <= 0 || a_rows <= 0 || a_cols <= 0 || w_rows <= 0 || w_cols <= 0 ||
        a_row_off < 0 || a_k_off < 0 || w_row_off < 0 || w_k_off < 0 || c_stride < 0)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "batched gemm: bad argument");
    if (lda % 8 || ldw % 8 || ldc % 8 || N % 8 || K % 8 || c_stride % 8 || a_cols > lda || w_cols > ldw || ldc < N || a_rows > INT32_MAX ||
        w_rows > INT32_MAX)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "batched gemm: ld / N / K / c_stride multiples of 8, extents inside the leading dimensions, ldc >= N");
    if (!aligned(A, 16) || !aligned(W, 16) || !aligned(C, 16)) return fail(nullptr, VQA_ERR_INVALID_ARG, "batched gemm: A / W / C 16-byte aligned");
    const long long last = nb - 1;
    if (last * a_row_off >= a_rows || last * w_row_off >= w_rows || last * a_k_off + K > a_cols || last * w_k_off + K > w_cols)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "batched gemm: every batch's first A / W row and its K columns must lie inside the extents");
    if (!batched_k_tail_ok(K, a_cols, w_cols))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "batched gemm: with K % 64 != 0, a_cols or w_cols must equal K");
    if (!gemm_variant_known(variant)) return fail(nullptr, VQA_ERR_INVALID_ARG, "batched gemm: unknown tile variant");
    Gemm g = abi_gemm(A, lda, W, ldw, (int)w_rows, C, ldc, M, N, K);
    g.batched(BatchSpec{nb, a_row_off, a_k_off, w_row_off, w_k_off, c_stride, a_rows, a_cols, w_rows, w_cols}, variant);
    return glue_launch(stream, [&](Forward& f) { return f.gemm(g); });
}

// One decoder layer's cross-attention as vqa_clipt5_score runs it: mode 0 the absorbed sequence (the encoder transpose, then
// clipt5_absorbed_cross_attention), mode 1 the reference association (clipt5_reference_cross_attention).
extern "C" int vqa_op_t5_cross_attention(const void* q, const void* x, const int32_t* seq_lens, const void* wkT, const void* wkv, void* out,
                                         int32_t B, int32_t T, int32_t S, int32_t H, int32_t d_model, int32_t mode, int32_t round_scores,
                                         void* workspace, size_t workspace_bytes, size_t* workspace_needed, void* stream) {
    if (!q || !x || !seq_lens || !wkv || !out || (mode == 0 && !wkT)) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 cross attention: null pointer");
    if (B <= 0 || T <= 0 || S <= 0 || H <= 0 || d_model <= 0 || d_model % 8 || (mode != 0 && mode != 1))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 cross attention: bad size (d_model a multiple of 8) or mode (0 or 1)");
    if (mode == 1 && T > 8) return fail(nullptr, VQA_ERR_UNSUPPORTED, "t5 cross attention: the reference association takes T <= 8");
    if (!aligned(q, 16) || !aligned(x, 16) || !aligned(wkT, 16) || !aligned(wkv, 16) || !aligned(out, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 cross attention: q / x / weights / out must be 16-byte aligned");
    const int inner = H * 64;
    Plan pl;
    CrossAttnBuffers xb{};
    size_t kv = 0;
    if (mode == 0) xb = take_cross_attn_buffers(pl, B, T, S, H, d_model);
    else kv = pl.take((size_t)B * S * 2 * inner * 2);
    if (workspace_needed) *workspace_needed = pl.off;
    if (!workspace || workspace_bytes < pl.off) return fail(nullptr, VQA_ERR_WORKSPACE, "t5 cross attention: workspace too small");
    if (!aligned(workspace, 256)) return fail(nullptr, VQA_ERR_INVALID_ARG, "t5 cross attention: workspace must be 256-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        if (mode == 1)
            return clipt5_reference_cross_attention(f, (const bf16*)q, (const bf16*)x, (const bf16*)wkv, f.at(kv), (bf16*)out, seq_lens, B, T, S, H,
                                                    d_model, round_scores);
        TRY(clipt5_transpose_encoder(f, (const bf16*)x, f.at(xb.xt), B, S, d_model));
        return clipt5_absorbed_cross_attention(f, AbsorbedCrossAttn{(const bf16*)q, (const bf16*)x, f.at(xb.xt), seq_lens, (const bf16*)wkT,
                                                                    (const bf16*)wkv + (size_t)inner * d_model, f.at(xb.qt), f.at(xb.csc),
                                                                    f.at(xb.ctx), (bf16*)out, B, T, S, H, d_model});
    }, workspace);
}

// LayerNorm of the CLIP tower's fp32 residual stream: x fp32 [rows, D] -> y bf16 [rows, D].
extern "C" int vqa_op_layernorm_f32(const float* x, const void* gamma, const void* beta, void* y, int32_t rows, int32_t D, float eps, void* stream) {
    if (!x || !gamma || !beta || !y || rows <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "fp32 layernorm: bad argument");
    if (D != 256 && D != 512 && D != 768 && D != 1024) return fail(nullptr, VQA_ERR_UNSUPPORTED, "fp32 layernorm: D must be 256, 512, 768 or 1024");
    if (!aligned(x, 16) || !aligned(gamma, 16) || !aligned(beta, 16) || !aligned(y, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "fp32 layernorm: pointers must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) { return f.layernorm_f32(x, (const bf16*)gamma, (const bf16*)beta, (bf16*)y, rows, D, eps); });
}

extern "C" int vqa_op_clip_embed_ln(const void* patch, const void* cls, const void* pos, const void* gamma, const void* beta, float* y,
                                    int32_t n_images, int32_t P, int32_t D, float eps, void* stream) {
    if (!patch || !cls || !pos || !gamma || !beta || !y || n_images <= 0 || P <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "clip embed: bad argument");
    if (D != 256 && D != 1024) return fail(nullptr, VQA_ERR_UNSUPPORTED, "clip embed: D must be 256 or 1024");
    if (!aligned(patch, 16) || !aligned(cls, 16) || !aligned(pos, 16) || !aligned(gamma, 16) || !aligned(beta, 16) || !aligned(y, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "clip embed: pointers must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        return clipt5_embed_ln(f, (const bf16*)patch, (const bf16*)cls, (const bf16*)pos, (const bf16*)gamma, (const bf16*)beta, y, n_images, P, D,
                               eps);
    });
}

extern "C" int vqa_op_patchify(const void* pixels, int32_t pixel_dtype, int32_t n_images, int32_t image_size, int32_t patch, int32_t kpad, void* out,
                               void* stream) {
    if (!pixels || !out) return fail(nullptr, VQA_ERR_INVALID_ARG, "patchify: null pointer");
    if (pixel_dtype != VQA_DTYPE_F32 && pixel_dtype != VQA_DTYPE_BF16) return fail(nullptr, VQA_ERR_INVALID_ARG, "patchify: pixels fp32 or bf16");
    if (n_images <= 0 || patch <= 0 || image_size < patch || kpad % 8 || kpad < 3 * patch * patch)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "patchify: bad size (patch <= image_size, kpad a multiple of 8 and >= 3 * patch^2)");
    if ((long long)n_images * (image_size / patch) * (image_size / patch) > INT32_MAX)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "patchify: too many patch rows");
    if (!aligned(pixels, pixel_dtype == VQA_DTYPE_F32 ? 4 : 2) || !aligned(out, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "patchify: pixels aligned to their element size, out 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        return clipt5_patchify(f, pixels, pixel_dtype, (bf16*)out, n_images, image_size, patch, kpad);
    });
}

extern "C" int vqa_op_splice_embed(const int32_t* ids, const int32_t* text_lens, const int32_t* image_index, const void* shared_emb, const void* feats,
                                   int32_t ldf, int32_t feat_row_offset, int32_t feat_rows_per_image, void* out, int32_t* seq_lens, int32_t B, int32_t L,
                                   int32_t P, int32_t D, int32_t image_token, void* stream) {
    if (!ids || !text_lens || !shared_emb || !feats || !out || !seq_lens) return fail(nullptr, VQA_ERR_INVALID_ARG, "splice: null pointer");
    if (B <= 0 || L <= 0 || P <= 0 || D <= 0 || D % 8 || ldf % 8 || ldf < D || feat_row_offset < 0 ||
        (long long)feat_row_offset + P > feat_rows_per_image || (long long)B * (L - 1 + P) > INT32_MAX)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "splice: bad size (D, ldf multiples of 8, ldf >= D, the P feature rows inside each image's block)");
    if (!aligned(ids, 4) || !aligned(text_lens, 4) || !aligned(image_index, 4) || !aligned(seq_lens, 4) || !aligned(shared_emb, 16) ||
        !aligned(feats, 16) || !aligned(out, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "splice: int32 arrays 4-byte aligned, embeddings / features / out 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        return clipt5_splice(f, ids, text_lens, image_index, (const bf16*)shared_emb, (const bf16*)feats, ldf, feat_row_offset, feat_rows_per_image,
                             (bf16*)out, seq_lens, B, L, P, D, image_token);
    });
}

extern "C" int vqa_op_decoder_embed(const int32_t* labels, const void* shared_emb, void* out, int32_t B, int32_t T, int32_t D, int32_t start_id,
                                    int32_t pad_id, void* stream) {
    if (!shared_emb || !out || (!labels && T != 1)) return fail(nullptr, VQA_ERR_INVALID_ARG, "decoder embed: null pointer (labels NULL needs T = 1)");
    if (B <= 0 || T <= 0 || D <= 0 || D % 8 || start_id < 0 || pad_id < 0 || (long long)B * T > INT32_MAX)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "decoder embed: bad size (D a multiple of 8, start / pad ids >= 0)");
    if (!aligned(labels, 4) || !aligned(shared_emb, 16) || !aligned(out, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "decoder embed: labels 4-byte aligned, embeddings / out 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) { return clipt5_decoder_embed(f, labels, (const bf16*)shared_emb, (bf16*)out, B, T, D, start_id, pad_id); });
}

extern "C" int vqa_op_t5_bias_table(const void* rel_emb, const int32_t* bucket_lut, int32_t max_distance, float* table, int32_t H, int32_t S,
                                    void* stream) {
    if (!rel_emb || !bucket_lut || !table) return fail(nullptr, VQA_ERR_INVALID_ARG, "bias table: null pointer");
    if (H <= 0 || S <= 0 || max_distance <= 0 || (long long)H * (2 * (long long)S - 1) > INT32_MAX)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "bias table: bad size");
    if (!aligned(rel_emb, 2) || !aligned(bucket_lut, 4) || !aligned(table, 4))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "bias table: rel_emb 2-byte, lut / table 4-byte aligned");
    return glue_launch(stream, [&](Forward& f) { return clipt5_bias_table(f, (const bf16*)rel_emb, bucket_lut, max_distance, table, H, S); });
}

extern "C" int vqa_op_lmhead_score(const void* Hs, int32_t ldh, const void* W, int32_t ldw, int32_t B, int32_t T, int32_t N, int32_t K,
                                   const int32_t* labels, float* scores, float* logprobs, float* scratch, size_t scratch_bytes, size_t* scratch_needed,
                                   void* stream) {
    if (!Hs || !W || !labels || !scores) return fail(nullptr, VQA_ERR_INVALID_ARG, "lmhead score: null pointer");
    if (B <= 0 || T <= 0 || N <= 0 || K <= 0 || K % 8 || ldh % 8 || ldw % 8 || ldh < K || ldw < K || (long long)B * T > INT32_MAX)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "lmhead score: bad size (K, ldh, ldw multiples of 8, ldh / ldw >= K)");
    if (!aligned(Hs, 16) || !aligned(W, 16) || !aligned(labels, 4) || !aligned(scores, 4) || !aligned(logprobs, 4))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "lmhead score: H / W 16-byte aligned, labels / scores / logprobs 4-byte aligned");
    const int M = B * T;
    const size_t need = lmhead_scratch_floats(M, N);
    if (scratch_needed) *scratch_needed = need * sizeof(float);
    if (!scratch || !aligned(scratch, 4) || scratch_bytes < need * sizeof(float))
        return fail(nullptr, VQA_ERR_WORKSPACE, "lmhead score: scratch smaller than lmhead_scratch_floats(B * T, N) floats");
    const size_t parts = (size_t)M * LMHEAD_PARTS * ((N + LMHEAD_BN - 1) / LMHEAD_BN);
    return glue_launch(stream, [&](Forward& f) {
        return lmhead_score(f, abi_gemm(Hs, ldh, W, ldw, N, nullptr, 0, M, N, K), labels, scratch, scratch + parts, scratch + 2 * parts, scores,
                            logprobs, B, T);
    });
}

extern "C" int vqa_op_row_ssq(const void* x, float* ssq, int32_t rows, int32_t D, int32_t stride, void* stream) {
    if (!x || !ssq) return fail(nullptr, VQA_ERR_INVALID_ARG, "row ssq: null pointer");
    if (rows <= 0 || D <= 0 || D % 8 || stride <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "row ssq: bad size (D a multiple of 8)");
    if (!aligned(x, 16) || !aligned(ssq, 4)) return fail(nullptr, VQA_ERR_INVALID_ARG, "row ssq: x 16-byte, ssq 4-byte aligned");
    return glue_launch(stream, [&](Forward& f) { return clipt5_row_ssq(f, (const bf16*)x, ssq, rows, D, stride); });
}

// ------------------------------------------------------------------------------------------------ kernel-level ABI: the Qwen2.5-VL scoring path

// rope_table_kernel into the caller's tables, then rope_inplace_kernel on n_heads heads of x; text_mode: bf16 table and bf16 products.
extern "C" int vqa_op_qwen_rope(const int32_t* positions, int32_t rows, const int32_t* axis_of_dim, const float* inv_freq, int32_t half, float* cos_t,
                                float* sin_t, void* x, int32_t ld, int32_t col0, int32_t n_heads, int32_t head_stride, int32_t head_dim,
                                int32_t text_mode, void* stream) {
    if (!positions || !axis_of_dim || !inv_freq || !cos_t || !sin_t || !x) return fail(nullptr, VQA_ERR_INVALID_ARG, "qwen rope: null pointer");
    if (rows <= 0 || n_heads <= 0 || head_dim <= 0 || head_dim % 16 || head_dim > head_stride || half * 2 != head_dim)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "qwen rope: bad size (head_dim a multiple of 16, <= head_stride, == 2 * half)");
    if (ld % 8 || col0 % 8 || head_stride % 8 || col0 < 0 || (long long)col0 + (long long)(n_heads - 1) * head_stride + head_dim > ld)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "qwen rope: ld, col0, head_stride multiples of 8, heads inside ld");
    if (!aligned(x, 16) || !aligned(cos_t, 16) || !aligned(sin_t, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "qwen rope: x and the tables must be 16-byte aligned");
    const int round = text_mode != 0 ? 1 : 0;
    return glue_launch(stream, [&](Forward& f) {
        TRY(qwen_rope_table(f, "rope table", positions, rows, axis_of_dim, inv_freq, half, cos_t, sin_t, round));
        return qwen_rope(f, "rope", (bf16*)x, ld, col0, n_heads, head_stride, head_dim, cos_t, sin_t, rows, round);
    });
}

extern "C" int vqa_op_gather_rows(const void* src, void* dst, const int32_t* index, int32_t rows, int32_t group, int32_t D, void* stream) {
    if (!src || !dst || !index) return fail(nullptr, VQA_ERR_INVALID_ARG, "gather rows: null pointer");
    if (rows <= 0 || group <= 0 || rows % group || D <= 0 || D % 8)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "gather rows: bad size (rows a multiple of group, D a multiple of 8)");
    if (!aligned(src, 16) || !aligned(dst, 16)) return fail(nullptr, VQA_ERR_INVALID_ARG, "gather rows: src / dst must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) { return qwen_gather_rows(f, "gather rows", (const bf16*)src, (bf16*)dst, index, rows, group, D); });
}

extern "C" int vqa_op_qwen_embed(const int32_t* ids, const int32_t* feat_index, const int32_t* seq_lens, const void* embed, const void* feats, void* out,
                                 int32_t rows, int32_t S, int32_t D, void* stream) {
    if (!ids || !feat_index || !seq_lens || !embed || !feats || !out) return fail(nullptr, VQA_ERR_INVALID_ARG, "qwen embed: null pointer");
    if (rows <= 0 || S <= 0 || rows % S || D <= 0 || D % 8)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "qwen embed: bad size (rows a multiple of S, D a multiple of 8)");
    if (!aligned(embed, 16) || !aligned(feats, 16) || !aligned(out, 16))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "qwen embed: embed / feats / out must be 16-byte aligned");
    return glue_launch(stream, [&](Forward& f) {
        return qwen_embed(f, ids, feat_index, seq_lens, (const bf16*)embed, (const bf16*)feats, (bf16*)out, rows, S, D);
    });
}

// The repetition-penalty bitmap of padded (cu_seqlens NULL) or packed rows, OR-ed into the caller's bitmap.
extern "C" int vqa_op_token_bitmap(const int32_t* ids, const int32_t* seq_lens, int32_t B, int32_t S, const int32_t* cu_seqlens, const int32_t* kv_prefix,
                                   const int32_t* pair_seq, int32_t max_prompt_len, int32_t vocab, uint32_t* bitmap, void* stream) {
    if (!ids || !bitmap) return fail(nullptr, VQA_ERR_INVALID_ARG, "token bitmap: null pointer");
    if (B <= 0 || vocab <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "token bitmap: bad size");
    if (!aligned(bitmap, 4)) return fail(nullptr, VQA_ERR_INVALID_ARG, "token bitmap: bitmap must be 4-byte aligned");
    if (cu_seqlens) {
        if (!pair_seq || max_prompt_len <= 0)
            return fail(nullptr, VQA_ERR_INVALID_ARG, "token bitmap: packed rows need pair_seq and max_prompt_len >= 1");
        return glue_launch(stream, [&](Forward& f) {
            return qwen_token_bitmap_packed(f, ids, cu_seqlens, kv_prefix, pair_seq, max_prompt_len, B, vocab, bitmap);
        });
    }
    if (!seq_lens || S <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "token bitmap: padded rows need seq_lens and S >= 1");
    return glue_launch(stream, [&](Forward& f) { return qwen_token_bitmap(f, ids, seq_lens, B, S, vocab, bitmap); });
}

// The trace output of vqa_qwen25vl_topk on caller logits [B, ldl].
extern "C" int vqa_op_topk_softmax(const void* logits, int64_t ldl, int32_t B, int32_t V, float temperature, const uint32_t* pen_bitmap,
                                   float repetition_penalty, int32_t K, int32_t* out_ids, float* out_probs, void* stream) {
    if (!logits || !out_ids || !out_probs) return fail(nullptr, VQA_ERR_INVALID_ARG, "top-k softmax: null pointer");
    if (B <= 0 || V <= 0 || ldl < V || K < 1 || K > TOPK_MAX) return fail(nullptr, VQA_ERR_INVALID_ARG, "top-k softmax: bad size (ldl >= V, 1 <= K <= 8)");
    if (!(temperature > 0.f) || !(repetition_penalty > 0.f))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "top-k softmax: temperature and repetition penalty must be > 0");
    if (!aligned(logits, 2) || !aligned(pen_bitmap, 4)) return fail(nullptr, VQA_ERR_INVALID_ARG, "top-k softmax: misaligned logits / bitmap");
    return glue_launch(stream, [&](Forward& f) {
        return qwen_topk_softmax(f, (const bf16*)logits, ldl, B, V, temperature, pen_bitmap, repetition_penalty, K, out_ids, out_probs);
    });
}

// ---------------------------------------------------------------------------------------------- image pre-processing (SURVEY 8(f)2)
extern "C" size_t vqa_clip_preprocess_workspace_bytes(const int32_t* heights, const int32_t* widths, int32_t n_images,
                                                      int32_t out_size, int32_t pad_to_square) {
    if (!heights || !widths || n_images <= 0 || out_size <= 0) return 0;
    PrePlan plan;
    std::vector<int64_t> off(n_images, 0);
    if (!pre_plan(heights, widths, off.data(), n_images, out_size, pad_to_square != 0, plan)) {
        fail(nullptr, VQA_ERR_INVALID_ARG, plan.error);
        return 0;
    }
    return plan.bytes();
}

template <int LAYOUT>
static int pre_launch(const PrePlan& plan, const void* src, int n_images, const uint8_t* background, const float* mean, const float* stdv,
                      PrePatchGeom geom, void* out, int32_t out_dtype, void* workspace, size_t workspace_bytes, void* host_staging,
                      cudaStream_t st) {
    if (workspace_bytes < plan.bytes()) return fail(nullptr, VQA_ERR_WORKSPACE, "pre-processing workspace too small");
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    cudaError_t e;
    if (host_staging) {
        // caller-owned (pinned) staging: one truly asynchronous copy; the caller keeps the buffer untouched until the stream passes it
        uint8_t* hs = static_cast<uint8_t*>(host_staging);
        memcpy(hs, plan.images.data(), plan.images.size() * sizeof(PreImage));
        memcpy(hs + plan.images_bytes(), plan.tables.data(), plan.tables.size() * sizeof(int));
        e = cudaMemcpyAsync(ws, hs, plan.bytes(), cudaMemcpyHostToDevice, st);
    } else {
        // pageable host -> device: the runtime stages the bytes before returning, so the plan may die with the caller's frame
        e = cudaMemcpyAsync(ws, plan.images.data(), plan.images.size() * sizeof(PreImage), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(ws + plan.images_bytes(), plan.tables.data(), plan.tables.size() * sizeof(int), cudaMemcpyHostToDevice, st);
    }
    if (e != cudaSuccess) return fail(nullptr, VQA_ERR_CUDA, std::string("pre-processing table upload: ") + cudaGetErrorString(e));
    const PreImage* d_images = reinterpret_cast<const PreImage*>(ws);
    const int* d_tables = reinterpret_cast<const int*>(ws + plan.images_bytes());
    const uchar3 bg = make_uchar3(background[0], background[1], background[2]);
    const float3 mu = make_float3(mean[0], mean[1], mean[2]), sd = make_float3(stdv[0], stdv[1], stdv[2]);
    dim3 grid(plan.max_tiles, n_images);
    if (out_dtype == VQA_DTYPE_F32) {
        e = cudaFuncSetAttribute(image_preprocess_kernel<float, LAYOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PRE_MAX_SMEM);
        if (e == cudaSuccess)
            image_preprocess_kernel<float, LAYOUT><<<grid, PRE_THREADS, plan.smem, st>>>(static_cast<const uint8_t*>(src), d_images, d_tables, bg,
                                                                                        mu, sd, geom, static_cast<float*>(out));
    } else {
        e = cudaFuncSetAttribute(image_preprocess_kernel<bf16, LAYOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PRE_MAX_SMEM);
        if (e == cudaSuccess)
            image_preprocess_kernel<bf16, LAYOUT><<<grid, PRE_THREADS, plan.smem, st>>>(static_cast<const uint8_t*>(src), d_images, d_tables, bg,
                                                                                       mu, sd, geom, static_cast<bf16*>(out));
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, VQA_ERR_CUDA, std::string("pre-processing launch: ") + cudaGetErrorString(e));
    return VQA_OK;
}

extern "C" int vqa_clip_preprocess(const void* src, const int64_t* offsets, const int32_t* heights, const int32_t* widths,
                                   int32_t n_images, int32_t out_size, int32_t pad_to_square, const uint8_t* background,
                                   const float* mean, const float* stdv, void* out, int32_t out_dtype, void* workspace,
                                   size_t workspace_bytes, void* host_staging, void* stream) {
    if (!src || !offsets || !heights || !widths || !background || !mean || !stdv || !out || !workspace)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "null pointer");
    if (n_images <= 0 || out_size <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad size");
    if (out_dtype != VQA_DTYPE_F32 && out_dtype != VQA_DTYPE_BF16) return fail(nullptr, VQA_ERR_INVALID_ARG, "out_dtype must be f32 or bf16");
    PrePlan plan;
    if (!pre_plan(heights, widths, offsets, n_images, out_size, pad_to_square != 0, plan)) return fail(nullptr, VQA_ERR_INVALID_ARG, plan.error);
    return pre_launch<PRE_CHW>(plan, src, n_images, background, mean, stdv, PrePatchGeom{1, 1, 1}, out, out_dtype, workspace, workspace_bytes,
                               host_staging, reinterpret_cast<cudaStream_t>(stream));
}

static int qwen_video_args(const int32_t* n_frames, const int32_t* heights, const int32_t* widths, const int32_t* is_video, int32_t n_items,
                           int32_t patch, int32_t temporal_patch, int32_t merge, int64_t min_pixels, int64_t max_pixels, int64_t* frames) {
    if (!n_frames || !heights || !widths || !is_video || n_items <= 0 || patch <= 0 || merge <= 0 || temporal_patch <= 0 || min_pixels <= 0 ||
        max_pixels < min_pixels)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "bad argument");
    int64_t total = 0;
    for (int i = 0; i < n_items; ++i) total += n_frames[i] > 0 ? n_frames[i] : 0;
    if (total > 65535) return fail(nullptr, VQA_ERR_INVALID_ARG, "more than 65535 frames in one call");     // gridDim.y of the launch
    *frames = total;
    return VQA_OK;
}

extern "C" int vqa_qwen_preprocess_video_plan(const int32_t* n_frames, const int32_t* heights, const int32_t* widths, const int32_t* is_video,
                                              int32_t n_items, int32_t patch, int32_t temporal_patch, int32_t merge, int64_t min_pixels,
                                              int64_t max_pixels, int32_t* grid_thw, int64_t* total_patches, size_t* workspace_bytes) {
    int64_t frames = 0;
    if (int rc = qwen_video_args(n_frames, heights, widths, is_video, n_items, patch, temporal_patch, merge, min_pixels, max_pixels, &frames))
        return rc;
    PrePlan plan;
    std::vector<int64_t> off(frames, 0);
    long long rows = 0;
    if (!pre_plan_qwen_video(n_frames, heights, widths, is_video, off.data(), n_items, patch, merge, temporal_patch, min_pixels, max_pixels,
                             plan, grid_thw, &rows))
        return fail(nullptr, VQA_ERR_INVALID_ARG, plan.error);
    if (total_patches) *total_patches = rows;
    if (workspace_bytes) *workspace_bytes = plan.bytes();
    return VQA_OK;
}

extern "C" int vqa_qwen_preprocess_video(const void* src, const int64_t* frame_offsets, const int32_t* n_frames, const int32_t* heights,
                                         const int32_t* widths, const int32_t* is_video, int32_t n_items, int32_t patch, int32_t temporal_patch,
                                         int32_t merge, int64_t min_pixels, int64_t max_pixels, const float* mean, const float* stdv, void* out,
                                         int32_t out_dtype, void* workspace, size_t workspace_bytes, void* host_staging, void* stream) {
    if (!src || !frame_offsets || !mean || !stdv || !out || !workspace) return fail(nullptr, VQA_ERR_INVALID_ARG, "null pointer");
    int64_t frames = 0;
    if (int rc = qwen_video_args(n_frames, heights, widths, is_video, n_items, patch, temporal_patch, merge, min_pixels, max_pixels, &frames))
        return rc;
    if (out_dtype != VQA_DTYPE_F32 && out_dtype != VQA_DTYPE_BF16) return fail(nullptr, VQA_ERR_INVALID_ARG, "out_dtype must be f32 or bf16");
    PrePlan plan;
    if (!pre_plan_qwen_video(n_frames, heights, widths, is_video, frame_offsets, n_items, patch, merge, temporal_patch, min_pixels, max_pixels,
                             plan, nullptr, nullptr))
        return fail(nullptr, VQA_ERR_INVALID_ARG, plan.error);
    const uint8_t no_bg[3] = {0, 0, 0};
    return pre_launch<PRE_QWEN_PATCHES>(plan, src, (int)plan.images.size(), no_bg, mean, stdv, PrePatchGeom{patch, merge, temporal_patch}, out,
                                        out_dtype, workspace, workspace_bytes, host_staging, reinterpret_cast<cudaStream_t>(stream));
}

// Process-wide forced tile plan of image_preprocess_kernel (tests / tuning): tile_rows output rows, min(tile_cols, out_w) output columns
// and chunk_groups groups of 4 canvas rows per pass for every image; all zero = the planner's choice (pre_tables).
extern "C" int vqa_debug_set_preprocess_tiles(int32_t tile_rows, int32_t tile_cols, int32_t chunk_groups) {
    const bool automatic = tile_rows == 0 && tile_cols == 0 && chunk_groups == 0;
    if (!automatic && (tile_rows < 1 || tile_rows > 32 || tile_cols < 1 || chunk_groups < 1 || chunk_groups > PRE_RG))
        return fail(nullptr, VQA_ERR_INVALID_ARG, "preprocess tiles: tile_rows in [1, 32], tile_cols >= 1 and chunk_groups 1 or 2, or all zero");
    g_pre_tile_override = PreTileOverride{tile_rows, tile_cols, chunk_groups};
    return VQA_OK;
}

// Host-only: the launch geometry the planner gives each item of a vqa_clip_preprocess (layout 0: heights / widths / n_items / out_size /
// pad_to_square) or vqa_qwen_preprocess_video call (layout 1: n_frames / is_video NULL = still images). geometry [n_items][5] =
// (tile_rows, tile_cols, col_tiles, chunk_groups, band_groups); the frames of a stack share their item's geometry.
extern "C" int vqa_debug_preprocess_geometry(int32_t layout, const int32_t* n_frames, const int32_t* heights, const int32_t* widths,
                                             const int32_t* is_video, int32_t n_items, int32_t out_size, int32_t pad_to_square, int32_t patch,
                                             int32_t temporal_patch, int32_t merge, int64_t min_pixels, int64_t max_pixels, int32_t* geometry) {
    if (!heights || !widths || !geometry || n_items <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad argument");
    PrePlan plan;
    std::vector<int> first(n_items);                       // index in plan.images of each item's first frame
    if (layout == PRE_CHW) {
        if (out_size <= 0) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad size");
        std::vector<int64_t> off(n_items, 0);
        if (!pre_plan(heights, widths, off.data(), n_items, out_size, pad_to_square != 0, plan)) return fail(nullptr, VQA_ERR_INVALID_ARG, plan.error);
        for (int i = 0; i < n_items; ++i) first[i] = i;
    } else if (layout == PRE_QWEN_PATCHES) {
        const std::vector<int32_t> one(n_items, 1), still(n_items, 0);
        if (!n_frames) n_frames = one.data();
        if (!is_video) is_video = still.data();
        int64_t frames = 0;
        if (int rc = qwen_video_args(n_frames, heights, widths, is_video, n_items, patch, temporal_patch, merge, min_pixels, max_pixels, &frames))
            return rc;
        std::vector<int64_t> off(frames, 0);
        if (!pre_plan_qwen_video(n_frames, heights, widths, is_video, off.data(), n_items, patch, merge, temporal_patch, min_pixels, max_pixels,
                                 plan, nullptr, nullptr))
            return fail(nullptr, VQA_ERR_INVALID_ARG, plan.error);
        for (int i = 0, f = 0; i < n_items; f += n_frames[i++]) first[i] = f;
    } else {
        return fail(nullptr, VQA_ERR_INVALID_ARG, "layout must be 0 (CLIP, channel planes) or 1 (Qwen patch rows)");
    }
    for (int i = 0; i < n_items; ++i) {
        const PreImage& im = plan.images[first[i]];
        const int32_t g[5] = {im.tile_rows, im.tile_cols, im.col_tiles, im.chunk_groups, im.band_groups};
        for (int j = 0; j < 5; ++j) geometry[5 * i + j] = g[j];
    }
    return VQA_OK;
}

static int qwen_video_aa_args(int32_t in_h, int32_t in_w, int32_t out_h, int32_t out_w, const int32_t* first_h, int32_t htaps,
                              const int32_t* first_v, int32_t vtaps, int32_t patch, int32_t temporal_patch, int32_t merge, int32_t total_frames,
                              PreAAGeom& g) {
    if (!first_h || !first_v || patch <= 0 || merge <= 0 || temporal_patch <= 0 || total_frames <= 0)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "bad argument");
    std::string error;
    if (!pre_plan_aa(in_h, in_w, out_h, out_w, first_h, htaps, first_v, vtaps, patch, merge, g, error))
        return fail(nullptr, VQA_ERR_INVALID_ARG, error);
    g.total_frames = total_frames;
    return VQA_OK;
}

static size_t qwen_video_aa_table_bytes(const PreAAGeom& g) {
    return ((size_t)g.out_w + g.out_h) * sizeof(int32_t) + ((size_t)g.out_w * g.htaps + (size_t)g.out_h * g.vtaps) * sizeof(float);
}

extern "C" int vqa_qwen_preprocess_video_aa_plan(int32_t in_h, int32_t in_w, int32_t out_h, int32_t out_w, const int32_t* first_h,
                                                 int32_t htaps, const int32_t* first_v, int32_t vtaps, int32_t patch, int32_t temporal_patch,
                                                 int32_t merge, int32_t total_frames, int64_t* total_patches, size_t* workspace_bytes) {
    PreAAGeom g;
    if (int rc = qwen_video_aa_args(in_h, in_w, out_h, out_w, first_h, htaps, first_v, vtaps, patch, temporal_patch, merge, total_frames, g))
        return rc;
    if (total_patches)
        *total_patches = (int64_t)((total_frames + temporal_patch - 1) / temporal_patch) * (out_h / patch) * (out_w / patch);
    if (workspace_bytes) *workspace_bytes = qwen_video_aa_table_bytes(g);
    return VQA_OK;
}

// Process-wide forced output rows per CTA of video_resize_aa_kernel (tests): 1 ... 32, 0 = the planner's choice (pre_plan_aa).
extern "C" int vqa_debug_set_preprocess_aa_rows(int32_t tile_rows) {
    if (tile_rows < 0 || tile_rows > 32) return fail(nullptr, VQA_ERR_INVALID_ARG, "preprocess aa rows: tile_rows in [1, 32], or 0");
    g_pre_aa_rows_override = tile_rows;
    return VQA_OK;
}

// Host-only: the launch geometry vqa_qwen_preprocess_video_aa would use for these windows, geometry[3] = (tile_rows, band_rows, tiles_x).
extern "C" int vqa_debug_preprocess_aa_geometry(int32_t in_h, int32_t in_w, int32_t out_h, int32_t out_w, const int32_t* first_h,
                                                int32_t htaps, const int32_t* first_v, int32_t vtaps, int32_t patch, int32_t merge,
                                                int32_t* geometry) {
    if (!geometry) return fail(nullptr, VQA_ERR_INVALID_ARG, "bad argument");
    PreAAGeom g;
    if (int rc = qwen_video_aa_args(in_h, in_w, out_h, out_w, first_h, htaps, first_v, vtaps, patch, 1, merge, 1, g)) return rc;
    geometry[0] = g.tile_rows; geometry[1] = g.band_rows; geometry[2] = g.tiles_x;
    return VQA_OK;
}

extern "C" int vqa_qwen_preprocess_video_aa(const void* src, int32_t n_frames, int32_t frame0, int32_t total_frames, int32_t in_h, int32_t in_w,
                                            int32_t out_h, int32_t out_w, const int32_t* first_h, const float* weights_h, int32_t htaps,
                                            const int32_t* first_v, const float* weights_v, int32_t vtaps, int32_t patch, int32_t temporal_patch,
                                            int32_t merge, const float* mean, const float* stdv, void* out, int32_t out_dtype, void* workspace,
                                            size_t workspace_bytes, void* host_staging, void* stream) {
    if (!src || !weights_h || !weights_v || !mean || !stdv || !out || !workspace) return fail(nullptr, VQA_ERR_INVALID_ARG, "null pointer");
    PreAAGeom g;
    if (int rc = qwen_video_aa_args(in_h, in_w, out_h, out_w, first_h, htaps, first_v, vtaps, patch, temporal_patch, merge, total_frames, g))
        return rc;
    if (n_frames <= 0 || n_frames > 65535 || frame0 < 0 || frame0 + n_frames > total_frames)
        return fail(nullptr, VQA_ERR_INVALID_ARG, "frames [frame0, frame0 + n_frames) must lie in the video, at most 65535 per call");
    if (out_dtype != VQA_DTYPE_F32 && out_dtype != VQA_DTYPE_BF16) return fail(nullptr, VQA_ERR_INVALID_ARG, "out_dtype must be f32 or bf16");
    g.frame0 = frame0;
    const size_t nb[4] = {(size_t)out_w * sizeof(int32_t), (size_t)out_h * sizeof(int32_t), (size_t)out_w * htaps * sizeof(float),
                          (size_t)out_h * vtaps * sizeof(float)};
    const void* parts[4] = {first_h, first_v, weights_h, weights_v};
    const size_t bytes = qwen_video_aa_table_bytes(g);
    if (workspace_bytes < bytes) return fail(nullptr, VQA_ERR_WORKSPACE, "pre-processing workspace too small");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    cudaError_t e = cudaSuccess;
    if (host_staging) {
        // caller-owned (pinned) staging: one truly asynchronous copy; the caller keeps the buffer untouched until the stream passes it
        uint8_t* hs = static_cast<uint8_t*>(host_staging);
        for (size_t i = 0, o = 0; i < 4; o += nb[i], ++i) memcpy(hs + o, parts[i], nb[i]);
        e = cudaMemcpyAsync(ws, hs, bytes, cudaMemcpyHostToDevice, st);
    } else {
        for (size_t i = 0, o = 0; i < 4 && e == cudaSuccess; o += nb[i], ++i) e = cudaMemcpyAsync(ws + o, parts[i], nb[i], cudaMemcpyHostToDevice, st);
    }
    if (e != cudaSuccess) return fail(nullptr, VQA_ERR_CUDA, std::string("pre-processing table upload: ") + cudaGetErrorString(e));
    const float3 mu = make_float3(mean[0], mean[1], mean[2]), sd = make_float3(stdv[0], stdv[1], stdv[2]);
    const PrePatchGeom geom{patch, merge, temporal_patch};
    const dim3 grid(g.tiles_x * ((out_h + g.tile_rows - 1) / g.tile_rows), n_frames);
    const size_t smem = pre_aa_smem_bytes(g.band_rows);
    const uint8_t* s8 = static_cast<const uint8_t*>(src);
    const int* tab = reinterpret_cast<const int*>(ws);
    if (out_dtype == VQA_DTYPE_F32) {
        e = cudaFuncSetAttribute(video_resize_aa_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, PRE_AA_MAX_SMEM);
        if (e == cudaSuccess) video_resize_aa_kernel<float><<<grid, PRE_THREADS, smem, st>>>(s8, tab, g, geom, mu, sd, static_cast<float*>(out));
    } else {
        e = cudaFuncSetAttribute(video_resize_aa_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, PRE_AA_MAX_SMEM);
        if (e == cudaSuccess) video_resize_aa_kernel<bf16><<<grid, PRE_THREADS, smem, st>>>(s8, tab, g, geom, mu, sd, static_cast<bf16*>(out));
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, VQA_ERR_CUDA, std::string("pre-processing launch: ") + cudaGetErrorString(e));
    return VQA_OK;
}

// Host-only: the fixed-point tap table of one resize axis, exactly as vqa_clip_preprocess builds it (for CPU tests of the host logic).
// bounds: [count][2] (first source index, taps used), kk: [count][ksize] with ksize = return value (call with kk = NULL to size it).
extern "C" int32_t vqa_resample_table(int32_t in_size, int32_t out_size, int32_t first, int32_t count, int32_t* bounds, int32_t* kk) {
    if (in_size <= 0 || out_size <= 0 || first < 0 || count <= 0 || first + count > out_size) {
        fail(nullptr, VQA_ERR_INVALID_ARG, "bad resample table request");
        return 0;
    }
    std::vector<int> tab;
    const int ksize = pre_build_table(in_size, out_size, first, count, tab);
    if (bounds) memcpy(bounds, tab.data(), (size_t)count * 2 * sizeof(int));
    if (kk) memcpy(kk, tab.data() + (size_t)count * 2, (size_t)count * ksize * sizeof(int));
    return ksize;
}

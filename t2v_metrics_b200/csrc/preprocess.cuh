// CLIP image pre-processing on the device (SURVEY 8(f)2): expand2square + bicubic resize + centre crop + rescale + normalise.
//
// What it replaces: t2v_metrics/models/vqascore_models/mm_utils.py:128-139 (expand2square) followed by the CLIP image processor
// of the v3.0 wrapper (resize shortest edge to S with PIL BICUBIC, centre crop SxS, /255, (x - mean) / std), i.e.
// oracle/clipt5_oracle.py:clip_preprocess. The resize is Pillow's (third-party dependency of the reference, not vendored;
// installed 12.2.0, src/libImaging/Resample.c): a separable convolution with per-output-pixel windows, coefficients normalised in
// double and quantised to 22-bit fixed point, the horizontal pass first, its result ROUNDED TO uint8, then the vertical pass. The
// coefficient tables are built on the host in double exactly as Pillow builds them (so the integers are identical), the two integer
// passes run here, and the result is bit-identical to PIL for every pixel.
//
// One CTA = one image x one tile of `tile_rows` output rows by `tile_cols` output columns. An image whose filter windows fit the
// shared-memory budget over its whole output width has one column tile; a wide canvas (frames concatenated side by side, then padded to
// a square) is split into column tiles too, and each CTA stages only the canvas columns its own columns' windows touch. The canvas rows
// the tile needs are staged up to 8 at a time into shared memory as three byte PLANES packed four pixels to a word (padding colour
// filled in, so the passes need no bounds checks). Each 22-bit tap is
// split on the host into three byte digits (k = d0 + 256 d1 + 65536 d2, d2 signed) and laid out in words aligned to the same groups of
// four pixels, so one `dp4a` multiplies four pixels by four tap digits: 3 dp4a per 4 taps per channel, exact in int32
// (acc0 + (acc1 << 8) + (acc2 << 16) is the same integer Pillow accumulates). The horizontal pass writes its uint8 result four ROWS
// to a word, which is the packing the vertical pass needs; a 768-entry table does /255, -mean, /std in exact fp32. The source is read
// once from HBM (plus the band overlap, absorbed by L2), the output written once.
#pragma once
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>
#include "ptx.cuh"

namespace vqa {

constexpr int PRE_PRECISION_BITS = 32 - 8 - 2;      // Resample.c PRECISION_BITS
constexpr int PRE_THREADS = 256;
constexpr int PRE_XL = 128;                         // x lanes; PRE_THREADS / PRE_XL row groups of 4 canvas rows each
constexpr int PRE_RG = PRE_THREADS / PRE_XL;
constexpr int PRE_MAX_SMEM = 200 * 1024;
constexpr int PRE_MAX_CANVAS = 65500;               // largest padded CLIP canvas side (libjpeg's largest dimension)

struct PreImage {            // one per image, lives in the workspace (device) and is built on the host
    long long src_off;       // byte offset of the HWC uint8 RGB image inside `src`
    int h, w;                // stored image
    int paste_x, paste_y;    // where the stored image sits on the (virtual) square canvas; 0 when not padded
    int canvas_h, canvas_w;  // canvas the resize reads (= max(h, w) squared when padded, else h x w)
    int htab, vtab;          // int offsets of the packed tap tables inside the workspace (layout: see pre_pack_table)
    int hnp, vnp;            // words of 4 taps per output pixel (horizontal / vertical)
    int tile_rows;           // output rows per CTA
    int tile_cols, col_tiles;  // output columns per CTA (= out_w when one tile spans the width) and column tiles per row tile
    int band_groups;         // groups of 4 canvas rows the band buffer holds
    int out_h, out_w;        // output window (after the crop) of this image
    long long out_off;       // element offset of this image's output inside `out`
    int chunk_groups;        // groups of 4 canvas rows staged per pass (1 or 2)
    int t0, nt;              // PRE_QWEN_PATCHES: temporal slots [t0, t0 + nt) of its patch rows this frame fills
};

enum PreLayout { PRE_CHW = 0, PRE_QWEN_PATCHES = 1 };
struct PrePatchGeom { int patch, merge, temporal; };     // PRE_QWEN_PATCHES only

// ---------------------------------------------------------------------------------------------- host: Pillow's coefficient tables
inline double pre_bicubic(double x) {                 // Resample.c bicubic_filter, a = -0.5
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}

// precompute_coeffs + normalize_coeffs_8bpc for output pixels [first, first + count) of an in_size -> out_size resize over the whole
// axis (box = [0, in_size)). Appends bounds (xmin, n) pairs then count * ksize fixed-point taps to `tab`; returns ksize.
inline int pre_build_table(int in_size, int out_size, int first, int count, std::vector<int>& tab) {
    const float in0 = 0.f, in1 = (float)in_size;
    double scale = (double)(in1 - in0) / out_size;
    double filterscale = scale;
    if (filterscale < 1.0) filterscale = 1.0;
    const double support = 2.0 * filterscale;          // BICUBIC.support = 2.0
    const int ksize = (int)std::ceil(support) * 2 + 1;
    const size_t base = tab.size();
    tab.resize(base + (size_t)count * 2 + (size_t)count * ksize, 0);
    int* bounds = tab.data() + base;
    int* kk = bounds + (size_t)count * 2;
    std::vector<double> k(ksize);
    for (int i = 0; i < count; ++i) {
        const int xx = first + i;
        const double center = in0 + (xx + 0.5) * scale;
        double ww = 0.0;
        const double ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        for (int x = 0; x < xmax; ++x) {
            const double w = pre_bicubic((x + xmin - center + 0.5) * ss);
            k[x] = w;
            ww += w;
        }
        for (int x = 0; x < xmax; ++x)
            if (ww != 0.0) k[x] /= ww;
        for (int x = 0; x < ksize; ++x) {
            const double v = x < xmax ? k[x] : 0.0;
            kk[(size_t)i * ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << PRE_PRECISION_BITS)) : (int)(0.5 + v * (1 << PRE_PRECISION_BITS));
        }
        bounds[2 * i] = xmin;
        bounds[2 * i + 1] = xmax;
    }
    return ksize;
}

// Tap words for the dp4a passes, from one axis' (bounds, kk) table of `count` outputs with `ksize` taps each. Appends to `tab`:
//   start4[count]          group (absolute position / 4) of the first tap word of each output
//   last4[count]           group of the last REAL tap
//   words[count][np][3]    byte digits d0 | d1 | d2 of the four taps of each word (zero where the window has no tap)
// and returns np = the largest number of words any output needs.
inline int pre_pack_table(const int* bounds, const int* kk, int count, int ksize, std::vector<int>& tab) {
    int np = 1;
    for (int i = 0; i < count; ++i) {
        const int x0 = bounds[2 * i], n = bounds[2 * i + 1];
        const int words = n > 0 ? (x0 + n - 1) / 4 - x0 / 4 + 1 : 1;
        if (words > np) np = words;
    }
    const size_t base = tab.size();
    tab.resize(base + (size_t)count * 2 + (size_t)count * np * 3, 0);
    int* start4 = tab.data() + base;
    int* last4 = start4 + count;
    unsigned* words = reinterpret_cast<unsigned*>(last4 + count);
    for (int i = 0; i < count; ++i) {
        const int x0 = bounds[2 * i], n = bounds[2 * i + 1];
        start4[i] = x0 / 4;
        last4[i] = n > 0 ? (x0 + n - 1) / 4 : x0 / 4;
        for (int x = 0; x < n; ++x) {
            const int a = x0 + x, w = a / 4 - start4[i], b = a % 4;
            const int k = kk[(size_t)i * ksize + x];
            unsigned* q = words + ((size_t)i * np + w) * 3;
            q[0] |= (unsigned)(k & 0xff) << (8 * b);
            q[1] |= (unsigned)((k >> 8) & 0xff) << (8 * b);
            q[2] |= (unsigned)((k >> 16) & 0xff) << (8 * b);          // arithmetic shift: the signed top digit
        }
    }
    return np;
}

// ---------------------------------------------------------------------------------------------- device
__device__ __forceinline__ int pre_clip8(int v) {     // Resample.c clip8: table lookup of (v >> PRECISION_BITS) clamped to [0, 255]
    v >>= PRE_PRECISION_BITS;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}
__device__ __forceinline__ unsigned pre_dp4a_uu(unsigned a, unsigned b, unsigned c) {      // 4 x (u8 * u8) + c
    unsigned d;
    asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int pre_dp4a_us(unsigned a, unsigned b, int c) {                // 4 x (u8 * s8) + c
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
// the integer Pillow accumulates, rounded and clipped: sum(px * k) + 2^21 with k = d0 + 256 d1 + 65536 d2
__device__ __forceinline__ unsigned pre_finish(unsigned a0, unsigned a1, int a2) {
    const unsigned t = a0 + (a1 << 8) + ((unsigned)a2 << 16) + (1u << (PRE_PRECISION_BITS - 1));
    return (unsigned)pre_clip8((int)t);
}

// out = ((u8 / 255) - mean[c]) / std[c] in fp32 with IEEE division and no fma, as numpy / torch compute it on the host; lut[3][256]
__device__ __forceinline__ void pre_fill_lut(float* lut, float3 mean, float3 stdv) {
    for (int i = threadIdx.x; i < 768; i += PRE_THREADS) {
        const int c = i >> 8;
        const float mu = c == 0 ? mean.x : (c == 1 ? mean.y : mean.z), sd = c == 0 ? stdv.x : (c == 1 ? stdv.y : stdv.z);
        lut[i] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)(i & 255), 255.0f), mu), sd);
    }
}

// PRE_QWEN_PATCHES output of pixel (y, x) with channel values v: the Qwen2-VL processor's patch rows (image_processing_qwen2_vl.py:191-220),
// row ((by * gw/m + bx) * m + iy) * m + ix for the 14x14 patch at grid (by*m+iy, bx*m+ix), column (c * temporal + t) * ps*ps + py * ps + px,
// written to temporal slots t in [t0, t0 + nt). gwm = patches per row / merge.
template <typename OUT>
__device__ __forceinline__ void pre_store_patch(OUT* dst, PrePatchGeom geom, int gwm, int y, int x, const float* v, int t0, int nt) {
    const int ps = geom.patch, mg = geom.merge, pp = geom.patch * geom.patch;
    const int gy = y / ps, py = y - gy * ps, gx = x / ps, px_ = x - gx * ps;
    const size_t row = (((size_t)(gy / mg) * gwm + gx / mg) * mg + gy % mg) * mg + gx % mg;
    OUT* q = dst + row * (size_t)(3 * geom.temporal * pp) + py * ps + px_;
#pragma unroll
    for (int c = 0; c < 3; ++c)
        for (int t = t0; t < t0 + nt; ++t) {
            if constexpr (sizeof(OUT) == 4) q[(size_t)(c * geom.temporal + t) * pp] = v[c];
            else q[(size_t)(c * geom.temporal + t) * pp] = __float2bfloat16_rn(v[c]);
        }
}

// LAYOUT PRE_CHW: out[c][y][x] per image ([3, out_h, out_w]). PRE_QWEN_PATCHES: the Qwen2-VL processor's patch rows
// (image_processing_qwen2_vl.py:191-220): row ((by * gw/m + bx) * m + iy) * m + ix for the 14x14 patch at grid (by*m+iy, bx*m+ix),
// column (c * temporal + t) * ps*ps + py * ps + px, the frame written to temporal slots t in [t0, t0 + nt): every slot for a still
// image, its own slot for a video frame (video_processing_qwen2_vl.py:255-272), and the remaining slots for the last frame of a stack.
template <typename OUT, int LAYOUT>
__global__ void __launch_bounds__(PRE_THREADS, 3)
image_preprocess_kernel(const uint8_t* __restrict__ src, const PreImage* __restrict__ images, const int* __restrict__ tables,
                        uchar3 background, float3 mean, float3 stdv, PrePatchGeom geom, OUT* __restrict__ out) {
    pdl_launch_dependents();
    extern __shared__ uint32_t pre_smem[];
    const PreImage im = images[blockIdx.y];
    const int ty = blockIdx.x / im.col_tiles, tx = blockIdx.x - ty * im.col_tiles;
    const int y0 = ty * im.tile_rows;
    if (y0 >= im.out_h) return;
    const int out_w = im.out_w, tw = im.tile_cols, x0 = tx * tw;
    const int ny = min(im.tile_rows, im.out_h - y0), nx = min(tw, out_w - x0);
    const int chunk_rows = im.chunk_groups * 4;
    const int* hstart = tables + im.htab;
    const uint32_t* hwords = reinterpret_cast<const uint32_t*>(hstart + 2 * out_w);
    // groups of 4 canvas columns [x_lo4, x_lo4 + span4) the tap words of this tile's columns touch: the windows are monotonic in x
    const int x_lo4 = hstart[x0];
    const int span4 = hstart[x0 + nx - 1] + im.hnp - x_lo4;
    float* lut = reinterpret_cast<float*>(pre_smem);                          // [3][256] normalised value of every grey level
    uint32_t* band = pre_smem + 768;                                           // [3][band_groups][tile_cols]: 4 canvas rows per word
    uint32_t* stage = band + (size_t)3 * im.band_groups * tw;                  // [3][chunk_rows][span4]: 4 canvas columns per word
    const int* vstart = tables + im.vtab;
    const int* vlast = vstart + im.out_h;
    const uint32_t* vwords = reinterpret_cast<const uint32_t*>(vstart + 2 * im.out_h);
    // groups of 4 canvas rows this band needs: the windows are monotonic in y
    const int g0 = vstart[y0];
    const int ng = vlast[y0 + ny - 1] - g0 + 1;
    const uint8_t* img = src + im.src_off;
    const unsigned bgc[3] = {background.x, background.y, background.z};
    const int lane_x = threadIdx.x % PRE_XL, grp = threadIdx.x / PRE_XL;

    pre_fill_lut(lut, mean, stdv);

    for (int cg = 0; cg < ng; cg += im.chunk_groups) {
        const int ngc = min(im.chunk_groups, ng - cg);
        // ---- stage canvas rows 4 (g0 + cg) ... as byte planes, 4 columns per word; outside the pasted image = padding colour
        for (int rr = 0; rr < ngc * 4; ++rr) {
            const int sy = 4 * (g0 + cg) + rr - im.paste_y;
            const bool row_in = sy >= 0 && sy < im.h;
            const uint8_t* row = img + (size_t)(row_in ? sy : 0) * im.w * 3;
            for (int gx = threadIdx.x; gx < span4; gx += PRE_THREADS) {
                const int sx0 = 4 * (x_lo4 + gx) - im.paste_x;
                uint32_t pr, pg, pb;
                if (row_in && sx0 >= 0 && sx0 + 3 < im.w) {
                    const uint8_t* p = row + (size_t)sx0 * 3;
                    if ((reinterpret_cast<uintptr_t>(p) & 3) == 0) {           // 12 aligned bytes: R0G0B0R1 G1B1R2G2 B2R3G3B3
                        const uint32_t w0 = reinterpret_cast<const uint32_t*>(p)[0], w1 = reinterpret_cast<const uint32_t*>(p)[1],
                                       w2 = reinterpret_cast<const uint32_t*>(p)[2];
                        pr = __byte_perm(__byte_perm(w0, w1, 0x0630), w2, 0x5210);
                        pg = __byte_perm(__byte_perm(w0, w1, 0x0741), w2, 0x6210);
                        pb = __byte_perm(__byte_perm(w0, w1, 0x0052), w2, 0x7410);
                    } else {
                        pr = p[0] | (p[3] << 8) | (p[6] << 16) | ((uint32_t)p[9] << 24);
                        pg = p[1] | (p[4] << 8) | (p[7] << 16) | ((uint32_t)p[10] << 24);
                        pb = p[2] | (p[5] << 8) | (p[8] << 16) | ((uint32_t)p[11] << 24);
                    }
                } else {
                    pr = pg = pb = 0;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int sx = sx0 + i;
                        const bool in = row_in && sx >= 0 && sx < im.w;
                        const uint8_t* p = row + (size_t)(in ? sx : 0) * 3;
                        pr |= (in ? (uint32_t)p[0] : bgc[0]) << (8 * i);
                        pg |= (in ? (uint32_t)p[1] : bgc[1]) << (8 * i);
                        pb |= (in ? (uint32_t)p[2] : bgc[2]) << (8 * i);
                    }
                }
                stage[(size_t)(0 * chunk_rows + rr) * span4 + gx] = pr;
                stage[(size_t)(1 * chunk_rows + rr) * span4 + gx] = pg;
                stage[(size_t)(2 * chunk_rows + rr) * span4 + gx] = pb;
            }
        }
        __syncthreads();
        // ---- horizontal pass (ImagingResampleHorizontal_8bpc): thread = one output column x one group of 4 canvas rows
        if (grp < ngc) {
            for (int xl = lane_x; xl < nx; xl += PRE_XL) {
                const int xx = x0 + xl;
                const int s4 = hstart[xx] - x_lo4;
                const uint32_t* kw = hwords + (size_t)xx * im.hnp * 3;
                unsigned a0[4][3], a1[4][3];
                int a2[4][3];
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int c = 0; c < 3; ++c) { a0[q][c] = 0; a1[q][c] = 0; a2[q][c] = 0; }
                for (int pw = 0; pw < im.hnp; ++pw) {
                    const uint32_t d0 = __ldg(kw + pw * 3), d1 = __ldg(kw + pw * 3 + 1), d2 = __ldg(kw + pw * 3 + 2);
#pragma unroll
                    for (int q = 0; q < 4; ++q)
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                            const uint32_t px = stage[(size_t)(c * chunk_rows + grp * 4 + q) * span4 + s4 + pw];
                            a0[q][c] = pre_dp4a_uu(px, d0, a0[q][c]);
                            a1[q][c] = pre_dp4a_uu(px, d1, a1[q][c]);
                            a2[q][c] = pre_dp4a_us(px, d2, a2[q][c]);
                        }
                }
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    uint32_t wv = 0;
#pragma unroll
                    for (int q = 0; q < 4; ++q) wv |= pre_finish(a0[q][c], a1[q][c], a2[q][c]) << (8 * q);
                    band[((size_t)c * im.band_groups + cg + grp) * tw + xl] = wv;
                }
            }
        }
        __syncthreads();
    }

    // ---- vertical pass (ImagingResampleVertical_8bpc) + normalisation
    OUT* dst = out + im.out_off;
    const int gwm = LAYOUT == PRE_QWEN_PATCHES ? out_w / (geom.patch * geom.merge) : 0;
    for (int yy = grp; yy < ny; yy += PRE_RG) {
        const int y = y0 + yy;
        const int gs = vstart[y] - g0;
        const uint32_t* kw = vwords + (size_t)y * im.vnp * 3;
        for (int xl = lane_x; xl < nx; xl += PRE_XL) {
            const int xx = x0 + xl;
            unsigned a0[3] = {0, 0, 0}, a1[3] = {0, 0, 0};
            int a2[3] = {0, 0, 0};
            for (int pw = 0; pw < im.vnp; ++pw) {
                const uint32_t d0 = __ldg(kw + pw * 3), d1 = __ldg(kw + pw * 3 + 1), d2 = __ldg(kw + pw * 3 + 2);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const uint32_t px = band[((size_t)c * im.band_groups + gs + pw) * tw + xl];
                    a0[c] = pre_dp4a_uu(px, d0, a0[c]);
                    a1[c] = pre_dp4a_uu(px, d1, a1[c]);
                    a2[c] = pre_dp4a_us(px, d2, a2[c]);
                }
            }
            float v[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) v[c] = lut[c * 256 + pre_finish(a0[c], a1[c], a2[c])];
            if constexpr (LAYOUT == PRE_CHW) {
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const size_t o = ((size_t)c * im.out_h + y) * out_w + xx;
                    if constexpr (sizeof(OUT) == 4) dst[o] = v[c];
                    else dst[o] = __float2bfloat16_rn(v[c]);
                }
            } else {
                pre_store_patch(dst, geom, gwm, y, xx, v, im.t0, im.nt);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- host: plan + launch
struct PrePlan {
    std::vector<PreImage> images;
    std::vector<int> tables;
    int max_tiles = 0;
    size_t smem = 0;
    std::string error;
    size_t images_bytes() const { return (images.size() * sizeof(PreImage) + 15) / 16 * 16; }
    size_t bytes() const { return images_bytes() + tables.size() * sizeof(int); }
};

struct PreTableKey { int ch, cw, nh, nw, top, left, oh, ow, htab, vtab, hnp, vnp, tile, tile_cols, col_tiles, band_groups, span4, chunk_groups; };
inline size_t pre_smem_bytes(int band_groups, int tile_cols, int chunk_groups, int span4) {
    return 768 * sizeof(float) + ((size_t)3 * band_groups * tile_cols + (size_t)3 * chunk_groups * 4 * span4) * sizeof(uint32_t);
}

// Process-wide forced tile plan (vqa_debug_set_preprocess_tiles; tests and tuning): every image gets tile_rows output rows and
// min(tile_cols, out_w) output columns per CTA and stages chunk_groups groups of 4 canvas rows per pass. All zero = the planner's choice.
struct PreTileOverride { int tile_rows, tile_cols, chunk_groups; };
inline PreTileOverride g_pre_tile_override{0, 0, 0};

// Tables + tile geometry for "resize the ch x cw canvas to nh x nw, keep the oh x ow window at (top, left)"; shared between images
// with the same geometry. Returns nullptr (plan.error set) when the filter windows cannot fit the shared-memory budget.
inline const PreTableKey* pre_tables(PrePlan& plan, std::vector<PreTableKey>& cache, int ch, int cw, int nh, int nw, int top, int left,
                                     int oh, int ow) {
    for (const PreTableKey& k : cache)
        if (k.ch == ch && k.cw == cw && k.nh == nh && k.nw == nw && k.top == top && k.left == left && k.oh == oh && k.ow == ow) return &k;
    PreTableKey k{ch, cw, nh, nw, top, left, oh, ow, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<int> raw;
    int ks = pre_build_table(cw, nw, left, ow, raw);
    k.htab = (int)plan.tables.size();
    k.hnp = pre_pack_table(raw.data(), raw.data() + (size_t)ow * 2, ow, ks, plan.tables);
    raw.clear();
    ks = pre_build_table(ch, nh, top, oh, raw);
    k.vtab = (int)plan.tables.size();
    k.vnp = pre_pack_table(raw.data(), raw.data() + (size_t)oh * 2, oh, ks, plan.tables);
    const int* hstart = plan.tables.data() + k.htab;
    const int* vstart = plan.tables.data() + k.vtab;
    // groups of 4 canvas rows the tallest band of `tile` output rows needs, and of 4 canvas columns the widest column tile of `tw` output
    // columns stages (windows are monotonic: first word of the first output .. last word of the last)
    auto band_of = [&](int tile) {
        int band = 0;
        for (int y0 = 0; y0 < oh; y0 += tile) {
            const int y1 = (y0 + tile < oh ? y0 + tile : oh) - 1;
            const int groups = vstart[y1] + k.vnp - vstart[y0];
            if (groups > band) band = groups;
        }
        return band;
    };
    auto span_of = [&](int tw) {
        int span = 0;
        for (int x0 = 0; x0 < ow; x0 += tw) {
            const int x1 = (x0 + tw < ow ? x0 + tw : ow) - 1;
            if (hstart[x1] + k.hnp - hstart[x0] > span) span = hstart[x1] + k.hnp - hstart[x0];
        }
        return span;
    };
    // groups of 4 canvas rows staged per pass (2 or 1): the most that fit; 0 when nothing does
    auto chunk_of = [&](int band, int tw, int span) {
        for (int chunk = PRE_RG; chunk >= 1; chunk >>= 1)
            if (pre_smem_bytes(band, tw, chunk, span) <= (size_t)PRE_MAX_SMEM) return chunk;
        return 0;
    };
    const PreTileOverride force = g_pre_tile_override;
    if (force.tile_rows) {
        const int tw = force.tile_cols < ow ? force.tile_cols : ow, band = band_of(force.tile_rows), span = span_of(tw);
        const size_t bytes = pre_smem_bytes(band, tw, force.chunk_groups, span);
        if (bytes > (size_t)PRE_MAX_SMEM) {
            plan.error = "the forced tile plan of vqa_debug_set_preprocess_tiles needs " + std::to_string(bytes) +
                         " bytes of shared memory for this image, over the " + std::to_string(PRE_MAX_SMEM) + "-byte budget";
            return nullptr;
        }
        k.tile = force.tile_rows; k.tile_cols = tw; k.col_tiles = (ow + tw - 1) / tw; k.band_groups = band; k.span4 = span;
        k.chunk_groups = force.chunk_groups;
        cache.push_back(k);
        return &cache.back();
    }
    // one column tile over the whole output width when it fits: the most output rows per CTA (<= 32)
    const int span_all = span_of(ow);
    for (int tile = 32; tile >= 1; tile >>= 1) {
        const int band = band_of(tile), chunk = chunk_of(band, ow, span_all);
        if (chunk) {
            k.tile = tile; k.tile_cols = ow; k.col_tiles = 1; k.band_groups = band; k.span4 = span_all; k.chunk_groups = chunk;
            cache.push_back(k);
            return &cache.back();
        }
    }
    // otherwise column tiles too: the (rows, columns) tile that fits with the least estimated work, counted in thread iterations of the
    // staging loop (weighted by its three loads and three stores per word), the horizontal and vertical tap loops, plus a fixed cost per CTA
    double best = 0.0;
    for (int tile = 32; tile >= 1; tile >>= 1) {
        const int band = band_of(tile), row_tiles = (oh + tile - 1) / tile;
        for (int nct = 2, prev = 0; nct <= ow; ++nct) {
            const int tw = (ow + nct - 1) / nct;
            if (tw == prev) continue;
            prev = tw;
            const int span = span_of(tw), chunk = chunk_of(band, tw, span);
            if (!chunk) continue;
            const int cols = (ow + tw - 1) / tw, lanes = (tw + PRE_XL - 1) / PRE_XL;
            const double stage = 4.0 * band * ((span + PRE_THREADS - 1) / PRE_THREADS);
            const double horiz = (double)((band + chunk - 1) / chunk) * lanes * k.hnp * 12;
            const double vert = (double)((tile + PRE_RG - 1) / PRE_RG) * lanes * k.vnp * 9;
            const double cost = (double)row_tiles * cols * (6.0 * stage + horiz + vert + 256.0);
            if (best == 0.0 || cost < best) {
                best = cost;
                k.tile = tile; k.tile_cols = tw; k.col_tiles = cols; k.band_groups = band; k.span4 = span; k.chunk_groups = chunk;
            }
        }
    }
    if (best == 0.0) { plan.error = "image too large for the device resize (filter windows exceed shared memory)"; return nullptr; }
    cache.push_back(k);
    return &cache.back();
}

inline void pre_finish_image(PrePlan& plan, PreImage& im, const PreTableKey& k) {
    im.htab = k.htab; im.vtab = k.vtab; im.hnp = k.hnp; im.vnp = k.vnp;
    im.tile_rows = k.tile; im.tile_cols = k.tile_cols; im.col_tiles = k.col_tiles; im.band_groups = k.band_groups;
    im.out_h = k.oh; im.out_w = k.ow; im.chunk_groups = k.chunk_groups;
    const int tiles = (k.oh + k.tile - 1) / k.tile * k.col_tiles;
    if (tiles > plan.max_tiles) plan.max_tiles = tiles;
    const size_t sm = pre_smem_bytes(k.band_groups, k.tile_cols, k.chunk_groups, k.span4);
    if (sm > plan.smem) plan.smem = sm;
}

// Geometry of CLIPImageProcessor for one image (shortest edge -> S, int() truncation of the long edge, centre crop S x S), on the
// padded canvas when pad_to_square. Output [n, 3, S, S].
inline bool pre_plan(const int32_t* heights, const int32_t* widths, const int64_t* offsets, int n, int S, bool pad, PrePlan& plan) {
    std::vector<PreTableKey> cache;
    cache.reserve(n);
    plan.images.resize(n);
    for (int i = 0; i < n; ++i) {
        const int h = heights[i], w = widths[i];
        if (h <= 0 || w <= 0) { plan.error = "image with non-positive size"; return false; }
        PreImage& im = plan.images[i];
        im.src_off = offsets[i]; im.h = h; im.w = w;
        const int side = h > w ? h : w;
        if (pad && side > PRE_MAX_CANVAS) { plan.error = "image too large for the device resize (padded canvas side over 65500 px)"; return false; }
        im.canvas_h = pad ? side : h; im.canvas_w = pad ? side : w;
        im.paste_x = pad ? (side - w) / 2 : 0; im.paste_y = pad ? (side - h) / 2 : 0;
        const int ch = im.canvas_h, cw = im.canvas_w;
        // get_resize_output_image_size(shortest_edge = S, default_to_square = False): short -> S, long -> int(S * long / short)
        const int nw = cw <= ch ? S : (int)((double)S * cw / ch);
        const int nh = cw <= ch ? (int)((double)S * ch / cw) : S;
        const PreTableKey* k = pre_tables(plan, cache, ch, cw, nh, nw, (nh - S) / 2, (nw - S) / 2, S, S);   // centre crop
        if (!k) return false;
        pre_finish_image(plan, im, *k);
        im.out_off = (long long)i * 3 * S * S;
    }
    return true;
}

// qwen_vl_utils / Qwen2VLImageProcessor smart_resize (image_processing_qwen2_vl.py:62-87): both sides multiples of `factor`, pixel
// count within [min_pixels, max_pixels]. Python's round() is round-half-even = nearbyint in the default rounding mode.
inline bool pre_smart_resize(int height, int width, int factor, long long min_pixels, long long max_pixels, int& h_bar, int& w_bar) {
    const int mx = height > width ? height : width, mn = height > width ? width : height;
    if ((double)mx / mn > 200.0) return false;
    h_bar = (int)std::nearbyint((double)height / factor) * factor;
    w_bar = (int)std::nearbyint((double)width / factor) * factor;
    if ((long long)h_bar * w_bar > max_pixels) {
        const double beta = std::sqrt(((double)height * width) / (double)max_pixels);
        h_bar = (int)std::floor((double)height / beta / factor) * factor;
        w_bar = (int)std::floor((double)width / beta / factor) * factor;
        if (h_bar < factor) h_bar = factor;
        if (w_bar < factor) w_bar = factor;
    } else if ((long long)h_bar * w_bar < min_pixels) {
        const double beta = std::sqrt((double)min_pixels / ((double)height * width));
        h_bar = (int)std::ceil((double)height * beta / factor) * factor;
        w_bar = (int)std::ceil((double)width * beta / factor) * factor;
    }
    return true;
}

// Qwen still images and frame stacks: one smart_resize per item (all frames of a stack share their size, so they share one set of
// tables), plain bicubic resize of the whole frame (no canvas, no crop), patch-row output. Item i has n_frames[i] frames at byte
// offsets frame_offsets[f0 .. f0 + n_frames[i]) of `src`; a still (is_video[i] == 0, one frame) fills every temporal slot of its rows,
// a video's frame f fills slot f % temporal of the rows of temporal group f / temporal, and its last frame also fills the slots after
// its own (the processor pads the stack with copies of the last frame, video_processing_qwen2_vl.py:245-249). Item i's rows start at
// sum_{j<i} t_j * gh_j * gw_j; grid_thw[i] = (t, gh, gw) with t = 1 for a still and ceil(n_frames / temporal) for a video.
inline bool pre_plan_qwen_video(const int32_t* n_frames, const int32_t* heights, const int32_t* widths, const int32_t* is_video,
                                const int64_t* frame_offsets, int n, int patch, int merge, int temporal, long long min_pixels,
                                long long max_pixels, PrePlan& plan, int32_t* grid_thw, long long* total_rows) {
    std::vector<PreTableKey> cache;
    cache.reserve(n);
    plan.images.clear();
    long long rows = 0;
    const long long row_elems = 3LL * temporal * patch * patch;
    for (int i = 0; i < n; ++i) {
        const int h = heights[i], w = widths[i], nf = n_frames[i];
        if (h <= 0 || w <= 0) { plan.error = "image with non-positive size"; return false; }
        if (nf <= 0 || (!is_video[i] && nf != 1)) { plan.error = "a video needs at least one frame and a still image exactly one"; return false; }
        int rh, rw;
        if (!pre_smart_resize(h, w, patch * merge, min_pixels, max_pixels, rh, rw)) {
            plan.error = "absolute aspect ratio must be smaller than 200";
            return false;
        }
        const PreTableKey* k = pre_tables(plan, cache, h, w, rh, rw, 0, 0, rh, rw);
        if (!k) return false;
        const long long frame_rows = (long long)(rh / patch) * (rw / patch);
        const int gt = is_video[i] ? (nf + temporal - 1) / temporal : 1;
        for (int f = 0; f < nf; ++f) {
            PreImage im{};
            im.src_off = frame_offsets[f]; im.h = h; im.w = w;
            im.canvas_h = h; im.canvas_w = w;
            pre_finish_image(plan, im, *k);
            im.out_off = (rows + (long long)(f / temporal) * frame_rows) * row_elems;
            im.t0 = is_video[i] ? f % temporal : 0;
            im.nt = f + 1 < nf ? 1 : temporal - im.t0;
            plan.images.push_back(im);
        }
        frame_offsets += nf;
        if (grid_thw) { grid_thw[3 * i] = gt; grid_thw[3 * i + 1] = rh / patch; grid_thw[3 * i + 2] = rw / patch; }
        rows += gt * frame_rows;
    }
    if (total_rows) *total_rows = rows;
    return true;
}

// ---------------------------------------------------------------------------------------------- torch's antialiased bicubic resize
// A video FILE reaches the Qwen processor through qwen_vl_utils fetch_video, which resizes the sampled frames as one tensor with
// torchvision resize(BICUBIC, antialias=True): uint8 -> fp32, torch's _upsample_bicubic2d_aa, clamp to [0, 255], round half to even, uint8.
// On the CPU that is separable_upsample_generic_Nd_kernel_impl (aten/src/ATen/native/cpu/UpSampleKernel.cpp): the horizontal pass into an
// fp32 buffer, then the vertical pass, each output t0 * w0 + t1 * w1 + ... accumulated in tap order. This kernel runs the same two fp32
// passes with fused multiply-adds in that order. The weights are torch's own fp32 values, read off on the host by resizing impulses
// (engine._aa_bicubic_taps); every output of an axis reads `taps` consecutive inputs from first[i], zero weights padding a shorter
// window (adding 0 * t leaves an fp32 sum unchanged). The uint8 result then goes through pre_store_patch like a still image's pixels.
//
// One CTA = one frame x a tile of tile_rows x PRE_AA_TX output pixels. It runs the horizontal pass for the band of input rows its output
// rows read (fp32 in shared memory, [3][band_rows][PRE_AA_TX]) and then the vertical pass out of that band.
constexpr int PRE_AA_TX = 64;
constexpr int PRE_AA_MAX_SMEM = 96 * 1024;

struct PreAAGeom {
    int in_h, in_w, out_h, out_w, htaps, vtaps;
    int tile_rows, band_rows, tiles_x;
    int frame0, total_frames;    // index in the video of the launch's first frame; frames of the whole video
};

inline size_t pre_aa_smem_bytes(int band_rows) { return (768 + (size_t)3 * band_rows * PRE_AA_TX) * sizeof(float); }

// tables: first_h[out_w] | first_v[out_h] | fp32 weights_h[out_w][htaps] | fp32 weights_v[out_h][vtaps]. `out` is the video's first patch
// row; frame f of the launch (frame frame0 + f of the video) fills slot (frame0 + f) % temporal of temporal group (frame0 + f) / temporal,
// and the video's last frame also the slots after its own (the processor pads with copies of the last frame).
template <typename OUT>
__global__ void __launch_bounds__(PRE_THREADS)
video_resize_aa_kernel(const uint8_t* __restrict__ src, const int* __restrict__ tables, PreAAGeom g, PrePatchGeom geom, float3 mean,
                       float3 stdv, OUT* __restrict__ out) {
    extern __shared__ float aa_smem[];
    float* lut = aa_smem;                                                   // [3][256]
    float* band = aa_smem + 768;                                            // [3][band_rows][PRE_AA_TX]
    const int x0 = (blockIdx.x % g.tiles_x) * PRE_AA_TX, y0 = (blockIdx.x / g.tiles_x) * g.tile_rows;
    const int nx = min(PRE_AA_TX, g.out_w - x0), ny = min(g.tile_rows, g.out_h - y0);
    const int* first_h = tables;
    const int* first_v = first_h + g.out_w;
    const float* w_h = reinterpret_cast<const float*>(first_v + g.out_h);
    const float* w_v = w_h + (size_t)g.out_w * g.htaps;
    const int r0 = first_v[y0], nr = first_v[y0 + ny - 1] + g.vtaps - r0;  // input rows of this tile (<= band_rows, windows monotonic)
    const uint8_t* img = src + (size_t)blockIdx.y * g.in_h * g.in_w * 3;
    pre_fill_lut(lut, mean, stdv);

    // ---- horizontal pass: thread = one output column x one input row, three channels
    for (int i = threadIdx.x; i < nr * PRE_AA_TX; i += PRE_THREADS) {
        const int r = i / PRE_AA_TX, xl = i - r * PRE_AA_TX;
        if (xl >= nx) continue;
        const int x = x0 + xl;
        const uint8_t* p = img + ((size_t)(r0 + r) * g.in_w + first_h[x]) * 3;
        const float* w = w_h + (size_t)x * g.htaps;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int j = 0; j < g.htaps; ++j) {
            const float wj = __ldg(w + j);
            a0 = __fmaf_rn((float)p[3 * j], wj, a0);
            a1 = __fmaf_rn((float)p[3 * j + 1], wj, a1);
            a2 = __fmaf_rn((float)p[3 * j + 2], wj, a2);
        }
        band[(0 * g.band_rows + r) * PRE_AA_TX + xl] = a0;
        band[(1 * g.band_rows + r) * PRE_AA_TX + xl] = a1;
        band[(2 * g.band_rows + r) * PRE_AA_TX + xl] = a2;
    }
    __syncthreads();

    // ---- vertical pass, round half to even, clamp, normalise, patch rows
    const int f = g.frame0 + blockIdx.y;
    const int t0 = f % geom.temporal, nt = f + 1 < g.total_frames ? 1 : geom.temporal - t0;
    const int gwm = g.out_w / (geom.patch * geom.merge);
    OUT* dst = out + (size_t)(f / geom.temporal) * (g.out_h / geom.patch) * (g.out_w / geom.patch) * (3 * geom.temporal * geom.patch * geom.patch);
    for (int i = threadIdx.x; i < ny * PRE_AA_TX; i += PRE_THREADS) {
        const int yl = i / PRE_AA_TX, xl = i - yl * PRE_AA_TX;
        if (xl >= nx) continue;
        const int y = y0 + yl;
        const float* w = w_v + (size_t)y * g.vtaps;
        const float* b = band + (first_v[y] - r0) * PRE_AA_TX + xl;
        float a[3] = {0.f, 0.f, 0.f};
        for (int j = 0; j < g.vtaps; ++j) {
            const float wj = __ldg(w + j);
#pragma unroll
            for (int c = 0; c < 3; ++c) a[c] = __fmaf_rn(b[(c * g.band_rows + j) * PRE_AA_TX], wj, a[c]);
        }
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = lut[c * 256 + min(max(__float2int_rn(a[c]), 0), 255)];
        pre_store_patch(dst, geom, gwm, y, x0 + xl, v, t0, nt);
    }
}

// Process-wide forced output rows per CTA of video_resize_aa_kernel (vqa_debug_set_preprocess_aa_rows; tests): 1 ... 32, 0 = the
// planner's choice.
inline int g_pre_aa_rows_override = 0;

// Host checks and launch geometry of video_resize_aa_kernel: every window inside its axis and the vertical windows monotonic; the
// output rows per CTA (<= 32, a power of two) are the most whose band of input rows fits PRE_AA_MAX_SMEM, or the forced count.
inline bool pre_plan_aa(int in_h, int in_w, int out_h, int out_w, const int32_t* first_h, int htaps, const int32_t* first_v, int vtaps,
                        int patch, int merge, PreAAGeom& g, std::string& error) {
    if (in_h <= 0 || in_w <= 0 || out_h <= 0 || out_w <= 0 || htaps <= 0 || vtaps <= 0 || htaps > in_w || vtaps > in_h) {
        error = "bad sizes or tap counts";
        return false;
    }
    if (out_h % (patch * merge) || out_w % (patch * merge)) { error = "the output size must be a multiple of patch * merge"; return false; }
    for (int x = 0; x < out_w; ++x)
        if (first_h[x] < 0 || first_h[x] > in_w - htaps) { error = "horizontal window outside the frame"; return false; }
    for (int y = 0; y < out_h; ++y)
        if (first_v[y] < 0 || first_v[y] > in_h - vtaps || (y && first_v[y] < first_v[y - 1])) {
            error = "vertical windows outside the frame or not monotonic";
            return false;
        }
    g = PreAAGeom{in_h, in_w, out_h, out_w, htaps, vtaps, 0, 0, (out_w + PRE_AA_TX - 1) / PRE_AA_TX, 0, 0};
    auto band_of = [&](int tile) {       // input rows of the tallest band of `tile` output rows
        int band = 0;
        for (int y0 = 0; y0 < out_h; y0 += tile) {
            const int y1 = (y0 + tile < out_h ? y0 + tile : out_h) - 1;
            if (first_v[y1] + vtaps - first_v[y0] > band) band = first_v[y1] + vtaps - first_v[y0];
        }
        return band;
    };
    if (const int tile = g_pre_aa_rows_override) {
        const int band = band_of(tile);
        if (pre_aa_smem_bytes(band) > (size_t)PRE_AA_MAX_SMEM) {
            error = "the forced row tile of vqa_debug_set_preprocess_aa_rows needs " + std::to_string(pre_aa_smem_bytes(band)) +
                    " bytes of shared memory for this resize, over the " + std::to_string(PRE_AA_MAX_SMEM) + "-byte budget";
            return false;
        }
        g.tile_rows = tile; g.band_rows = band;
        return true;
    }
    for (int tile = 32; tile >= 1; tile >>= 1) {
        const int band = band_of(tile);
        if (pre_aa_smem_bytes(band) <= (size_t)PRE_AA_MAX_SMEM) { g.tile_rows = tile; g.band_rows = band; return true; }
    }
    error = "downscale too steep for the device resize (vertical window exceeds shared memory)";
    return false;
}

}  // namespace vqa

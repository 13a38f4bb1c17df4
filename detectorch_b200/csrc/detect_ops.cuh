// detectorch_b200 -- the non-GEMM device stages of the detector, all on-device and sync-free:
//   stem image packing, maxpool, P6 subsample               (torchvision trunk glue, detector.py:183,250)
//   rpn_select_*_kernel, rpn_proposals_kernel, rpn_nms_scan_kernel  top-k + decode + clip + filter + NMS(0.7)   generate_proposals.py:31-122
//   collect_kernel         merge levels, top-N, FPN level map           collect_and_distribute...py:84-128,
//                                                                       multilevel_rois.py:41-53
//   collect_outputs_kernel collected RoIs / scale + their RPN scores       result_utils.py:77 (propose_images only)
//   fast_props_kernel      pre-computed proposals -> scaled, deduplicated preprocess_sample.py:37-47,61-69,
//                          RoIs in hash order + FPN level               multilevel_rois.py:19-39
//   softmax_split_kernel   class softmax + split cls/bbox               detector.py:277-284
//   det_class_kernel / det_limit_kernel  decode, clip, score>0.05, per-class NMS(0.5), top-100
//                                                                       result_utils.py:76-168, boxes.py:150-208
//   mask_rois_kernel       detections -> scaled RoIs + FPN level        eval_mask_FPN.ipynb cell 10, multilevel_rois.py:19-39
// The reference runs all of these on the host with numpy/Cython between device syncs.
#pragma once
#include "common.cuh"
#include "sort_nms.cuh"

namespace dt {

static constexpr float kBBoxXformClip = 4.135166556742356f;   // log(1000/16), boxes.py:73

// image NCHW [B,3,H,W] -> zero-bordered NHWC4 [B,Hp,Wp,4] (3-pixel border = the conv1 padding; channel 3 = 0).  im_info (may be null):
// everything outside image b is written as zero, whatever the canvas holds there (NaN included)
static __global__ void stem_pack_nhwc4_kernel(const float* __restrict__ img, int B, int H, int W, int Hp, int Wp, float* __restrict__ x4,
                                              const float* __restrict__ im_info) {
    const long long total = (long long)B * Hp * Wp;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int xp = (int)(i % Wp);
        const int yp = (int)((i / Wp) % Hp);
        const int b = (int)(i / ((long long)Wp * Hp));
        const int x = xp - 3, y = yp - 3;
        const ImageInfo g = image_info(im_info, b, 1, H, W);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x >= 0 && x < g.w && y >= 0 && y < g.h) {
            const size_t o = ((size_t)b * 3 * H + y) * W + x;
            v.x = __ldg(img + o); v.y = __ldg(img + o + (size_t)H * W); v.z = __ldg(img + o + 2 * (size_t)H * W);
        }
        reinterpret_cast<float4*>(x4)[i] = v;
    }
}

// fp16 hi/lo split of four fp32 values (h = fp16(v), l = fp16(v - h): the operand format of the kind::f16 three-term product); `bad`
// is raised when a value does not fit fp16
__device__ __forceinline__ void split_planes4(float4 v, uint2* hi, uint2* lo, bool* bad) {
    const float f[4] = {v.x, v.y, v.z, v.w};
    __half h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        h[j] = __float2half_rn(f[j]);
        l[j] = __float2half_rn(f[j] - __half2float(h[j]));
        *bad = *bad || !(fabsf(f[j]) < 65504.f);
    }
    *hi = *reinterpret_cast<const uint2*>(h);
    *lo = *reinterpret_cast<const uint2*>(l);
}

// stem_pack_nhwc4_kernel emitting the two fp16 planes [B, Hp, Wp, 4] the kind::f16 stem loads straight into its operand tiles
static __global__ void stem_pack_nhwc4_planes_kernel(const float* __restrict__ img, int B, int H, int W, int Hp, int Wp, uint2* __restrict__ xh,
                                                     uint2* __restrict__ xl, int* __restrict__ range_flag, const float* __restrict__ im_info) {
    const long long total = (long long)B * Hp * Wp;
    bool bad = false;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int xp = (int)(i % Wp);
        const int yp = (int)((i / Wp) % Hp);
        const int b = (int)(i / ((long long)Wp * Hp));
        const int x = xp - 3, y = yp - 3;
        const ImageInfo g = image_info(im_info, b, 1, H, W);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x >= 0 && x < g.w && y >= 0 && y < g.h) {
            const size_t o = ((size_t)b * 3 * H + y) * W + x;
            v.x = __ldg(img + o); v.y = __ldg(img + o + (size_t)H * W); v.z = __ldg(img + o + 2 * (size_t)H * W);
        }
        uint2 h, l;
        split_planes4(v, &h, &l, &bad);
        xh[i] = h; xl[i] = l;
    }
    if (bad && range_flag) *range_flag = 1;
}

// NHWC 3x3 stride-2 pad-1 max pool (torchvision maxpool).  im_info (may be null): the window ends at image b's extent (the input is the
// stride-2 map), and outputs past it are zero.
static __global__ void maxpool3x3s2_nhwc_kernel(const float* __restrict__ x, int B, int H, int W, int C, int Ho, int Wo, float* __restrict__ y,
                                                const float* __restrict__ im_info) {
    const int C4 = C >> 2;
    const long long total = (long long)B * Ho * Wo * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        long long m = i / C4;
        const int wo = (int)(m % Wo); m /= Wo;
        const int ho = (int)(m % Ho);
        const int b = (int)(m / Ho);
        const ImageInfo g = image_info(im_info, b, 2, H, W);
        float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int dy = 0; dy < 3; ++dy) {
            const int yy = ho * 2 - 1 + dy;
            if (yy < 0 || yy >= g.h) continue;
            for (int dx = 0; dx < 3; ++dx) {
                const int xx = wo * 2 - 1 + dx;
                if (xx < 0 || xx >= g.w) continue;
                const float4 v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)b * H + yy) * W + xx) * C) + c4);
                best.x = fmaxf(best.x, v.x); best.y = fmaxf(best.y, v.y); best.z = fmaxf(best.z, v.z); best.w = fmaxf(best.w, v.w);
            }
        }
        if (ho * 2 >= g.h || wo * 2 >= g.w) best = make_float4(0.f, 0.f, 0.f, 0.f);
        reinterpret_cast<float4*>(y)[i] = best;
    }
}

// P6 = max_pool2d(P5, kernel 1, stride 2) == stride-2 subsample (detector.py:250).  With per-image sizes no mask is needed: output
// (ho, wo) reads P5 at (2 ho, 2 wo), which lies inside image b's P5 extent exactly when (ho, wo) lies inside its P6 extent
// ceil(H5 / 2), and P5 is zero outside (the conv epilogue).
static __global__ void subsample2_nhwc_kernel(const float* __restrict__ x, int B, int H, int W, int C, int Ho, int Wo, float* __restrict__ y) {
    const int C4 = C >> 2;
    const long long total = (long long)B * Ho * Wo * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        long long m = i / C4;
        const int wo = (int)(m % Wo); m /= Wo;
        const int ho = (int)(m % Ho);
        const int b = (int)(m / Ho);
        reinterpret_cast<float4*>(y)[i] = __ldg(reinterpret_cast<const float4*>(x + (((size_t)b * H + ho * 2) * W + wo * 2) * C) + c4);
    }
}

// global average pool of the res5 head: x [R, S, C] (S = 7*7 positions, NHWC) -> y [R, C]   (torchvision avgpool, detector.py:136,191)
static __global__ void avgpool_nhwc_kernel(const float* __restrict__ x, int R, int S, int C, float* __restrict__ y) {
    const int C4 = C >> 2;
    const long long total = (long long)R * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        const long long r = i / C4;
        const float4* p = reinterpret_cast<const float4*>(x + (size_t)r * S * C) + c4;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < S; ++s) {
            const float4 v = __ldg(p + (size_t)s * C4);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        const float inv = 1.f / (float)S;
        reinterpret_cast<float4*>(y)[i] = make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
    }
}

// ---------------------------------------------------------------------------------- box decode helpers
// generate_proposals.py:165-214 / boxes.py:168-208: separate mul and add (torch / numpy evaluate op by op)
__device__ __forceinline__ float4 decode_box(float4 box, float dx, float dy, float dw, float dh) {
    const float w = __fadd_rn(__fsub_rn(box.z, box.x), 1.0f);
    const float h = __fadd_rn(__fsub_rn(box.w, box.y), 1.0f);
    const float cx = __fadd_rn(box.x, __fmul_rn(0.5f, w));
    const float cy = __fadd_rn(box.y, __fmul_rn(0.5f, h));
    dw = fminf(dw, kBBoxXformClip);
    dh = fminf(dh, kBBoxXformClip);
    const float pcx = __fadd_rn(__fmul_rn(dx, w), cx);
    const float pcy = __fadd_rn(__fmul_rn(dy, h), cy);
    const float pw = __fmul_rn(expf(dw), w);
    const float ph = __fmul_rn(expf(dh), h);
    float4 o;
    o.x = __fsub_rn(pcx, __fmul_rn(0.5f, pw));
    o.y = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
    o.z = __fsub_rn(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), 1.f);
    o.w = __fsub_rn(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), 1.f);
    return o;
}
__device__ __forceinline__ float4 clip_box(float4 b, float wmax, float hmax) {   // wmax = W-1, hmax = H-1
    b.x = fmaxf(fminf(b.x, wmax), 0.f); b.y = fmaxf(fminf(b.y, hmax), 0.f);
    b.z = fmaxf(fminf(b.z, wmax), 0.f); b.w = fmaxf(fminf(b.w, hmax), 0.f);
    return b;
}

// ---------------------------------------------------------------------------------- RPN proposals
struct RpnLevel {
    const float* rpn_out;    // NHWC [B,H,W,ch_stride]: ch [0,A) = objectness prob, [A+4a, A+4a+4) = deltas of anchor a
    int H, W, A, ch_stride;
    float stride;            // 1/spatial_scale
    float anchors[15 * 4];   // base anchors (x1,y1,x2,y2), generate_anchors.py
    long long ws_off;        // offset (in elements) of this level's per-image sort workspace
    int n;                   // H*W*A
};
struct RpnParams {
    RpnLevel lv[5];
    int num_levels, B;
    int pre_nms, post_nms;
    float nms_thresh, min_size, scaling_factor;
    float im_h, im_w;
    const float* im_info;    // per-image sizes and scales (image_info), null = every image fills the canvas
    long long ws_per_image;  // elements of sort workspace per image (sum over levels)
    uint32_t *k0, *k1;       // [B * ws_per_image]
    int *v0, *v1;
    float4* cand;            // [B * L * pre_nms] decoded candidates (score-sorted)
    float* cand_score;
    float* out_props;        // [B, L, post_nms, 4]
    float* out_scores;       // [B, L, post_nms]
    int* out_counts;         // [B, L]
    // optional teacher-forcing taps (may be null)
    int* dbg_order;          // [B, L, pre_nms] flat anchor index of the sorted top-k
    // multi-CTA selection (rpn_select_*_kernel): per (image, level) two 2048-bin digit histograms, per-chunk selected counts, (b1, b2, total)
    uint32_t* sel_hist;      // [B, L, 2, 2048], zeroed before every run
    int sel_chunks;          // ceil(largest level / kRpnChunk): the x extent of the selection grid
    int* sel_chunk_counts;   // [B, L, sel_chunks]
    int* sel_info;           // [B, L, 4]: b1, b2, total (-1: not narrowed -> full sort), unused
    // NMS at full-GPU width (nms_mask_kernel + rpn_nms_scan_kernel) when nms_thresh > 0: rpn_proposals_kernel then stops after decode / filter
    int nms_chunks;          // ceil(pre_nms / 64)
    int* cand_counts;        // [B, L] candidates that passed the filter
    unsigned long long* nms_mask;   // [B, L, pre_nms, nms_chunks]: bit b of word (i, w) set <=> candidate i suppresses candidate w*64 + b (> i)
};
static constexpr int kRpnChunk = 4096;        // anchors per CTA of the selection kernels (1024 threads x 4)

__host__ __device__ __forceinline__ bool rpn_level_selects(int n, int K) { return n > 4 * K && n > 8192; }

// Image b's anchors on level lv: the ceil(net / stride) rows and columns of its valid region, n = h * w * A of them, numbered
// (y * w + x) * A + a like those of a batch-1 run at that size (the top-k tie order and dbg_order follow this image-local index).
struct RpnImageLevel { int n, w; };
__device__ __forceinline__ RpnImageLevel rpn_image_level(const RpnParams& P, const RpnLevel& lv, int b) {
    if (!P.im_info) return {lv.n, lv.W};
    const ImageInfo g = image_info(P.im_info, b, (int)lv.stride, lv.H, lv.W);
    return {g.h * g.w * lv.A, g.w};
}
// canvas cell (row-major over the level's W columns) of image-local cell `cell` of an image w cells wide
__device__ __forceinline__ size_t rpn_canvas_cell(int cell, int w, int W) { return (size_t)(cell / w) * W + (cell % w); }

// first bin with c0 + prefix >= K among 2048 bins (warp-collective, all 32 lanes of ONE warp must call); h may be global or shared
__device__ __forceinline__ void rpn_find_bin(const uint32_t* h, uint32_t c0, uint32_t K, uint32_t* out_bin, uint32_t* out_c) {
    const int lane = threadIdx.x & 31;
    uint32_t sum = 0;
    for (int t = 0; t < 64; ++t) sum += h[lane * 64 + t];
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    const uint32_t excl = c0 + incl - sum;
    const bool hit = excl + sum >= K;
    const unsigned hits = __ballot_sync(0xffffffffu, hit);
    const uint32_t all = __shfl_sync(0xffffffffu, incl, 31);
    if (hits == 0) { if (lane == 0) { *out_bin = 2048; *out_c = c0 + all; } }
    else if (lane == __ffs(hits) - 1) {
        uint32_t c = excl, bb = (uint32_t)lane * 64;
        for (; bb < (uint32_t)lane * 64 + 64; ++bb) { if (c + h[bb] >= K) break; c += h[bb]; }
        *out_bin = bb; *out_c = c;
    }
}

// ---- selection pass 1: keys in (H,W,A) order + first-level digit histogram.  grid (chunks, L, B), 1024 threads.
static __global__ void __launch_bounds__(1024) rpn_select_keys_kernel(const __grid_constant__ RpnParams P) {
    __shared__ uint32_t hist[2048];
    const int l = blockIdx.y, b = blockIdx.z;
    const RpnLevel& lv = P.lv[l];
    const RpnImageLevel il = rpn_image_level(P, lv, b);
    const int n = il.n, i0 = blockIdx.x * kRpnChunk;
    if (i0 >= n) return;
    const int K = (P.pre_nms <= 0 || P.pre_nms >= n) ? n : P.pre_nms;
    const bool select = rpn_level_selects(n, K);
    uint32_t* k0 = P.k0 + (size_t)b * P.ws_per_image + lv.ws_off;
    int* v0 = P.v0 + (size_t)b * P.ws_per_image + lv.ws_off;
    const float* base = lv.rpn_out + (size_t)b * lv.H * lv.W * lv.ch_stride;
    if (select) { for (int i = threadIdx.x; i < 2048; i += blockDim.x) hist[i] = 0; __syncthreads(); }
    uint32_t k[4];
    bool valid[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = i0 + j * 1024 + threadIdx.x;
        valid[j] = i < n;
        k[j] = 0u;
        if (valid[j]) { const int a = i % lv.A, cell = i / lv.A; k[j] = float_desc_key(base[rpn_canvas_cell(cell, il.w, lv.W) * lv.ch_stride + a]); }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = i0 + j * 1024 + threadIdx.x;
        if (valid[j]) { k0[i] = k[j]; v0[i] = i; }
        if (select) {
            const unsigned act = __ballot_sync(0xffffffffu, valid[j]);
            if (valid[j]) {
                const uint32_t d = k[j] >> 21;
                const unsigned m = __match_any_sync(act, d);
                if ((m & ((1u << (threadIdx.x & 31)) - 1u)) == 0) atomicAdd(&hist[d], (uint32_t)__popc(m));
            }
        }
    }
    if (!select) return;
    __syncthreads();
    uint32_t* g = P.sel_hist + ((size_t)b * P.num_levels + l) * 4096;
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) if (hist[i]) atomicAdd(&g[i], hist[i]);      // integer counts: order-independent
}

// ---- selection pass 2: second-level digit histogram inside the boundary bin b1
static __global__ void __launch_bounds__(1024) rpn_select_hist2_kernel(const __grid_constant__ RpnParams P) {
    __shared__ uint32_t hist[2048];
    __shared__ uint32_t sel[2];
    const int l = blockIdx.y, b = blockIdx.z;
    const RpnLevel& lv = P.lv[l];
    const RpnImageLevel il = rpn_image_level(P, lv, b);
    const int n = il.n, i0 = blockIdx.x * kRpnChunk;
    if (i0 >= n) return;
    const int K = (P.pre_nms <= 0 || P.pre_nms >= n) ? n : P.pre_nms;
    if (!rpn_level_selects(n, K)) return;
    uint32_t* g = P.sel_hist + ((size_t)b * P.num_levels + l) * 4096;
    // the bin search walks the histogram serially: do it on a shared-memory copy (one coalesced load), not on 64 dependent L2 reads
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) hist[i] = g[i];
    __syncthreads();
    if (threadIdx.x < 32) rpn_find_bin(hist, 0u, (uint32_t)K, &sel[0], &sel[1]);
    __syncthreads();
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const uint32_t b1 = sel[0];
    const uint32_t* k0 = P.k0 + (size_t)b * P.ws_per_image + lv.ws_off;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = i0 + j * 1024 + threadIdx.x;
        const uint32_t key = i < n ? k0[i] : 0xffffffffu;
        const bool valid = (i < n) && ((key >> 21) == b1);
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const uint32_t d = (key >> 10) & 2047u;
            const unsigned m = __match_any_sync(act, d);
            if ((m & ((1u << (threadIdx.x & 31)) - 1u)) == 0) atomicAdd(&hist[d], (uint32_t)__popc(m));
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) if (hist[i]) atomicAdd(&g[2048 + i], hist[i]);
}

// ---- selection pass 3: per-chunk count of the selected keys; chunk 0 publishes (b1, b2, total)
static __global__ void __launch_bounds__(1024) rpn_select_count_kernel(const __grid_constant__ RpnParams P) {
    __shared__ uint32_t sel[4];
    __shared__ int scratch[33];
    __shared__ uint32_t hh[4096];
    const int l = blockIdx.y, b = blockIdx.z;
    const RpnLevel& lv = P.lv[l];
    const RpnImageLevel il = rpn_image_level(P, lv, b);
    const int n = il.n, i0 = blockIdx.x * kRpnChunk;
    if (i0 >= n) return;
    const int K = (P.pre_nms <= 0 || P.pre_nms >= n) ? n : P.pre_nms;
    if (!rpn_level_selects(n, K)) return;
    const uint32_t* g = P.sel_hist + ((size_t)b * P.num_levels + l) * 4096;
    for (int i = threadIdx.x; i < 4096; i += blockDim.x) hh[i] = g[i];      // both histograms into shared memory (see rpn_select_hist2_kernel)
    __syncthreads();
    if (threadIdx.x < 32) {
        rpn_find_bin(hh, 0u, (uint32_t)K, &sel[0], &sel[1]);
        __syncwarp();
        rpn_find_bin(hh + 2048, sel[1], (uint32_t)K, &sel[2], &sel[3]);
        __syncwarp();
        if (threadIdx.x == 0 && sel[2] < 2048u) sel[3] += hh[2048 + sel[2]];
    }
    __syncthreads();
    const uint32_t b1 = sel[0], b2 = sel[2], total = sel[3];
    int* info = P.sel_info + ((size_t)b * P.num_levels + l) * 4;
    if (blockIdx.x == 0 && threadIdx.x == 0) { info[0] = (int)b1; info[1] = (int)b2; info[2] = total <= 8192u ? (int)total : -1; }
    if (total > 8192u) return;
    const uint32_t* k0 = P.k0 + (size_t)b * P.ws_per_image + lv.ws_off;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = i0 + 4 * threadIdx.x + j;
        if (i < n) { const uint32_t key = k0[i], d1 = key >> 21; cnt += ((d1 < b1) || (d1 == b1 && ((key >> 10) & 2047u) <= b2)) ? 1 : 0; }
    }
    int tot;
    block_rank_count(cnt, scratch, &tot);
    if (threadIdx.x == 0) P.sel_chunk_counts[((size_t)b * P.num_levels + l) * P.sel_chunks + blockIdx.x] = tot;
}

// ---- selection pass 4: ordered compaction (ascending anchor index) into (k1, v1)
static __global__ void __launch_bounds__(1024) rpn_select_scatter_kernel(const __grid_constant__ RpnParams P) {
    __shared__ int scratch[33];
    __shared__ int offset;
    const int l = blockIdx.y, b = blockIdx.z;
    const RpnLevel& lv = P.lv[l];
    const RpnImageLevel il = rpn_image_level(P, lv, b);
    const int n = il.n, i0 = blockIdx.x * kRpnChunk;
    if (i0 >= n) return;
    const int K = (P.pre_nms <= 0 || P.pre_nms >= n) ? n : P.pre_nms;
    if (!rpn_level_selects(n, K)) return;
    const int* info = P.sel_info + ((size_t)b * P.num_levels + l) * 4;
    if (info[2] < 0) return;
    const uint32_t b1 = (uint32_t)info[0], b2 = (uint32_t)info[1];
    if (threadIdx.x == 0) {
        const int* cc = P.sel_chunk_counts + ((size_t)b * P.num_levels + l) * P.sel_chunks;
        int o = 0;
        for (int c = 0; c < (int)blockIdx.x; ++c) o += cc[c];
        offset = o;
    }
    __syncthreads();
    const uint32_t* k0 = P.k0 + (size_t)b * P.ws_per_image + lv.ws_off;
    uint32_t* k1 = P.k1 + (size_t)b * P.ws_per_image + lv.ws_off;
    int* v1 = P.v1 + (size_t)b * P.ws_per_image + lv.ws_off;
    uint32_t k[4];
    bool f[4];
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = i0 + 4 * threadIdx.x + j;
        k[j] = i < n ? k0[i] : 0xffffffffu;
        const uint32_t d1 = k[j] >> 21;
        f[j] = (i < n) && ((d1 < b1) || (d1 == b1 && ((k[j] >> 10) & 2047u) <= b2));
        cnt += f[j] ? 1 : 0;
    }
    int tot;
    int r = offset + block_rank_count(cnt, scratch, &tot);
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (f[j]) { k1[r] = k[j]; v1[r] = i0 + 4 * threadIdx.x + j; ++r; }
}


// grid (L, B), 1024 threads
static __global__ void __launch_bounds__(1024) rpn_proposals_kernel(const __grid_constant__ RpnParams P) {
    __shared__ uint32_t hist[32 * 256];
    __shared__ int scratch[33];
    const int l = blockIdx.x, b = blockIdx.y;
    const RpnLevel& lv = P.lv[l];
    const RpnImageLevel il = rpn_image_level(P, lv, b);
    const int n = il.n;
    uint32_t* k0 = P.k0 + (size_t)b * P.ws_per_image + lv.ws_off;
    uint32_t* k1 = P.k1 + (size_t)b * P.ws_per_image + lv.ws_off;
    int* v0 = P.v0 + (size_t)b * P.ws_per_image + lv.ws_off;
    int* v1 = P.v1 + (size_t)b * P.ws_per_image + lv.ws_off;
    const float* base = lv.rpn_out + (size_t)b * lv.H * lv.W * lv.ch_stride;
    // 1. keys in (H,W,A) order (generate_proposals.py:64,72): rpn_select_keys_kernel left them in (k0, v0)
    // 2. top-K by descending score (:77-86).  A full sort of ~180k keys by one CTA costs >1 ms, so rpn_select_*_kernel first narrowed
    //    the set with a two-level 11+11-bit radix select on the key (exact: every key below the boundary sub-bin plus the whole boundary
    //    sub-bin is kept): (k1, v1) hold those `total` pairs in ascending index order, and only they are stable-sorted here.  A level
    //    that does not select, or whose boundary sub-bin left more than 8192 keys (total < 0), is sorted whole.
    const int K = (P.pre_nms <= 0 || P.pre_nms >= n) ? n : P.pre_nms;
    const int total = rpn_level_selects(n, K) ? P.sel_info[((size_t)b * P.num_levels + l) * 4 + 2] : -1;
    const bool narrowed = total >= 0;
    block_radix_sort_asc_u32(narrowed ? k1 : k0, narrowed ? v1 : v0, narrowed ? k0 : k1, narrowed ? v0 : v1, narrowed ? total : n, hist);
    const int* vs = narrowed ? v1 : v0;     // the sorted anchor indices
    // 3. decode + clip + filter on the top K (:96-112), order preserved
    float4* cand = P.cand + ((size_t)b * P.num_levels + l) * P.pre_nms;
    float* cscore = P.cand_score + ((size_t)b * P.num_levels + l) * P.pre_nms;
    int nc = 0;
    // clip and centre filter against this image's network-input size
    const ImageInfo img = image_info(P.im_info, b, 1, (int)P.im_h, (int)P.im_w, P.scaling_factor);
    const float im_h = (float)img.h, im_w = (float)img.w;
    const float min_size = P.min_size * img.scale;
    for (int base_i = 0; base_i < K; base_i += blockDim.x) {
        const int i = base_i + threadIdx.x;
        bool keep = false;
        float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
        float sc = 0.f;
        if (i < K) {
            const int idx = vs[i];
            if (P.dbg_order) P.dbg_order[((size_t)b * P.num_levels + l) * P.pre_nms + i] = idx;
            const int a = idx % lv.A, cell = idx / lv.A;
            const int x = cell % il.w, y = cell / il.w;
            const size_t ccell = (size_t)y * lv.W + x;
            const float sx = (float)x * lv.stride, sy = (float)y * lv.stride;
            const float4 anc = make_float4(lv.anchors[a * 4 + 0] + sx, lv.anchors[a * 4 + 1] + sy, lv.anchors[a * 4 + 2] + sx,
                                           lv.anchors[a * 4 + 3] + sy);
            const float* d = base + ccell * lv.ch_stride + lv.A + a * 4;
            sc = base[ccell * lv.ch_stride + a];
            box = clip_box(decode_box(anc, d[0], d[1], d[2], d[3]), im_w - 1.f, im_h - 1.f);
            // filter_boxes (:151-163)
            const float ws = __fadd_rn(__fsub_rn(box.z, box.x), 1.f), hs = __fadd_rn(__fsub_rn(box.w, box.y), 1.f);
            const float xc = __fadd_rn(box.x, __fdiv_rn(ws, 2.f)), yc = __fadd_rn(box.y, __fdiv_rn(hs, 2.f));
            keep = (ws >= min_size) && (hs >= min_size) && (xc < im_w) && (yc < im_h);
        }
        int tot;
        const int r = block_rank(keep, scratch, &tot);
        if (keep) { cand[nc + r] = box; cscore[nc + r] = sc; }
        nc += tot;
    }
    __syncthreads();
    if (P.nms_thresh > 0.f) {
        // 4. NMS (:114-120) of the candidates (already in descending-score order) continues in nms_mask_kernel (all pair tests, every SM)
        // and rpn_nms_scan_kernel (the sequential survivor walk)
        if (threadIdx.x == 0) P.cand_counts[b * P.num_levels + l] = nc;
        return;
    }
    float* op = P.out_props + ((size_t)b * P.num_levels + l) * P.post_nms * 4;
    float* os = P.out_scores + ((size_t)b * P.num_levels + l) * P.post_nms;
    const int nout = min(nc, P.post_nms);
    for (int i = threadIdx.x; i < nout; i += blockDim.x) {
        const float4 bx = cand[i];
        op[i * 4 + 0] = bx.x; op[i * 4 + 1] = bx.y; op[i * 4 + 2] = bx.z; op[i * 4 + 3] = bx.w;
        os[i] = cscore[i];
    }
    if (threadIdx.x == 0) P.out_counts[b * P.num_levels + l] = nout;
}

// ---- RPN NMS, part 2 (part 1 is nms_mask_kernel over the (level, image) sets): the survivor walk over the bit-matrix + the first
// post_nms survivors out (generate_proposals.py:114-120).  grid (L, B), 1024 threads.
static __global__ void __launch_bounds__(1024) rpn_nms_scan_kernel(const __grid_constant__ RpnParams P) {
    __shared__ unsigned long long removed[128];   // up to 8192 candidates
    __shared__ NmsWalkSmem wsm;
    __shared__ int scratch[33];
    const int l = blockIdx.x, b = blockIdx.y, lb = b * P.num_levels + l;
    const int n = P.cand_counts[lb];
    block_nms_walk(P.nms_mask + (size_t)lb * P.pre_nms * P.nms_chunks, n, P.nms_chunks, P.post_nms, removed, &wsm);
    // ordered compaction of the survivors
    const float4* cand = P.cand + (size_t)lb * P.pre_nms;
    const float* cscore = P.cand_score + (size_t)lb * P.pre_nms;
    float* op = P.out_props + (size_t)lb * P.post_nms * 4;
    float* os = P.out_scores + (size_t)lb * P.post_nms;
    int nout = 0;
    for (int base_i = 0; base_i < n; base_i += blockDim.x) {
        const int i = base_i + threadIdx.x;
        const bool keep = (i < n) && !((removed[i >> 6] >> (i & 63)) & 1ull);
        int tot;
        const int r = block_rank(keep, scratch, &tot);
        const int pos = nout + r;
        if (keep && (P.post_nms <= 0 || pos < P.post_nms)) {
            const float4 bx = cand[i];
            op[pos * 4 + 0] = bx.x; op[pos * 4 + 1] = bx.y; op[pos * 4 + 2] = bx.z; op[pos * 4 + 3] = bx.w;
            os[pos] = cscore[i];
        }
        nout += tot;
    }
    if (P.post_nms > 0 && nout > P.post_nms) nout = P.post_nms;
    if (threadIdx.x == 0) P.out_counts[lb] = nout;
}

// ---------------------------------------------------------------------------------- collect + distribute
// FPN level heuristic, multilevel_rois.py:41-53 (fp32 numpy arithmetic)
__device__ __forceinline__ int fpn_level(float4 box, int k_min, int k_max) {
    const float area = box_area_p1(box);
    const float s = sqrtf(area);
    float lvl = floorf(__fadd_rn(4.f, log2f(__fadd_rn(__fdiv_rn(s, 224.f), 1e-6f))));
    lvl = fminf(fmaxf(lvl, (float)k_min), (float)k_max);
    return (int)lvl;
}

struct CollectParams {
    const float* props;      // [B, L, post_nms, 4]
    const float* scores;     // [B, L, post_nms]
    const int* counts;       // [B, L]
    int B, L, post_nms, top_n;
    int k_min, k_max;
    uint32_t *k0, *k1;       // [B, L*post_nms]
    int *v0, *v1;
    float* rois;             // [B, top_n, 5] (batch idx, x1,y1,x2,y2); rows >= count are zero
    int* levels;             // [B, top_n] level index (lvl - k_min)
    int* roi_counts;         // [B]
};

// grid B, 1024 threads
static __global__ void __launch_bounds__(1024) collect_kernel(const __grid_constant__ CollectParams P) {
    __shared__ uint32_t hist[32 * 256];
    __shared__ int seg_off[8];
    const int b = blockIdx.x;
    const int cap = P.L * P.post_nms;
    uint32_t* k0 = P.k0 + (size_t)b * cap; uint32_t* k1 = P.k1 + (size_t)b * cap;
    int* v0 = P.v0 + (size_t)b * cap; int* v1 = P.v1 + (size_t)b * cap;
    if (threadIdx.x == 0) {
        int o = 0;
        for (int l = 0; l < P.L; ++l) { seg_off[l] = o; o += P.counts[b * P.L + l]; }
        seg_off[P.L] = o;
    }
    __syncthreads();
    const int n = seg_off[P.L];
    // concatenation in level order (collect...py:98-100); value = l*post_nms + i
    for (int l = 0; l < P.L; ++l) {
        const int c = seg_off[l + 1] - seg_off[l];
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            k0[seg_off[l] + i] = float_desc_key(P.scores[((size_t)b * P.L + l) * P.post_nms + i]);
            v0[seg_off[l] + i] = l * P.post_nms + i;
        }
    }
    __syncthreads();
    block_radix_sort_asc_u32(k0, v0, k1, v1, n, hist);      // torch.sort(-scores) (:102)
    const int m = min(n, P.top_n);
    for (int i = threadIdx.x; i < P.top_n; i += blockDim.x) {
        float* r = P.rois + ((size_t)b * P.top_n + i) * 5;
        if (i < m) {
            const float* p = P.props + ((size_t)b * cap + v0[i]) * 4;
            const float4 box = make_float4(p[0], p[1], p[2], p[3]);
            r[0] = (float)b; r[1] = box.x; r[2] = box.y; r[3] = box.z; r[4] = box.w;
            P.levels[(size_t)b * P.top_n + i] = fpn_level(box, P.k_min, P.k_max) - P.k_min;
        } else {
            r[0] = (float)b; r[1] = r[2] = r[3] = r[4] = 0.f;
            P.levels[(size_t)b * P.top_n + i] = 0;
        }
    }
    if (threadIdx.x == 0) P.roi_counts[b] = m;
}

// The collected RoIs in original-image coordinates (rois / scaling_factor in fp32, as postprocess_output divides them) and each one's
// RPN score, read through the collect's sort order (v0 after the sort); rows >= roi_counts[b] are zero.  Not part of the engine
// program: dt_engine_proposals launches it after a run that ended at ST_COLLECT.  grid B
static __global__ void collect_outputs_kernel(const __grid_constant__ CollectParams P, const float* __restrict__ im_info, float scaling_factor,
                                              float* __restrict__ out_boxes, float* __restrict__ out_scores) {
    const int b = blockIdx.x;
    const int cap = P.L * P.post_nms;
    const int m = P.roi_counts[b];
    const float s = image_info(im_info, b, 1, 0, 0, scaling_factor).scale;
    for (int i = threadIdx.x; i < P.top_n; i += blockDim.x) {
        float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
        float score = 0.f;
        if (i < m) {
            const float* r = P.rois + ((size_t)b * P.top_n + i) * 5;
            box = make_float4(__fdiv_rn(r[1], s), __fdiv_rn(r[2], s), __fdiv_rn(r[3], s), __fdiv_rn(r[4], s));
            score = P.scores[(size_t)b * cap + P.v0[(size_t)b * cap + i]];
        }
        reinterpret_cast<float4*>(out_boxes)[(size_t)b * P.top_n + i] = box;
        out_scores[(size_t)b * P.top_n + i] = score;
    }
}

// ---------------------------------------------------------------------------------- pre-computed proposals (Fast R-CNN, FPN)
// preprocess_sample.py:37-47,61-69 followed by add_multilevel_rois_for_test and the roi_original_idx restore of forward(), per image:
// p = box * scale in fp32 (numpy multiplies the float32 roidb boxes by the Python-float scale in float32), the hash of the rounded
// p / 16, np.unique(return_index=True) -- ascending hash, first occurrence of each -- and the FPN level of each surviving p.
// numpy sums r0*1e3 + r1*1e6 + r2*1e9 + r3*1e12 in float64, where every term and partial sum is an exact integer while |r| < 8998
// (the host rejects larger coordinates); an exact int64 key therefore has the same equalities and the same order.
struct FastPropsParams {
    const float* boxes;      // [B, top_n, 4] original-image coordinates
    const int* counts;       // [B]
    const float* im_info;    // per-image scaling factor (image_info), null = scaling_factor
    float scaling_factor;
    int top_n, k_min, k_max;
    float* rois;             // [B, top_n, 5] (batch idx, x1,y1,x2,y2) in hash order; rows >= count are (b, 0, 0, 0, 0) as collect_kernel leaves them
    int* levels;             // [B, top_n] level index (lvl - k_min)
    int* roi_counts;         // [B] number of distinct hashes
};

// grid B, 1024 threads, dynamic shared memory top_n * 9 bytes.  At most ~1000 boxes per image: the stable sort is a rank count over
// shared memory (the rank of a first occurrence = the number of first occurrences with a smaller key).
static __global__ void __launch_bounds__(1024) fast_props_kernel(const __grid_constant__ FastPropsParams P) {
    extern __shared__ long long keys[];                                        // [top_n]
    unsigned char* first = reinterpret_cast<unsigned char*>(keys + P.top_n);   // [top_n]
    const int b = blockIdx.x;
    const int n = min(max(P.counts[b], 0), P.top_n);
    const float scale = image_info(P.im_info, b, 1, 0, 0, P.scaling_factor).scale;
    const float* bx = P.boxes + (size_t)b * P.top_n * 4;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        long long k = 0, w = 1000;
#pragma unroll
        for (int c = 0; c < 4; ++c, w *= 1000) k += (long long)rintf(__fmul_rn(__fmul_rn(bx[i * 4 + c], scale), 0.0625f)) * w;
        keys[i] = k;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const long long k = keys[i];
        bool f = true;
        for (int j = 0; j < i && f; ++j) f = keys[j] != k;
        first[i] = f;
    }
    __syncthreads();
    int m = 0;
    for (int base = 0; base < n; base += blockDim.x) m += __syncthreads_count(base + threadIdx.x < n && first[base + threadIdx.x]);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (!first[i]) continue;
        const long long k = keys[i];
        int u = 0;
        for (int j = 0; j < n; ++j) u += first[j] & (keys[j] < k);
        const float4 p = make_float4(__fmul_rn(bx[i * 4 + 0], scale), __fmul_rn(bx[i * 4 + 1], scale), __fmul_rn(bx[i * 4 + 2], scale),
                                     __fmul_rn(bx[i * 4 + 3], scale));
        float* r = P.rois + ((size_t)b * P.top_n + u) * 5;
        r[0] = (float)b; r[1] = p.x; r[2] = p.y; r[3] = p.z; r[4] = p.w;
        P.levels[(size_t)b * P.top_n + u] = fpn_level(p, P.k_min, P.k_max) - P.k_min;
    }
    for (int i = m + threadIdx.x; i < P.top_n; i += blockDim.x) {
        float* r = P.rois + ((size_t)b * P.top_n + i) * 5;
        r[0] = (float)b; r[1] = r[2] = r[3] = r[4] = 0.f;
        P.levels[(size_t)b * P.top_n + i] = 0;
    }
    if (threadIdx.x == 0) P.roi_counts[b] = m;
}

// ---------------------------------------------------------------------------------- box head tail
// head [M, stride] with [0,NC) class logits and [NC, NC+4NC) box deltas -> cls_prob [M,NC] (softmax), bbox [M,4NC]
// one warp per row
static __global__ void softmax_split_kernel(const float* __restrict__ head, int M, int stride, int NC, int do_softmax,
                                     float* __restrict__ cls, float* __restrict__ bbox) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const float* h = head + (size_t)row * stride;
    float mx = -INFINITY;
    for (int c = lane; c < NC; c += 32) mx = fmaxf(mx, h[c]);
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int c = lane; c < NC; c += 32) sum += expf(h[c] - mx);
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    for (int c = lane; c < NC; c += 32) cls[(size_t)row * NC + c] = do_softmax ? __fdiv_rn(expf(h[c] - mx), sum) : h[c];
    for (int c = lane; c < 4 * NC; c += 32) bbox[(size_t)row * 4 * NC + c] = h[NC + c];
}

// ---------------------------------------------------------------------------------- detection post-processing
struct DetParams {
    const float* rois;        // [B, R, 5] image-scale RoIs (col 0 = batch)
    const int* roi_counts;    // [B] (null -> R)
    const float* cls;         // [B*R, NC]
    const float* bbox;        // [B*R, 4*NC]
    int B, R, NC;
    float scaling_factor, im_h, im_w;      // original image size = network size / scaling_factor
    const float* im_info;                  // per-image scale and original size (image_info), null = the scalars above
    float wx, wy, ww, wh;                  // bbox_reg_weights (10,10,5,5)
    float score_thresh, nms_thresh;
    int max_dets, out_cap;                 // 100, and the padded capacity of the outputs (>= max_dets)
    // per (image, class) scratch: kept flags over RoIs, decoded boxes
    unsigned char* keep_flag;   // [B, NC, R]
    float4* dec_box;            // [B, NC, R]
    int* cls_counts;            // [B, NC]
    // sort scratch for the limit step
    uint32_t *k0, *k1;          // [B, NC*R]
    int *v0, *v1;
    // outputs, class-major then ascending RoI index (result_utils.py:165-168)
    float* out_boxes;           // [B, out_cap, 4]
    float* out_scores;          // [B, out_cap]
    int* out_classes;           // [B, out_cap]
    int* out_roi_idx;           // [B, out_cap]
    int* out_counts;            // [B] rows written, <= out_cap
    int* out_total;             // [B] the reference's count: more than out_counts when ties at the limit overflow out_cap
};

// grid (NC-1, B), 256 threads; one CTA = one (image, foreground class).  R <= 1024.
static __global__ void __launch_bounds__(256) det_class_kernel(const __grid_constant__ DetParams P) {
    __shared__ unsigned long long skey[1024];       // (score desc, roi idx asc) sort keys
    __shared__ float4 sbox[1024];
    __shared__ NmsSmem nsm;
    __shared__ unsigned long long removed[16];
    __shared__ int scratch[33];
    const int j = blockIdx.x + 1, b = blockIdx.y;
    const int R = P.roi_counts ? min(P.roi_counts[b], P.R) : P.R;
    const ImageInfo img = image_info(P.im_info, b, 1, 0, 0, P.scaling_factor, P.im_h, P.im_w);
    unsigned char* flag = P.keep_flag + ((size_t)b * P.NC + j) * P.R;
    float4* dbox = P.dec_box + ((size_t)b * P.NC + j) * P.R;
    // candidates: score > thresh (strict, result_utils.py:127), ascending RoI order
    int nc = 0;
    for (int base = 0; base < P.R; base += blockDim.x) {
        const int i = base + threadIdx.x;
        float sc = 0.f;
        bool c = false;
        if (i < R) { sc = P.cls[((size_t)b * P.R + i) * P.NC + j]; c = sc > P.score_thresh; }
        if (i < P.R) flag[i] = 0;
        int tot;
        const int r = block_rank(c, scratch, &tot);
        if (c) {
            // ascending radix order of the 64-bit key == (score desc, idx asc)
            skey[nc + r] = ((unsigned long long)float_desc_key(sc) << 32) | (unsigned)i;
        }
        nc += tot;
    }
    __syncthreads();
    if (nc == 0) { if (threadIdx.x == 0) P.cls_counts[b * P.NC + j] = 0; return; }
    // bitonic sort of nc keys padded to a power of two
    int np2 = 1; while (np2 < nc) np2 <<= 1;
    for (int i = nc + threadIdx.x; i < np2; i += blockDim.x) skey[i] = ~0ull;
    __syncthreads();
    for (int k = 2; k <= np2; k <<= 1) {
        for (int s = k >> 1; s > 0; s >>= 1) {
            for (int i = threadIdx.x; i < np2; i += blockDim.x) {
                const int p = i ^ s;
                if (p > i) {
                    const unsigned long long a = skey[i], c = skey[p];
                    const bool up = ((i & k) == 0);
                    if ((a > c) == up) { skey[i] = c; skey[p] = a; }
                }
            }
            __syncthreads();
        }
    }
    // decode + clip the candidates of this class (boxes.py:168-208,150-165), sorted order
    for (int i = threadIdx.x; i < nc; i += blockDim.x) {
        const int ri = (int)(skey[i] & 0xffffffffu);
        const float* r = P.rois + ((size_t)b * P.R + ri) * 5;
        const float4 box = make_float4(__fdiv_rn(r[1], img.scale), __fdiv_rn(r[2], img.scale), __fdiv_rn(r[3], img.scale),
                                       __fdiv_rn(r[4], img.scale));
        const float* d = P.bbox + ((size_t)b * P.R + ri) * 4 * P.NC + 4 * j;
        float4 o = decode_box(box, __fdiv_rn(d[0], P.wx), __fdiv_rn(d[1], P.wy), __fdiv_rn(d[2], P.ww), __fdiv_rn(d[3], P.wh));
        o = clip_box(o, img.orig_w - 1.f, img.orig_h - 1.f);
        sbox[i] = o;
        dbox[ri] = o;
    }
    __syncthreads();
    const int kept = block_nms_sorted(sbox, nc, P.nms_thresh, removed, &nsm);
    for (int i = threadIdx.x; i < nc; i += blockDim.x)
        if (!((removed[i >> 6] >> (i & 63)) & 1ull)) flag[(int)(skey[i] & 0xffffffffu)] = 1;
    if (threadIdx.x == 0) P.cls_counts[b * P.NC + j] = kept;
}

// grid B, 1024 threads: limit to max_dets over all classes (result_utils.py:152-168) and emit.
// The kept flags of a class are swept by ONE WARP (ballot + popc over 32 RoIs at a time, no block barriers): class counts -> exclusive
// class offsets -> ordered writes.  Two such sweeps (gather keys, emit) replace two block-wide scans of the NC*R flags (79 iterations x 3
// __syncthreads each).  Order and arithmetic are unchanged: class-major, ascending RoI index.
// The reference keeps every detection scoring >= the max_dets-th largest score, so ties at that score can make more than max_dets,
// and more than out_cap.  Then every detection scoring above the threshold is written (there are fewer than max_dets <= out_cap of
// them), the remaining rows take the tied ones in class-major, RoI-ascending order, and out_total holds the reference's count.
static __global__ void __launch_bounds__(1024) det_limit_kernel(const __grid_constant__ DetParams P) {
    __shared__ uint32_t hist[32 * 256];
    __shared__ int cls_cnt[128], cls_off[129], cls_tie[128];
    __shared__ float s_thresh;
    const int b = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const size_t cap = (size_t)P.NC * P.R;
    uint32_t* k0 = P.k0 + b * cap; uint32_t* k1 = P.k1 + b * cap;
    int* v0 = P.v0 + b * cap; int* v1 = P.v1 + b * cap;
    const unsigned char* flag = P.keep_flag + (size_t)b * P.NC * P.R;
    const unsigned lt = (1u << lane) - 1u;
    // exclusive offsets of the classes from per-class counts (class 0 = background: empty); returns the total
    auto scan_classes = [&]() {
        __syncthreads();
        if (threadIdx.x == 0) {
            int o = 0;
            for (int j = 0; j < P.NC; ++j) { cls_off[j] = o; o += cls_cnt[j]; }
            cls_off[P.NC] = o;
        }
        __syncthreads();
        return cls_off[P.NC];
    };
    // sweep 1: kept per class
    if (threadIdx.x < 128) { cls_cnt[threadIdx.x] = 0; cls_tie[threadIdx.x] = 0; }
    __syncthreads();
    for (int j = 1 + warp; j < P.NC; j += nwarps) {
        int c = 0;
#pragma unroll 8
        for (int base = 0; base < P.R; base += 32) {
            const int ri = base + lane;
            c += __popc(__ballot_sync(0xffffffffu, ri < P.R && flag[(size_t)j * P.R + ri]));
        }
        if (lane == 0) cls_cnt[j] = c;
    }
    const int n = scan_classes();
    float thresh = -INFINITY;
    if (P.max_dets > 0 && n > P.max_dets) {
        // image_thresh = np.sort(image_scores)[-max_dets]  == max_dets-th largest: gather the kept scores (class-major, RoI ascending), sort
        for (int j = 1 + warp; j < P.NC; j += nwarps) {
            int o = cls_off[j];
    #pragma unroll 8
        for (int base = 0; base < P.R; base += 32) {
                const int ri = base + lane;
                const bool f = ri < P.R && flag[(size_t)j * P.R + ri];
                const unsigned m = __ballot_sync(0xffffffffu, f);
                if (f) {
                    const int pos = o + __popc(m & lt);
                    k0[pos] = float_desc_key(P.cls[((size_t)b * P.R + ri) * P.NC + j]);
                    v0[pos] = j * P.R + ri;
                }
                o += __popc(m);
            }
        }
        __syncthreads();
        block_radix_sort_asc_u32(k0, v0, k1, v1, n, hist);
        if (threadIdx.x == 0) {
            const int i = v0[P.max_dets - 1];
            const int j = i / P.R, ri = i - j * P.R;
            s_thresh = P.cls[((size_t)b * P.R + ri) * P.NC + j];
        }
        __syncthreads();
        thresh = s_thresh;
        // sweep 2: per class, how many of the kept pass score >= thresh (:162), and how many of those tie at it
        __syncthreads();
        for (int j = 1 + warp; j < P.NC; j += nwarps) {
            int c = 0, t = 0;
    #pragma unroll 8
        for (int base = 0; base < P.R; base += 32) {
                const int ri = base + lane;
                const bool f = ri < P.R && flag[(size_t)j * P.R + ri];
                const float sc = f ? P.cls[((size_t)b * P.R + ri) * P.NC + j] : 0.f;
                c += __popc(__ballot_sync(0xffffffffu, f && sc >= thresh));
                t += __popc(__ballot_sync(0xffffffffu, f && sc == thresh));
            }
            if (lane == 0) { cls_cnt[j] = c; cls_tie[j] = t; }
        }
    }
    int nout = scan_classes();
    const int total = nout;
    const bool cut_ties = nout > P.out_cap && thresh > -INFINITY;
    if (cut_ties) {
        // the ties overflow out_cap: all above-threshold detections, then cls_tie[j] becomes the number of class j's ties written
        if (threadIdx.x == 0) {
            int room = P.out_cap;
            for (int j = 1; j < P.NC; ++j) room -= cls_cnt[j] - cls_tie[j];
            for (int j = 1; j < P.NC; ++j) {
                const int t = min(cls_tie[j], room);
                room -= t;
                cls_cnt[j] += t - cls_tie[j];
                cls_tie[j] = t;
            }
        }
        nout = scan_classes();
    }
    // emit in class-major / RoI-ascending order
    for (int j = 1 + warp; j < P.NC; j += nwarps) {
        int o = cls_off[j], ties = 0;
        const int tie_room = cls_tie[j];
#pragma unroll 8
        for (int base = 0; base < P.R; base += 32) {
            const int ri = base + lane;
            bool f = ri < P.R && flag[(size_t)j * P.R + ri];
            float sc = 0.f;
            if (f) { sc = P.cls[((size_t)b * P.R + ri) * P.NC + j]; f = sc >= thresh; }
            if (cut_ties) {
                const bool tie = f && sc == thresh;
                const unsigned mt = __ballot_sync(0xffffffffu, tie);
                if (tie) f = ties + __popc(mt & lt) < tie_room;
                ties += __popc(mt);
            }
            const unsigned m = __ballot_sync(0xffffffffu, f);
            const int pos = o + __popc(m & lt);
            if (f && pos < P.out_cap) {
                const float4 bx = P.dec_box[((size_t)b * P.NC + j) * P.R + ri];
                float* ob = P.out_boxes + ((size_t)b * P.out_cap + pos) * 4;
                ob[0] = bx.x; ob[1] = bx.y; ob[2] = bx.z; ob[3] = bx.w;
                P.out_scores[(size_t)b * P.out_cap + pos] = sc;
                P.out_classes[(size_t)b * P.out_cap + pos] = j;
                P.out_roi_idx[(size_t)b * P.out_cap + pos] = ri;
            }
            o += __popc(m);
        }
    }
    for (int i = min(nout, P.out_cap) + threadIdx.x; i < P.out_cap; i += blockDim.x) {
        float* ob = P.out_boxes + ((size_t)b * P.out_cap + i) * 4;
        ob[0] = ob[1] = ob[2] = ob[3] = 0.f;
        P.out_scores[(size_t)b * P.out_cap + i] = 0.f;
        P.out_classes[(size_t)b * P.out_cap + i] = 0;
        P.out_roi_idx[(size_t)b * P.out_cap + i] = -1;
    }
    if (threadIdx.x == 0) { P.out_counts[b] = min(nout, P.out_cap); P.out_total[b] = total; }
}

// detections -> mask RoIs: boxes_final * scaling_factor, FPN level (eval_mask_FPN.ipynb cell 10; multilevel_rois.py:19-39).
// im_info (may be null): image b's own scaling factor (image_info)
static __global__ void mask_rois_kernel(const float* __restrict__ boxes, const int* __restrict__ counts, int B, int cap, float scaling_factor,
                                 int k_min, int k_max, float* __restrict__ rois5, int* __restrict__ levels, const float* __restrict__ im_info) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * cap) return;
    const int b = i / cap, d = i - b * cap;
    float* r = rois5 + (size_t)i * 5;
    r[0] = (float)b;
    if (d < counts[b]) {
        scaling_factor = image_info(im_info, b, 1, 0, 0, scaling_factor).scale;
        const float* s = boxes + (size_t)i * 4;
        const float4 box = make_float4(__fmul_rn(s[0], scaling_factor), __fmul_rn(s[1], scaling_factor), __fmul_rn(s[2], scaling_factor),
                                       __fmul_rn(s[3], scaling_factor));
        r[1] = box.x; r[2] = box.y; r[3] = box.z; r[4] = box.w;
        levels[i] = fpn_level(box, k_min, k_max) - k_min;
    } else {
        r[1] = r[2] = r[3] = r[4] = 0.f;
        levels[i] = 0;
    }
}

// mask logits NHWC [D, S, S, stride] -> per-detection mask of its own class [D, S, S] (+sigmoid), and optionally
// the full public tensor [D, NC, S, S]
static __global__ void mask_select_kernel(const float* __restrict__ logits, const int* __restrict__ classes, int D, int S, int stride, int NC,
                                   int apply_sigmoid, float* __restrict__ sel, float* __restrict__ full) {
    const long long total = (long long)D * S * S;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int d = (int)(i / (S * S));
        const int p = (int)(i - (long long)d * S * S);
        const float* src = logits + ((size_t)d * S * S + p) * stride;
        if (sel) {
            const int c = classes ? classes[d] : 0;
            float v = src[c];
            if (apply_sigmoid) v = 1.f / (1.f + expf(-v));
            sel[i] = v;
        }
        if (full) {
            for (int c = 0; c < NC; ++c) {
                float v = src[c];
                if (apply_sigmoid) v = 1.f / (1.f + expf(-v));
                full[((size_t)d * NC + c) * S * S + p] = v;
            }
        }
    }
}

}  // namespace dt

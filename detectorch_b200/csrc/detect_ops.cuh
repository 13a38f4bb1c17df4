// detectorch_b200 -- the non-GEMM device stages of the detector, all on-device and sync-free:
//   stem im2col, maxpool, P6 subsample                      (torchvision trunk glue, detector.py:183,250)
//   rpn_proposals_kernel   top-k + decode + clip + filter + NMS(0.7)   generate_proposals.py:31-122
//   collect_kernel         merge levels, top-N, FPN level map           collect_and_distribute...py:84-128,
//                                                                       multilevel_rois.py:41-53
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

// ---------------------------------------------------------------------------------- stem im2col
// image NCHW [B,3,H,W] -> col [B*Ho*Wo, 160], k = c*49 + ky*7 + kx (torch weight order), k >= 147 zero.
// 7x7 stride 2 pad 3 (torchvision resnet conv1).
static __global__ void stem_im2col_kernel(const float* __restrict__ img, int B, int H, int W, int Ho, int Wo, float* __restrict__ col) {
    const long long total = (long long)B * Ho * Wo * 40;   // float4 granules
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k4 = (int)(i % 40);
        long long m = i / 40;
        const int wo = (int)(m % Wo); m /= Wo;
        const int ho = (int)(m % Ho);
        const int b = (int)(m / Ho);
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k4 * 4 + j;
            float x = 0.f;
            if (k < 147) {
                const int c = k / 49, r = k - c * 49, ky = r / 7, kx = r - ky * 7;
                const int y = ho * 2 - 3 + ky, xx = wo * 2 - 3 + kx;
                if (y >= 0 && y < H && xx >= 0 && xx < W) x = __ldg(img + (((size_t)b * 3 + c) * H + y) * W + xx);
            }
            v[j] = x;
        }
        reinterpret_cast<float4*>(col)[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// image NCHW [B,3,H,W] -> zero-bordered NHWC4 [B,Hp,Wp,4] (3-pixel border = the conv1 padding; channel 3 = 0)
static __global__ void stem_pack_nhwc4_kernel(const float* __restrict__ img, int B, int H, int W, int Hp, int Wp, float* __restrict__ x4) {
    const long long total = (long long)B * Hp * Wp;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int xp = (int)(i % Wp);
        const int yp = (int)((i / Wp) % Hp);
        const int b = (int)(i / ((long long)Wp * Hp));
        const int x = xp - 3, y = yp - 3;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x >= 0 && x < W && y >= 0 && y < H) {
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
                                                     uint2* __restrict__ xl, int* __restrict__ range_flag) {
    const long long total = (long long)B * Hp * Wp;
    bool bad = false;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int xp = (int)(i % Wp);
        const int yp = (int)((i / Wp) % Hp);
        const int b = (int)(i / ((long long)Wp * Hp));
        const int x = xp - 3, y = yp - 3;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x >= 0 && x < W && y >= 0 && y < H) {
            const size_t o = ((size_t)b * 3 * H + y) * W + x;
            v.x = __ldg(img + o); v.y = __ldg(img + o + (size_t)H * W); v.z = __ldg(img + o + 2 * (size_t)H * W);
        }
        uint2 h, l;
        split_planes4(v, &h, &l, &bad);
        xh[i] = h; xl[i] = l;
    }
    if (bad && range_flag) *range_flag = 1;
}

// NHWC 3x3 stride-2 pad-1 max pool (torchvision maxpool); PLANES: the result leaves as two fp16 planes (hi, lo) for plane-input convs
template <bool PLANES>
static __global__ void maxpool3x3s2_nhwc_kernel(const float* __restrict__ x, int B, int H, int W, int C, int Ho, int Wo, float* __restrict__ y,
                                                int* __restrict__ range_flag) {
    const int C4 = C >> 2;
    const long long total = (long long)B * Ho * Wo * C4;
    bool bad = false;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        long long m = i / C4;
        const int wo = (int)(m % Wo); m /= Wo;
        const int ho = (int)(m % Ho);
        const int b = (int)(m / Ho);
        float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int dy = 0; dy < 3; ++dy) {
            const int yy = ho * 2 - 1 + dy;
            if (yy < 0 || yy >= H) continue;
            for (int dx = 0; dx < 3; ++dx) {
                const int xx = wo * 2 - 1 + dx;
                if (xx < 0 || xx >= W) continue;
                const float4 v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)b * H + yy) * W + xx) * C) + c4);
                best.x = fmaxf(best.x, v.x); best.y = fmaxf(best.y, v.y); best.z = fmaxf(best.z, v.z); best.w = fmaxf(best.w, v.w);
            }
        }
        if constexpr (PLANES) {
            uint2 h, l;
            split_planes4(best, &h, &l, &bad);
            reinterpret_cast<uint2*>(y)[i] = h;
            reinterpret_cast<uint2*>(y)[total + i] = l;       // the low plane follows the high plane (ProgBuilder::conv, planes_in)
        } else {
            reinterpret_cast<float4*>(y)[i] = best;
        }
    }
    if (PLANES && bad && range_flag) *range_flag = 1;
}

// P6 = max_pool2d(P5, kernel 1, stride 2) == stride-2 subsample (detector.py:250)
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

// exclusive prefix of a per-thread count over the block (all threads must call); *total receives the block total.  scratch: 33 ints
__device__ __forceinline__ int block_rank_count(int cnt, int* scratch, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    __syncthreads();
    if (lane == 31) scratch[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const int x = lane < nw ? scratch[lane] : 0;
        int w = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
        scratch[lane] = w - x;
        if (lane == 31) scratch[32] = w;
    }
    __syncthreads();
    *total = scratch[32];
    return scratch[warp] + incl - cnt;
}

// block-wide ordered compaction helper: returns the exclusive rank of `flag` among threads of this block
// sweep (all threads must call); *total receives the block total.  scratch: 33 ints of shared memory.
__device__ __forceinline__ int block_rank(bool flag, int* scratch, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const unsigned b = __ballot_sync(0xffffffffu, flag);
    __syncthreads();
    if (lane == 0) scratch[warp] = __popc(b);
    __syncthreads();
    if (warp == 0) {
        int v = lane < nw ? scratch[lane] : 0, inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        scratch[lane] = inc - v;
        if (lane == 31) scratch[32] = inc;
    }
    __syncthreads();
    *total = scratch[32];
    return scratch[warp] + __popc(b & ((1u << lane) - 1u));
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
    int* sel_chunk_counts;   // [B, L, kRpnMaxChunks]
    int* sel_info;           // [B, L, 4]: b1, b2, total (-1: not narrowed -> full sort), unused
    int split;               // 1: selection done by the multi-CTA kernels, rpn_proposals_kernel only finishes
    // NMS at full-GPU width (rpn_nms_mask_kernel + rpn_nms_scan_kernel): rpn_proposals_kernel then stops after decode / filter
    int nms_split;
    int nms_chunks;          // ceil(pre_nms / 64)
    int* cand_counts;        // [B, L] candidates that passed the filter
    unsigned long long* nms_mask;   // [B, L, pre_nms, nms_chunks]: bit b of word (i, w) set <=> candidate i suppresses candidate w*64 + b (> i)
};
static constexpr int kRpnChunk = 4096;        // anchors per CTA of the selection kernels (1024 threads x 4)
static constexpr int kRpnMaxChunks = 64;      // >= ceil(largest level / kRpnChunk): 182 400 / 4096 = 45 at 800x1216; levels above this use the one-CTA path

__host__ __device__ __forceinline__ bool rpn_level_selects(int n, int K) { return n > 4 * K && n > 8192; }

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
    const int n = lv.n, i0 = blockIdx.x * kRpnChunk;
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
        if (valid[j]) { const int a = i % lv.A, cell = i / lv.A; k[j] = float_desc_key(base[(size_t)cell * lv.ch_stride + a]); }
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
    const int n = lv.n, i0 = blockIdx.x * kRpnChunk;
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
    const int n = lv.n, i0 = blockIdx.x * kRpnChunk;
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
    if (threadIdx.x == 0) P.sel_chunk_counts[((size_t)b * P.num_levels + l) * kRpnMaxChunks + blockIdx.x] = tot;
}

// ---- selection pass 4: ordered compaction (ascending anchor index, like the one-CTA path) into (k1, v1)
static __global__ void __launch_bounds__(1024) rpn_select_scatter_kernel(const __grid_constant__ RpnParams P) {
    __shared__ int scratch[33];
    __shared__ int offset;
    const int l = blockIdx.y, b = blockIdx.z;
    const RpnLevel& lv = P.lv[l];
    const int n = lv.n, i0 = blockIdx.x * kRpnChunk;
    if (i0 >= n) return;
    const int K = (P.pre_nms <= 0 || P.pre_nms >= n) ? n : P.pre_nms;
    if (!rpn_level_selects(n, K)) return;
    const int* info = P.sel_info + ((size_t)b * P.num_levels + l) * 4;
    if (info[2] < 0) return;
    const uint32_t b1 = (uint32_t)info[0], b2 = (uint32_t)info[1];
    if (threadIdx.x == 0) {
        const int* cc = P.sel_chunk_counts + ((size_t)b * P.num_levels + l) * kRpnMaxChunks;
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
    __shared__ __align__(16) uint32_t hist[32 * 256];
    __shared__ NmsSmem nsm;
    __shared__ unsigned long long removed[128];   // up to 8192 candidates
    __shared__ int scratch[33];
    const int l = blockIdx.x, b = blockIdx.y;
    const RpnLevel& lv = P.lv[l];
    const int n = lv.n;
    uint32_t* k0 = P.k0 + (size_t)b * P.ws_per_image + lv.ws_off;
    uint32_t* k1 = P.k1 + (size_t)b * P.ws_per_image + lv.ws_off;
    int* v0 = P.v0 + (size_t)b * P.ws_per_image + lv.ws_off;
    int* v1 = P.v1 + (size_t)b * P.ws_per_image + lv.ws_off;
    const float* base = lv.rpn_out + (size_t)b * lv.H * lv.W * lv.ch_stride;
    // 1. keys in (H,W,A) order (generate_proposals.py:64,72)
    // 2. top-K by descending score (:77-86).  A full sort of ~180k keys by one CTA costs >1 ms, so first narrow the set
    //    with a two-level 11+11-bit radix select on the key (exact: every key below the boundary sub-bin plus the whole
    //    boundary sub-bin is kept, in index order), then stable-sort only those candidates.
    //    The passes over the level are latency-bound (one CTA): every thread keeps 4 independent loads in flight.
    const int K = (P.pre_nms <= 0 || P.pre_nms >= n) ? n : P.pre_nms;
    const int* vs = v0;                 // sorted anchor indices end up here
    bool narrowed = false;
    // P.split: the keys, the two-level radix select and the ordered compaction were done at full-GPU width by rpn_select_*_kernel
    // (one CTA per 4096 anchors instead of one CTA per level: the 182 400-anchor P2 level was the long pole of this kernel); (k1, v1)
    // hold the `total` selected (key, index) pairs in ascending index order, (k0, v0) all keys.  What remains is per (level, image).
    if (P.split && n <= kRpnChunk * kRpnMaxChunks) {
        if (rpn_level_selects(n, K)) {
            const int total = P.sel_info[((size_t)b * P.num_levels + l) * 4 + 2];
            if (total >= 0) {
                block_radix_sort_asc_u32(k1, v1, k0, v0, total, hist);
                vs = v1;
                narrowed = true;
            }
        }
    } else {
        const bool select = n > 4 * K && n > 8192;
        uint32_t* h1 = hist;                // 2048 bins
        uint32_t* h2 = hist + 2048;         // 2048 bins
        __shared__ uint32_t sel[4];         // b1, c1, b2, count
        if (select) {
            for (int i = threadIdx.x; i < 4096; i += blockDim.x) hist[i] = 0;
            __syncthreads();
        }
        for (int base_i = 0; base_i < n; base_i += 4 * blockDim.x) {
            uint32_t k[4];
            bool valid[4];
    #pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = base_i + j * blockDim.x + threadIdx.x;
                valid[j] = i < n;
                k[j] = 0u;
                if (valid[j]) {
                    const int a = i % lv.A, cell = i / lv.A;
                    k[j] = float_desc_key(base[(size_t)cell * lv.ch_stride + a]);
                }
            }
    #pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = base_i + j * blockDim.x + threadIdx.x;
                if (valid[j]) { k0[i] = k[j]; v0[i] = i; }
                if (select) {
                    // objectness scores cluster in a few exponent bins: aggregate equal digits inside the warp before touching shared memory
                    const unsigned act = __ballot_sync(0xffffffffu, valid[j]);
                    if (valid[j]) {
                        const uint32_t d = k[j] >> 21;
                        const unsigned m = __match_any_sync(act, d);
                        if ((m & ((1u << (threadIdx.x & 31)) - 1u)) == 0) atomicAdd(&h1[d], (uint32_t)__popc(m));
                    }
                }
            }
        }
        __syncthreads();
        // first bin b with c + h[b] >= K (c = keys in the bins before it), by warp 0: 64 bins per lane, warp prefix, serial scan of one lane's bins
        auto find_bin = [&](const uint32_t* h, uint32_t c0, uint32_t* out_bin, uint32_t* out_c) {
            if (threadIdx.x < 32) {
                const int lane = threadIdx.x;
                uint32_t sum = 0;
                for (int t = 0; t < 64; ++t) sum += h[lane * 64 + t];
                uint32_t incl = sum;
    #pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
                const uint32_t excl = c0 + incl - sum;
                const bool hit = excl + sum >= (uint32_t)K;            // the crossing lies in or before this lane's bins
                const unsigned hits = __ballot_sync(0xffffffffu, hit);
                if (hits == 0) { if (lane == 0) { *out_bin = 2048; *out_c = c0 + __shfl_sync(0xffffffffu, incl, 31); } }
                else if (lane == __ffs(hits) - 1) {
                    uint32_t c = excl, bb = (uint32_t)lane * 64;
                    for (; bb < (uint32_t)lane * 64 + 64; ++bb) { if (c + h[bb] >= (uint32_t)K) break; c += h[bb]; }
                    *out_bin = bb; *out_c = c;
                }
            }
        };
        if (select) {
            find_bin(h1, 0u, &sel[0], &sel[1]);
            __syncthreads();
            const uint32_t b1 = sel[0], c1 = sel[1];
            for (int base_i = 0; base_i < n; base_i += 4 * blockDim.x) {
                uint32_t k[4];
    #pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = base_i + j * blockDim.x + threadIdx.x;
                    k[j] = i < n ? k0[i] : 0xffffffffu;
                }
    #pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = base_i + j * blockDim.x + threadIdx.x;
                    const bool valid = (i < n) && ((k[j] >> 21) == b1);
                    const unsigned act = __ballot_sync(0xffffffffu, valid);
                    if (valid) {
                        const uint32_t d = (k[j] >> 10) & 2047u;
                        const unsigned m = __match_any_sync(act, d);
                        if ((m & ((1u << (threadIdx.x & 31)) - 1u)) == 0) atomicAdd(&h2[d], (uint32_t)__popc(m));
                    }
                }
            }
            __syncthreads();
            find_bin(h2, c1, &sel[2], &sel[3]);
            __syncthreads();
            if (threadIdx.x == 0 && sel[2] < 2048u) sel[3] += h2[sel[2]];
            __syncthreads();
            const uint32_t b2 = sel[2], total = sel[3];
            if (total <= 8192u) {
                // ordered compaction: a thread owns 4 consecutive indices, one block scan per 4096 keys
                int m = 0;
                for (int base_i = 0; base_i < n; base_i += 4 * blockDim.x) {
                    const int i0 = base_i + 4 * threadIdx.x;
                    uint32_t k[4];
                    bool f[4];
                    int cnt = 0;
    #pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int i = i0 + j;
                        k[j] = i < n ? k0[i] : 0xffffffffu;
                    }
    #pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t d1 = k[j] >> 21;
                        f[j] = (i0 + j < n) && ((d1 < b1) || (d1 == b1 && ((k[j] >> 10) & 2047u) <= b2));
                        cnt += f[j] ? 1 : 0;
                    }
                    int tot;
                    int r = m + block_rank_count(cnt, scratch, &tot);
    #pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (f[j]) { k1[r] = k[j]; v1[r] = i0 + j; ++r; }
                    m += tot;
                }
                __syncthreads();
                block_radix_sort_asc_u32(k1, v1, k0, v0, m, hist);
                vs = v1;
                narrowed = true;
            }
        }
    }
    if (!narrowed) block_radix_sort_asc_u32(k0, v0, k1, v1, n, hist);
    // 3. decode + clip + filter on the top K (:96-112), order preserved
    float4* cand = P.cand + ((size_t)b * P.num_levels + l) * P.pre_nms;
    float* cscore = P.cand_score + ((size_t)b * P.num_levels + l) * P.pre_nms;
    int nc = 0;
    const float min_size = P.min_size * P.scaling_factor;
    for (int base_i = 0; base_i < K; base_i += blockDim.x) {
        const int i = base_i + threadIdx.x;
        bool keep = false;
        float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
        float sc = 0.f;
        if (i < K) {
            const int idx = vs[i];
            if (P.dbg_order) P.dbg_order[((size_t)b * P.num_levels + l) * P.pre_nms + i] = idx;
            const int a = idx % lv.A, cell = idx / lv.A;
            const int x = cell % lv.W, y = cell / lv.W;
            const float sx = (float)x * lv.stride, sy = (float)y * lv.stride;
            const float4 anc = make_float4(lv.anchors[a * 4 + 0] + sx, lv.anchors[a * 4 + 1] + sy, lv.anchors[a * 4 + 2] + sx,
                                           lv.anchors[a * 4 + 3] + sy);
            const float* d = base + (size_t)cell * lv.ch_stride + lv.A + a * 4;
            sc = base[(size_t)cell * lv.ch_stride + a];
            box = clip_box(decode_box(anc, d[0], d[1], d[2], d[3]), P.im_w - 1.f, P.im_h - 1.f);
            // filter_boxes (:151-163)
            const float ws = __fadd_rn(__fsub_rn(box.z, box.x), 1.f), hs = __fadd_rn(__fsub_rn(box.w, box.y), 1.f);
            const float xc = __fadd_rn(box.x, __fdiv_rn(ws, 2.f)), yc = __fadd_rn(box.y, __fdiv_rn(hs, 2.f));
            keep = (ws >= min_size) && (hs >= min_size) && (xc < P.im_w) && (yc < P.im_h);
        }
        int tot;
        const int r = block_rank(keep, scratch, &tot);
        if (keep) { cand[nc + r] = box; cscore[nc + r] = sc; }
        nc += tot;
    }
    __syncthreads();
    if (P.nms_split && P.nms_thresh > 0.f) {
        // the greedy NMS of the <= pre_nms candidates continues in rpn_nms_mask_kernel (all pair tests, every SM) and
        // rpn_nms_scan_kernel (the sequential survivor walk): in this CTA the per-box sweep over the survivors was 45 % of the kernel
        if (threadIdx.x == 0) P.cand_counts[b * P.num_levels + l] = nc;
        return;
    }
    // 4. NMS (:114-120); candidates are already in descending-score order
    float* op = P.out_props + ((size_t)b * P.num_levels + l) * P.post_nms * 4;
    float* os = P.out_scores + ((size_t)b * P.num_levels + l) * P.post_nms;
    int nout = 0;
    if (P.nms_thresh > 0.f) {
        // the sort is over: its 32 KB histogram area holds up to 2048 candidate boxes, so the NMS reads them from shared memory
        // instead of paying an L2 round trip per chunk (the FPN levels have at most 1000 candidates; the C4 level's 6000 stay global)
        const float4* nms_boxes = cand;
        if (nc <= 2048) {
            float4* sb = reinterpret_cast<float4*>(hist);
            for (int i = threadIdx.x; i < nc; i += blockDim.x) sb[i] = cand[i];
            __syncthreads();
            nms_boxes = sb;
        }
        block_nms_sorted(nms_boxes, nc, P.nms_thresh, P.post_nms, removed, &nsm);
        for (int base_i = 0; base_i < nc; base_i += blockDim.x) {
            const int i = base_i + threadIdx.x;
            const bool keep = (i < nc) && !((removed[i >> 6] >> (i & 63)) & 1ull);
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
    } else {
        nout = min(nc, P.post_nms);
        for (int i = threadIdx.x; i < nout; i += blockDim.x) {
            const float4 bx = cand[i];
            op[i * 4 + 0] = bx.x; op[i * 4 + 1] = bx.y; op[i * 4 + 2] = bx.z; op[i * 4 + 3] = bx.w;
            os[i] = cscore[i];
        }
    }
    if (threadIdx.x == 0) P.out_counts[b * P.num_levels + l] = nout;
}

// ---- RPN NMS, part 1: the suppression bit-matrix of every (level, image), at full-GPU width.
// grid (chunks, chunks, L*B), 64 threads: block (bj, bi) with bj >= bi fills word (i, bj) for the 64 candidates i of chunk bi:
// bit b set <=> candidate i suppresses candidate bj*64 + b (only later candidates; cython_nms.pyx:76-85 semantics, iou_suppresses)
static __global__ void __launch_bounds__(64) rpn_nms_mask_kernel(const __grid_constant__ RpnParams P) {
    const int bj = blockIdx.x, bi = blockIdx.y, lb = blockIdx.z;      // lb = b * L + l
    if (bj < bi) return;
    const int n = P.cand_counts[lb];
    if (bi * 64 >= n || bj * 64 >= n) return;
    __shared__ float4 jb[64];
    __shared__ float ja[64];
    const float4* boxes = P.cand + (size_t)lb * P.pre_nms;
    const int j0 = bj * 64, i = bi * 64 + threadIdx.x;
    const int jn = min(64, n - j0);
    if ((int)threadIdx.x < jn) { const float4 bx = boxes[j0 + threadIdx.x]; jb[threadIdx.x] = bx; ja[threadIdx.x] = box_area_p1(bx); }
    __syncthreads();
    if (i >= n) return;
    const float4 me = boxes[i];
    const float ma = box_area_p1(me);
    unsigned long long bits = 0ull;
    for (int t = 0; t < jn; ++t)
        if (j0 + t > i && iou_suppresses(me, ma, jb[t], ja[t], P.nms_thresh)) bits |= 1ull << t;
    P.nms_mask[((size_t)lb * P.pre_nms + i) * P.nms_chunks + bj] = bits;
}

// ---- RPN NMS, part 2: the sequential survivor walk over the bit-matrix + the first post_nms survivors out (generate_proposals.py:114-120).
// grid (L, B), 1024 threads.
static __global__ void __launch_bounds__(1024) rpn_nms_scan_kernel(const __grid_constant__ RpnParams P) {
    __shared__ unsigned long long removed[128];   // up to 8192 candidates
    __shared__ unsigned long long diag[64];
    __shared__ int kept_list[64];
    __shared__ int kcount, total_kept;
    __shared__ int scratch[33];
    const int l = blockIdx.x, b = blockIdx.y, lb = b * P.num_levels + l;
    const int n = P.cand_counts[lb];
    const int nchunks = (n + 63) >> 6, NCH = P.nms_chunks;
    const unsigned long long* mask = P.nms_mask + (size_t)lb * P.pre_nms * NCH;
    for (int i = threadIdx.x; i < 128; i += blockDim.x) removed[i] = 0ull;
    if (threadIdx.x == 0) total_kept = 0;
    __syncthreads();
    for (int c = 0; c < nchunks; ++c) {
        const int cn = min(64, n - c * 64);
        if ((int)threadIdx.x < cn) diag[threadIdx.x] = mask[(size_t)(c * 64 + threadIdx.x) * NCH + c];
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned long long valid = (cn == 64) ? ~0ull : ((1ull << cn) - 1ull);
            unsigned long long alive = ~removed[c] & valid, kept = 0ull;
            int kc = 0, tot = total_kept;
            while (alive) {
                const int t = __ffsll((long long)alive) - 1;
                if (P.post_nms > 0 && tot >= P.post_nms) break;
                kept |= 1ull << t;
                kept_list[kc++] = c * 64 + t;
                ++tot;
                alive &= ~diag[t];
                alive &= ~(1ull << t);
            }
            removed[c] = ~kept;
            kcount = kc;
            total_kept = tot;
        }
        __syncthreads();
        if (P.post_nms > 0 && total_kept >= P.post_nms) {
            for (int i = c + 1 + threadIdx.x; i < nchunks; i += blockDim.x) removed[i] = ~0ull;
            __syncthreads();
            break;
        }
        // the survivors of this chunk suppress later candidates: OR their matrix rows into `removed`, one (survivor, word) pair per thread
        const int kc = kcount, words = nchunks - c - 1;
        for (int p = threadIdx.x; p < kc * words; p += blockDim.x) {
            const int k = p / words, wd = c + 1 + (p - k * words);
            const unsigned long long v = mask[(size_t)kept_list[k] * NCH + wd];
            if (v) atomicOr(&removed[wd], v);
        }
        __syncthreads();
    }
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
    int* out_counts;            // [B]
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
        const float4 box = make_float4(__fdiv_rn(r[1], P.scaling_factor), __fdiv_rn(r[2], P.scaling_factor),
                                       __fdiv_rn(r[3], P.scaling_factor), __fdiv_rn(r[4], P.scaling_factor));
        const float* d = P.bbox + ((size_t)b * P.R + ri) * 4 * P.NC + 4 * j;
        float4 o = decode_box(box, __fdiv_rn(d[0], P.wx), __fdiv_rn(d[1], P.wy), __fdiv_rn(d[2], P.ww), __fdiv_rn(d[3], P.wh));
        o = clip_box(o, P.im_w - 1.f, P.im_h - 1.f);
        sbox[i] = o;
        dbox[ri] = o;
    }
    __syncthreads();
    const int kept = block_nms_sorted(sbox, nc, P.nms_thresh, 0, removed, &nsm);
    for (int i = threadIdx.x; i < nc; i += blockDim.x)
        if (!((removed[i >> 6] >> (i & 63)) & 1ull)) flag[(int)(skey[i] & 0xffffffffu)] = 1;
    if (threadIdx.x == 0) P.cls_counts[b * P.NC + j] = kept;
}

// grid B, 1024 threads: limit to max_dets over all classes (result_utils.py:152-168) and emit.
// The kept flags of a class are swept by ONE WARP (ballot + popc over 32 RoIs at a time, no block barriers): class counts -> exclusive
// class offsets -> ordered writes.  Two such sweeps (gather keys, emit) replace two block-wide scans of the NC*R flags (79 iterations x 3
// __syncthreads each).  Order and arithmetic are unchanged: class-major, ascending RoI index.
static __global__ void __launch_bounds__(1024) det_limit_kernel(const __grid_constant__ DetParams P) {
    __shared__ uint32_t hist[32 * 256];
    __shared__ int cls_cnt[128], cls_off[129];
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
    if (threadIdx.x < 128) cls_cnt[threadIdx.x] = 0;
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
        // sweep 2: per class, how many of the kept pass score >= thresh (:162)
        __syncthreads();
        for (int j = 1 + warp; j < P.NC; j += nwarps) {
            int c = 0;
    #pragma unroll 8
        for (int base = 0; base < P.R; base += 32) {
                const int ri = base + lane;
                const bool f = ri < P.R && flag[(size_t)j * P.R + ri] && P.cls[((size_t)b * P.R + ri) * P.NC + j] >= thresh;
                c += __popc(__ballot_sync(0xffffffffu, f));
            }
            if (lane == 0) cls_cnt[j] = c;
        }
    }
    const int nout = scan_classes();
    // emit in class-major / RoI-ascending order
    for (int j = 1 + warp; j < P.NC; j += nwarps) {
        int o = cls_off[j];
#pragma unroll 8
        for (int base = 0; base < P.R; base += 32) {
            const int ri = base + lane;
            bool f = ri < P.R && flag[(size_t)j * P.R + ri];
            float sc = 0.f;
            if (f) { sc = P.cls[((size_t)b * P.R + ri) * P.NC + j]; f = sc >= thresh; }
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
    if (threadIdx.x == 0) P.out_counts[b] = min(nout, P.out_cap);
}

// detections -> mask RoIs: boxes_final * scaling_factor, FPN level (eval_mask_FPN.ipynb cell 10; multilevel_rois.py:19-39)
static __global__ void mask_rois_kernel(const float* __restrict__ boxes, const int* __restrict__ counts, int B, int cap, float scaling_factor,
                                 int k_min, int k_max, float* __restrict__ rois5, int* __restrict__ levels) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * cap) return;
    const int b = i / cap, d = i - b * cap;
    float* r = rois5 + (size_t)i * 5;
    r[0] = (float)b;
    if (d < counts[b]) {
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

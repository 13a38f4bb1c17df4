// detectorch_b200 -- proposal recall on the device: Detectron's evaluate_box_proposals (json_dataset_evaluator.py:238-320), the
// per-image part, bit for bit.
//
//   proposal_recall_kernel   one CTA per (image, (area range, limit) combination): the image's ground truth inside the area range
//                            (both bounds inclusive), its first `limit` proposals, and the greedy assignment of the reference's loop:
//                            min(P, G) rounds of "the best-covered GT column and the first proposal row that covers it best",
//                            after which that row and column read -1.  Each GT's recorded overlap goes out in round order, zeros
//                            after the last round.
//
// The IoU is cython_bbox.bbox_overlaps as its generated C computes it (+1.0 widths in double, float areas and union, the iw > 0 / ih > 0
// gates, iw * ih / ua in float), every operation an explicit _rn intrinsic: that C is compiled without contraction.  The matrix is never stored: each column keeps its max and
// first argmax over the live rows, and only the columns whose argmax was the retired row are recomputed (one warp per column).
// Retired rows count as -1 in a recompute and retired columns as -1 in the column choice, as the reference's overwritten matrix does.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace dt {

struct RecallParams {
    int num_images;
    const int64_t* prop_off;   // [I + 1] each image's first proposal
    const float4* props;       // [NP] proposals (x1, y1, x2, y2), float32
    const int64_t* gt_off;     // [I + 1] each image's first ground-truth box (gt_classes > 0, not crowd)
    const float4* gts;         // [NG]
    const double* gt_area;     // [NG] seg_areas
    const double* area_rng;    // [C, 2] inclusive area range per combination
    const int64_t* limits;     // [C] proposal limit per combination, < 0: none
    const int64_t* out_off;    // [C, I] first output of (combination, image); G outputs when the image has proposals
    double* out;               // recorded overlaps
    int* flag;                 // bit 0: a chosen overlap < 0 (the reference asserts), bit 1: ua == 0 (Cython raises ZeroDivisionError)
    int max_gts, row_words;    // shared-memory sizing: ground-truth boxes of the largest image, 32-bit words of its row mask
};

constexpr int kRecallThreads = 128;

__host__ __device__ inline size_t proposal_recall_smem(int max_gts, int row_words) {
    return (size_t)max_gts * (sizeof(float4) + 2 * sizeof(float) + sizeof(int)) + (size_t)row_words * sizeof(uint32_t);
}

// bbox_overlaps' (n, k) entry: boxes[n] against query_boxes[k].  The generated C adds the literal 1.0 in double: the widths are
// float differences + 1.0 in double, the areas and the union are double expressions rounded to float on assignment, iw * ih is a
// float product (Cython min / max: b < a ? b : a and b > a ? b : a)
__device__ __forceinline__ float recall_side(float hi, float lo) { return __double2float_rn(__dadd_rn((double)__fsub_rn(hi, lo), 1.0)); }
__device__ __forceinline__ double recall_area(float4 b) {
    return __dmul_rn(__dadd_rn((double)__fsub_rn(b.z, b.x), 1.0), __dadd_rn((double)__fsub_rn(b.w, b.y), 1.0));
}
__device__ __forceinline__ float recall_iou(float4 b, float4 q, float qarea, bool* zero_ua) {
    const float iw = recall_side(q.z < b.z ? q.z : b.z, q.x > b.x ? q.x : b.x);
    if (!(iw > 0.f)) return 0.f;
    const float ih = recall_side(q.w < b.w ? q.w : b.w, q.y > b.y ? q.y : b.y);
    if (!(ih > 0.f)) return 0.f;
    const float inter = __fmul_rn(iw, ih);
    const float ua = __double2float_rn(__dsub_rn(__dadd_rn(recall_area(b), (double)qarea), (double)inter));
    if (ua == 0.f) { *zero_ua = true; return 0.f; }
    return __fdiv_rn(inter, ua);
}

// (value, row) of a column over rows [0, n): max, then the first row holding it (numpy argmax); retired rows read -1
__device__ __forceinline__ void recall_column(const float4* __restrict__ props, int n, const uint32_t* dead, float4 q, float qarea,
                                              float* val, int* row, bool* zero_ua) {
    const int lane = threadIdx.x & 31;
    float bv = -INFINITY;
    int bi = 0;
    for (int r = lane; r < n; r += 32) {
        const float v = (dead[r >> 5] >> (r & 31)) & 1u ? -1.f : recall_iou(props[r], q, qarea, zero_ua);
        if (v > bv) { bv = v; bi = r; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_down_sync(0xffffffffu, bv, o);
        const int oi = __shfl_down_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    *val = bv;
    *row = bi;
}

static __global__ void __launch_bounds__(kRecallThreads) proposal_recall_kernel(const __grid_constant__ RecallParams P) {
    extern __shared__ __align__(16) unsigned char recall_smem[];
    float4* gbox = reinterpret_cast<float4*>(recall_smem);
    float* garea = reinterpret_cast<float*>(gbox + P.max_gts);
    float* bval = garea + P.max_gts;
    int* brow = reinterpret_cast<int*>(bval + P.max_gts);     // argmax row of each live column, -1 once retired
    uint32_t* dead = reinterpret_cast<uint32_t*>(brow + P.max_gts);
    __shared__ int s_g, s_row, s_col;
    const int img = blockIdx.x, c = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int64_t p0 = P.prop_off[img], np_all = P.prop_off[img + 1] - p0;
    if (np_all == 0) return;                                  // no proposals: nothing recorded (num_pos is counted on the host)
    const int64_t lim = P.limits[c];
    const int np = (int)(lim >= 0 && np_all > lim ? lim : np_all);
    const double lo = P.area_rng[2 * c], hi = P.area_rng[2 * c + 1];
    const int64_t g0 = P.gt_off[img], ng = P.gt_off[img + 1] - g0;
    double* out = P.out + P.out_off[(size_t)c * P.num_images + img];
    // the ground truth inside the area range, in roidb order
    if (warp == 0) {
        int g = 0;
        for (int64_t base = 0; base < ng; base += 32) {
            const int64_t k = base + lane;
            bool sel = false;
            if (k < ng) { const double a = P.gt_area[g0 + k]; sel = a >= lo && a <= hi; }
            const unsigned m = __ballot_sync(0xffffffffu, sel);
            if (sel) {
                const int pos = g + __popc(m & ((1u << lane) - 1u));
                const float4 q = P.gts[g0 + k];
                gbox[pos] = q;
                garea[pos] = __double2float_rn(recall_area(q));
            }
            g += __popc(m);
        }
        if (lane == 0) s_g = g;
    }
    __syncthreads();
    const int G = s_g;
    if (G == 0) return;
    for (int i = threadIdx.x; i < G; i += blockDim.x) out[i] = 0.0;
    for (int i = threadIdx.x; i < (np + 31) / 32; i += blockDim.x) dead[i] = 0u;
    if (np == 0) return;                                      // limit 0: every GT keeps its 0
    __syncthreads();
    const float4* props = P.props + p0;
    bool zero_ua = false;
    for (int k = warp; k < G; k += nwarps) {
        float v; int r;
        recall_column(props, np, dead, gbox[k], garea[k], &v, &r, &zero_ua);
        if (lane == 0) { bval[k] = v; brow[k] = r; }
    }
    __syncthreads();
    const int rounds = min(np, G);
    for (int j = 0; j < rounds; ++j) {
        if (warp == 0) {
            // max_overlaps.argmax(): the first column holding the largest column max
            float bv = -INFINITY;
            int bi = 0x7fffffff;
            for (int k = lane; k < G; k += 32)
                if (bval[k] > bv) { bv = bval[k]; bi = k; }
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                const float ov = __shfl_down_sync(0xffffffffu, bv, o);
                const int oi = __shfl_down_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) {
                const int r = brow[bi];
                out[j] = (double)bv;
                if (!(bv >= 0.f) || r < 0) atomicOr(P.flag, 1);
                if (r >= 0) dead[r >> 5] |= 1u << (r & 31);
                bval[bi] = -1.f;
                brow[bi] = -1;
                s_row = r;
                s_col = bi;
            }
        }
        __syncthreads();
        const int r = s_row;
        if (r < 0) break;                                     // flagged: the host raises
        // the retired row now reads -1: columns whose first max was on it (or whose max was <= -1) look again
        for (int k = warp; k < G; k += nwarps) {
            if (brow[k] < 0 || (brow[k] != r && bval[k] > -1.f)) continue;
            float v; int rr;
            recall_column(props, np, dead, gbox[k], garea[k], &v, &rr, &zero_ua);
            if (lane == 0) { bval[k] = v; brow[k] = rr; }
        }
        __syncthreads();
    }
    if (zero_ua) atomicOr(P.flag, 2);
}

inline cudaError_t proposal_recall_launch(const RecallParams& P, int num_combos, cudaStream_t s) {
    const size_t smem = proposal_recall_smem(P.max_gts, P.row_words);
    cudaError_t e = cudaFuncSetAttribute(proposal_recall_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    proposal_recall_kernel<<<dim3(P.num_images, num_combos), kRecallThreads, smem, s>>>(P);
    return cudaGetLastError();
}

}  // namespace dt

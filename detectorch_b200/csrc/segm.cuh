// detectorch_b200 -- mask paste + COCO run-length encoding on the device (SURVEY.md 8f rank 1).
// Reference: lib/utils/result_utils.py:170-228 (segm_results): per detection, zero-pad the MxM mask by one cell, expand the
// reference box by (M+2)/M (lib/utils/boxes.py:245-261, fp32), truncate to int32, cv2.resize(INTER_LINEAR, float32) to the
// box size, threshold, paste into an im_h x im_w uint8 image, pycocotools RLE-encode (maskApi.c rleEncode + rleToString).
//
// One CTA per (image, detection slot); each image has its own canvas size and live detection count.  Nothing of size im_h x im_w
// is materialised for the RLE: a thread owns image columns, walks the rows of the pasted region evaluating OpenCV's two-pass
// bilinear resize on the fly (float coefficient tables exactly as cv::resize builds them: double scale, float fx/fy, x clamped
// with weight (1,0), y by clipping the row index), and records the positions of the column-major flattening where the bit
// changes.  A block scan turns per-column transition counts into offsets, the differences of consecutive positions are the run
// lengths, and a second scan packs the LEB128-like string.  One more block scans the string lengths of all slots, and the strings
// are gathered into one packed buffer at those offsets.
#pragma once
#include "common.cuh"

namespace dt {

struct SegmGeom {
    int bx0, by0;            // expanded int32 box origin (may be negative)
    int w, h;                // resize target size (>= 1)
    int x0, x1, y0, y1;      // pasted region, clipped to the image; empty if x1 <= x0 or y1 <= y0
};

// boxes.expand_boxes (fp32 arithmetic on fp32 boxes) + .astype(np.int32) (truncation) + result_utils.py:200-212
__device__ __forceinline__ SegmGeom segm_geom(const float* b, const int* exp_box, float scale, int im_h, int im_w) {
    int e[4];
    if (exp_box) {
        e[0] = exp_box[0]; e[1] = exp_box[1]; e[2] = exp_box[2]; e[3] = exp_box[3];
    } else {
        float w_half = __fmul_rn(__fsub_rn(b[2], b[0]), .5f), h_half = __fmul_rn(__fsub_rn(b[3], b[1]), .5f);
        const float x_c = __fmul_rn(__fadd_rn(b[2], b[0]), .5f), y_c = __fmul_rn(__fadd_rn(b[3], b[1]), .5f);
        w_half = __fmul_rn(w_half, scale); h_half = __fmul_rn(h_half, scale);
        e[0] = (int)__fsub_rn(x_c, w_half); e[2] = (int)__fadd_rn(x_c, w_half);
        e[1] = (int)__fsub_rn(y_c, h_half); e[3] = (int)__fadd_rn(y_c, h_half);
    }
    SegmGeom g;
    g.bx0 = e[0]; g.by0 = e[1];
    g.w = max(e[2] - e[0] + 1, 1); g.h = max(e[3] - e[1] + 1, 1);
    g.x0 = max(e[0], 0); g.x1 = min(e[2] + 1, im_w);
    g.y0 = max(e[1], 0); g.y1 = min(e[3] + 1, im_h);
    if (g.x1 <= g.x0 || g.y1 <= g.y0) { g.x1 = g.x0 = 0; g.y1 = g.y0 = 0; }
    return g;
}

struct AxisCoef { int s; float w0, w1; };     // source cell, weights of cell s and s+1

// cv::resize coefficient set-up (INTER_LINEAR): fx = (float)((d + 0.5) * scale - 0.5) with scale = 1.0 / ((double)dst / src)
__device__ __forceinline__ AxisCoef resize_coef(int d, double scale) {
    float f = (float)(((double)d + 0.5) * scale - 0.5);
    const int s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    AxisCoef c; c.s = s; c.w1 = f; c.w0 = __fsub_rn(1.f, f);
    return c;
}
// x axis: clamped cells get weight (1, 0) and the clamped index
__device__ __forceinline__ AxisCoef resize_coef_x(int d, double scale, int n) {
    AxisCoef c = resize_coef(d, scale);
    if (c.s < 0) { c.s = 0; c.w0 = 1.f; c.w1 = 0.f; }
    if (c.s >= n - 1) { c.s = n - 1; c.w0 = 1.f; c.w1 = 0.f; }
    return c;
}

// horizontal pass of one source row at one destination column
__device__ __forceinline__ float segm_hrow(const float* pm, int S, int r, const AxisCoef& cx) {
    const int s1 = min(cx.s + 1, S - 1);
    return __fadd_rn(__fmul_rn(pm[r * S + cx.s], cx.w0), __fmul_rn(pm[r * S + s1], cx.w1));
}

// cv::resize switches INTER_LINEAR to the "area fast" kernel when both scale factors are exactly 2 (dst = S/2 x S/2): a 2x2 box
// average whose 4-wide SIMD body sums (a+b)+(c+d) and whose scalar tail (columns >= w & ~3) sums ((a+b)+c)+d, times 0.25f
__device__ __forceinline__ float segm_area2(const float* pm, int S, int dx, int dy, int w) {
    const float a = pm[(2 * dy) * S + 2 * dx], b = pm[(2 * dy) * S + 2 * dx + 1];
    const float c = pm[(2 * dy + 1) * S + 2 * dx], d = pm[(2 * dy + 1) * S + 2 * dx + 1];
    const float sum = dx < (w & ~3) ? __fadd_rn(__fadd_rn(a, b), __fadd_rn(c, d)) : __fadd_rn(__fadd_rn(__fadd_rn(a, b), c), d);
    return __fmul_rn(sum, 0.25f);
}

// value of the pasted mask at pixel (dx, dy) of the resized box: the area-fast average when both sides halve (area2), else the vertical
// pass over h0, h1, the horizontal passes (segm_hrow) of the source rows cy.s and cy.s + 1, with the row weights w0, w1
__device__ __forceinline__ float segm_pixel(const float* pm, int S, bool area2, int dx, int dy, int w, float h0, float h1, float w0, float w1) {
    return area2 ? segm_area2(pm, S, dx, dy, w) : __fadd_rn(__fmul_rn(h0, w0), __fmul_rn(h1, w1));
}

// exclusive scan of a[0..n) in shared memory by the whole block; returns the total.  scratch: 33 ints
__device__ __forceinline__ int block_exclusive_scan(int* a, int n, int* scratch) {
    const int T = blockDim.x, tid = threadIdx.x;
    const int chunk = (n + T - 1) / T;
    const int lo = min(tid * chunk, n), hi = min(lo + chunk, n);
    int sum = 0;
    for (int i = lo; i < hi; ++i) sum += a[i];
    int incl = sum;
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    __syncthreads();
    if (lane == 31) scratch[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int v = lane < (T >> 5) ? scratch[lane] : 0;
        int w = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
        scratch[lane] = w - v;
        if (lane == 31) scratch[32] = w;
    }
    __syncthreads();
    int run = scratch[warp] + incl - sum;
    for (int i = lo; i < hi; ++i) { const int v = a[i]; a[i] = run; run += v; }
    __syncthreads();
    return scratch[32];
}

// exclusive prefix of one value per thread over the block; *total = sum.  scratch: 33 values
template <typename T>
__device__ __forceinline__ T block_scan_value(T v, T* scratch, T* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const T u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
    __syncthreads();
    if (lane == 31) scratch[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const T x = lane < (int)(blockDim.x >> 5) ? scratch[lane] : T(0);
        T w = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const T u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
        scratch[lane] = w - x;
        if (lane == 31) scratch[32] = w;
    }
    __syncthreads();
    *total = scratch[32];
    return scratch[warp] + incl - v;
}

struct SegmRowCoef { int s; float w0, w1; int pad; };

// Image side of the tables of dt_segm_rle_batch_append's launch, whatever its batch holds (include/detectorch_b200.h).
constexpr int kSegmMaxSide = 8192;

// Grid (cap, B): block (d, b) is detection slot d of image b, i.e. slot s = b * cap + d of the flat per-slot arrays.
// masks: [B*cap, K, M, M] (class-specific: K classes, cls[s] selects) or [B*cap, M, M] (K == 1 / cls == NULL)
// im_sizes: int32 [B, 2] (im_h, im_w) of each image's canvas, or NULL (every image is max_h x max_w).  The shared row / column tables
// are sized for max_h x max_w; an image whose size is not within [1, max] produces empty results, and raises *size_flag (atomicOr 1)
// when size_flag is not NULL.
// num_dets_dev: int32 [B] live slots per image (NULL: all); slots at or past the count produce empty results
// outputs per slot s: counts[s*runs_cap ..] (uint32 run lengths), num_counts[s], strings (cap str_cap per slot), str_len[s];
// *overflow: atomicMax of the runs a slot needed when runs_cap or str_cap was too small
static __global__ void __launch_bounds__(256) segm_rle_kernel(const float* __restrict__ masks, const int* __restrict__ cls, int K, int M,
                                                              const float* __restrict__ ref_boxes, const int* __restrict__ exp_boxes,
                                                              const int* __restrict__ num_dets_dev, const int* __restrict__ im_sizes,
                                                              int max_h, int max_w, float thresh,
                                                              uint32_t* __restrict__ positions, uint32_t* __restrict__ counts,
                                                              int* __restrict__ num_counts, int runs_cap,
                                                              uint8_t* __restrict__ strings, int* __restrict__ str_len, int str_cap,
                                                              int* __restrict__ overflow, int* __restrict__ size_flag) {
    extern __shared__ __align__(16) uint8_t segm_smem[];
    const int b = blockIdx.y, det = blockIdx.x;
    const size_t d = (size_t)b * gridDim.x + det;
    const int S = M + 2;
    float* pm = reinterpret_cast<float*>(segm_smem);                                     // [S][S] zero-padded mask
    SegmRowCoef* rows = reinterpret_cast<SegmRowCoef*>(pm + ((S * S + 3) & ~3));          // [max_h]
    int* colcnt = reinterpret_cast<int*>(rows + max_h);                                  // [max_w + 2]
    int* scratch = colcnt + max_w + 2;                                                   // [40]
    const int im_h = im_sizes ? im_sizes[2 * b] : max_h, im_w = im_sizes ? im_sizes[2 * b + 1] : max_w;
    if (size_flag && det == 0 && threadIdx.x == 0 && (im_h < 1 || im_w < 1 || im_h > max_h || im_w > max_w)) atomicOr(size_flag, 1);
    if ((num_dets_dev && det >= num_dets_dev[b]) || im_h < 1 || im_w < 1 || im_h > max_h || im_w > max_w) {
        if (threadIdx.x == 0) { num_counts[d] = 0; str_len[d] = 0; }
        return;
    }
    const SegmGeom g = segm_geom(ref_boxes ? ref_boxes + d * 4 : nullptr, exp_boxes ? exp_boxes + d * 4 : nullptr,
                                 (float)(((double)M + 2.0) / (double)M), im_h, im_w);
    const float* msrc = masks + (d * K + (cls ? cls[d] : 0)) * M * M;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) {
        const int r = i / S, c = i - r * S;
        pm[i] = (r >= 1 && r <= M && c >= 1 && c <= M) ? msrc[(r - 1) * M + (c - 1)] : 0.f;
    }
    const double scale_x = 1.0 / ((double)g.w / (double)S), scale_y = 1.0 / ((double)g.h / (double)S);
    for (int y = g.y0 + threadIdx.x; y < g.y1; y += blockDim.x) {
        const AxisCoef c = resize_coef(y - g.by0, scale_y);
        SegmRowCoef rc; rc.s = c.s; rc.w0 = c.w0; rc.w1 = c.w1; rc.pad = 0;
        rows[y] = rc;
    }
    __syncthreads();
    // value of the pasted mask at an in-region pixel
    const bool area2 = g.w * 2 == S && g.h * 2 == S;
    auto bit_at = [&](int x, int y) -> int {
        // the area-fast value needs no coefficients: returning it before they are read keeps the kernel at 40 registers rather than 48
        // (CUDA 12.9), one more CTA per SM
        if (area2) return segm_area2(pm, S, x - g.bx0, y - g.by0, g.w) > thresh ? 1 : 0;
        const AxisCoef cx = resize_coef_x(x - g.bx0, scale_x, S);
        const SegmRowCoef rc = rows[y];
        const float h0 = segm_hrow(pm, S, min(max(rc.s, 0), S - 1), cx), h1 = segm_hrow(pm, S, min(max(rc.s + 1, 0), S - 1), cx);
        return segm_pixel(pm, S, area2, x - g.bx0, y - g.by0, g.w, h0, h1, rc.w0, rc.w1) > thresh ? 1 : 0;
    };
    const bool empty = g.x1 <= g.x0;
    const int xe = empty ? -1 : (g.x1 < im_w ? g.x1 : g.x1 - 1);        // last column that can hold a transition (pseudo column x1)
    const int ncols = empty ? 0 : xe - g.x0 + 1;
    uint32_t* my_counts = counts + d * runs_cap;
    uint32_t* my_pos = positions + d * runs_cap;
    // one sweep of a column; EMIT(pos) is called in increasing order of the column-major position
#define DT_SEGM_SWEEP(EMIT)                                                                                              \
    {                                                                                                                    \
        const bool incol = x < g.x1;                                                                                     \
        int prev = (x > g.x0 && g.y1 == im_h) ? bit_at(x - 1, im_h - 1) : 0;                                             \
        int ys = g.y0;                                                                                                   \
        if (!(incol && g.y0 == 0)) {                                                                                     \
            if (prev) { EMIT((long long)x * im_h); }                                                                     \
            prev = 0;                                                                                                    \
        }                                                                                                                \
        if (incol) {                                                                                                     \
            const AxisCoef cx = resize_coef_x(x - g.bx0, scale_x, S);                                                    \
            int cur_s = -1000; float h0 = 0.f, h1 = 0.f;                                                                 \
            for (int y = ys; y < g.y1; ++y) {                                                                            \
                const SegmRowCoef rc = rows[y];                                                                          \
                if (rc.s != cur_s) {                                                                                     \
                    cur_s = rc.s;                                                                                        \
                    h0 = segm_hrow(pm, S, min(max(rc.s, 0), S - 1), cx);                                                 \
                    h1 = segm_hrow(pm, S, min(max(rc.s + 1, 0), S - 1), cx);                                             \
                }                                                                                                        \
                const float val = segm_pixel(pm, S, area2, x - g.bx0, y - g.by0, g.w, h0, h1, rc.w0, rc.w1);             \
                const int cur = val > thresh ? 1 : 0;                                                                    \
                if (cur != prev) { EMIT((long long)x * im_h + y); prev = cur; }                                          \
            }                                                                                                            \
            if (g.y1 < im_h && prev) { EMIT((long long)x * im_h + g.y1); }                                               \
        }                                                                                                                \
    }
    for (int ci = threadIdx.x; ci < ncols; ci += blockDim.x) {
        const int x = g.x0 + ci;
        int n = 0;
#define DT_EMIT_COUNT(pos) ++n
        DT_SEGM_SWEEP(DT_EMIT_COUNT)
#undef DT_EMIT_COUNT
        colcnt[ci] = n;
    }
    __syncthreads();
    const int ntrans = ncols ? block_exclusive_scan(colcnt, ncols, scratch) : 0;
    const int m = ntrans + 1;                                           // number of runs
    if (m > runs_cap) {
        if (threadIdx.x == 0) { atomicMax(overflow, m); num_counts[d] = m; str_len[d] = 0; }
        return;
    }
    // second sweep: positions of the transitions
    for (int ci = threadIdx.x; ci < ncols; ci += blockDim.x) {
        const int x = g.x0 + ci;
        int k = colcnt[ci];
#define DT_EMIT_POS(pos) my_pos[k++] = (uint32_t)(pos)
        DT_SEGM_SWEEP(DT_EMIT_POS)
#undef DT_EMIT_POS
    }
#undef DT_SEGM_SWEEP
    __syncthreads();
    const long long total = (long long)im_h * im_w;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        const long long hi = i < ntrans ? (long long)my_pos[i] : total;
        const long long lo = i > 0 ? (long long)my_pos[i - 1] : 0;
        my_counts[i] = (uint32_t)(hi - lo);
    }
    __syncthreads();
    // maskApi.c rleToString: x = cnts[i] - (i > 2 ? cnts[i-2] : 0); 5 data bits per char, bit 5 = continuation, + 48
    const int chunk = (m + blockDim.x - 1) / blockDim.x;
    const int lo_i = min((int)threadIdx.x * chunk, m), hi_i = min(lo_i + chunk, m);
    int nchar = 0;
    for (int i = lo_i; i < hi_i; ++i) {
        long long x = (long long)my_counts[i];
        if (i > 2) x -= (long long)my_counts[i - 2];
        bool more = true;
        while (more) {
            const int c = (int)(x & 0x1f);
            x >>= 5;
            more = (c & 0x10) ? x != -1 : x != 0;
            ++nchar;
        }
    }
    int total_chars;
    int off = block_scan_value(nchar, scratch, &total_chars);
    if (total_chars > str_cap) {
        if (threadIdx.x == 0) { atomicMax(overflow, m); num_counts[d] = m; str_len[d] = 0; }
        return;
    }
    uint8_t* my_str = strings + d * str_cap;
    for (int i = lo_i; i < hi_i; ++i) {
        long long x = (long long)my_counts[i];
        if (i > 2) x -= (long long)my_counts[i - 2];
        bool more = true;
        while (more) {
            int c = (int)(x & 0x1f);
            x >>= 5;
            more = (c & 0x10) ? x != -1 : x != 0;
            if (more) c |= 0x20;
            my_str[off++] = (uint8_t)(c + 48);
        }
    }
    if (threadIdx.x == 0) { num_counts[d] = m; str_len[d] = total_chars; }
}

// offsets[0..D] = base + exclusive scan of str_len[0..D) (offsets[D] = base + total), one block: each thread sums a contiguous chunk, a
// block scan of the chunk sums gives each chunk's start.  Without a cursor base is 0.  With one (a batch appended to a char arena) base
// is *cursor, and the batch is committed, *cursor advanced by the total, only if no slot overflowed (flags[0]), every image was within
// the tables (flags[1]) and base + total <= capacity; a batch that does not fit sets flags[2] and leaves the cursor.
static __global__ void __launch_bounds__(1024) segm_offsets_kernel(const int* __restrict__ str_len, int D, long long* __restrict__ cursor,
                                                                   long long capacity, int* __restrict__ flags, long long* __restrict__ offsets) {
    __shared__ long long scratch[33];
    const long long base = cursor ? *cursor : 0;    // read by every thread before the scan's barriers, written after them
    const int chunk = (D + blockDim.x - 1) / blockDim.x;
    const int lo = min((int)threadIdx.x * chunk, D), hi = min(lo + chunk, D);
    long long sum = 0;
    for (int i = lo; i < hi; ++i) sum += str_len[i];
    long long total;
    long long run = base + block_scan_value(sum, scratch, &total);
    for (int i = lo; i < hi; ++i) { offsets[i] = run; run += str_len[i]; }
    if (threadIdx.x == 0) {
        offsets[D] = base + total;
        if (cursor && flags[0] == 0 && flags[1] == 0) {
            if (base + total <= capacity) *cursor = base + total;
            else flags[2] = 1;
        }
    }
}

// gathers the per-slot strings into one contiguous buffer at the scanned offsets; one warp per slot.  Given flags (an arena batch),
// only a committed batch is written: none of the flags of segm_rle_kernel and segm_offsets_kernel raised.
static __global__ void __launch_bounds__(256) segm_compact_kernel(const uint8_t* __restrict__ strings, const int* __restrict__ str_len, int D,
                                                                  int str_cap, const long long* __restrict__ offsets,
                                                                  const int* __restrict__ flags, uint8_t* __restrict__ packed) {
    const int d = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (d >= D || (flags && (flags[0] || flags[1] || flags[2]))) return;
    const int n = str_len[d];
    uint8_t* dst = packed + offsets[d];
    const uint8_t* src = strings + (size_t)d * str_cap;
    for (int i = lane; i < n; i += 32) dst[i] = src[i];
}

// pasted binary masks [D, im_h, im_w] uint8 (for callers that want the image-sized mask rather than its RLE)
static __global__ void __launch_bounds__(256) segm_paste_kernel(const float* __restrict__ masks, const int* __restrict__ cls, int K, int M,
                                                                const float* __restrict__ ref_boxes, const int* __restrict__ exp_boxes,
                                                                const int* __restrict__ num_dets_dev, int im_h, int im_w, float thresh,
                                                                uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t segm_smem[];
    const int d = blockIdx.x;
    const int S = M + 2;
    float* pm = reinterpret_cast<float*>(segm_smem);
    uint8_t* o = out + (size_t)d * im_h * im_w;
    const bool live = !(num_dets_dev && d >= *num_dets_dev);
    SegmGeom g = segm_geom(ref_boxes ? ref_boxes + (size_t)d * 4 : nullptr, exp_boxes ? exp_boxes + (size_t)d * 4 : nullptr,
                           (float)(((double)M + 2.0) / (double)M), im_h, im_w);
    if (!live) { g.x0 = g.x1 = g.y0 = g.y1 = 0; }
    const float* msrc = masks + ((size_t)d * K + (cls && live ? cls[d] : 0)) * M * M;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) {
        const int r = i / S, c = i - r * S;
        pm[i] = (live && r >= 1 && r <= M && c >= 1 && c <= M) ? msrc[(r - 1) * M + (c - 1)] : 0.f;
    }
    __syncthreads();
    const double scale_x = 1.0 / ((double)g.w / (double)S), scale_y = 1.0 / ((double)g.h / (double)S);
    const bool area2 = g.w * 2 == S && g.h * 2 == S;
    for (int y = 0; y < im_h; ++y) {
        const bool inrow = y >= g.y0 && y < g.y1;
        AxisCoef cy; cy.s = 0; cy.w0 = cy.w1 = 0.f;
        if (inrow) cy = resize_coef(y - g.by0, scale_y);
        const int r0 = min(max(cy.s, 0), S - 1), r1 = min(max(cy.s + 1, 0), S - 1);
        for (int x = threadIdx.x; x < im_w; x += blockDim.x) {
            uint8_t v = 0;
            if (inrow && x >= g.x0 && x < g.x1) {
                const AxisCoef cx = resize_coef_x(x - g.bx0, scale_x, S);
                const float val = segm_pixel(pm, S, area2, x - g.bx0, y - g.by0, g.w, segm_hrow(pm, S, r0, cx), segm_hrow(pm, S, r1, cx),
                                             cy.w0, cy.w1);
                v = val > thresh ? 1 : 0;
            }
            o[(size_t)y * im_w + x] = v;
        }
    }
}

// ---------------------------------------------------------------------------------- image pre-processing (SURVEY 8f rank 3)
// lib/utils/blob.py:57-87 prep_im_for_blob (uint8 BGR HWC -> float32, minus the per-channel mean, cv2.resize(fx = fy = im_scale,
// INTER_LINEAR)) fused with blob.py:27-55 im_list_to_blob (zero-pad to blob_h x blob_w, HWC -> CHW).  The resize is OpenCV's own
// float kernel: coefficients from scale = 1 / im_scale (the fx/fy form of cv::resize), horizontal then vertical pass with separately
// rounded products; im_scale == 0.5 takes OpenCV's area-fast path (2x2 box, ((a+b)+c)+d times 0.25f for 3 channels).  On an odd side
// whose half rounds up (cvRound(n / 2) = (n + 1) / 2) the last column / row / corner cell is partial: OpenCV sums its in-range pixels
// row-major from 0 and divides by their count.
static __global__ void __launch_bounds__(256) prep_image_kernel(const uint8_t* __restrict__ im, int h, int w, double m0, double m1, double m2,
                                                                double inv_scale, int out_h, int out_w, int area2,
                                                                float* __restrict__ blob, int blob_h, int blob_w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= blob_w) return;
    const size_t plane = (size_t)blob_h * blob_w;
    float* o = blob + (size_t)y * blob_w + x;
    if (y >= out_h || x >= out_w) { o[0] = 0.f; o[plane] = 0.f; o[2 * plane] = 0.f; return; }
    const double mean[3] = {m0, m1, m2};
    auto px = [&](int r, int cidx, int c) -> float { return (float)((double)im[((size_t)r * w + cidx) * 3 + c] - mean[c]); };
    if (area2) {
        const int nr = min(h - 2 * y, 2), nc = min(w - 2 * x, 2);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (nr == 2 && nc == 2) {
                const float a = px(2 * y, 2 * x, c), b = px(2 * y, 2 * x + 1, c), cc = px(2 * y + 1, 2 * x, c), d = px(2 * y + 1, 2 * x + 1, c);
                o[c * plane] = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(a, b), cc), d), 0.25f);
            } else {
                float s = 0.f;
                for (int r = 0; r < nr; ++r)
                    for (int q = 0; q < nc; ++q) s = __fadd_rn(s, px(2 * y + r, 2 * x + q, c));
                o[c * plane] = __fdiv_rn(s, (float)(nr * nc));
            }
        }
        return;
    }
    const AxisCoef cx = resize_coef_x(x, inv_scale, w);
    const AxisCoef cy = resize_coef(y, inv_scale);
    const int r0 = min(max(cy.s, 0), h - 1), r1 = min(max(cy.s + 1, 0), h - 1);
    const int x1 = min(cx.s + 1, w - 1);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float h0 = __fadd_rn(__fmul_rn(px(r0, cx.s, c), cx.w0), __fmul_rn(px(r0, x1, c), cx.w1));
        const float h1 = __fadd_rn(__fmul_rn(px(r1, cx.s, c), cx.w0), __fmul_rn(px(r1, x1, c), cx.w1));
        o[c * plane] = __fadd_rn(__fmul_rn(h0, cy.w0), __fmul_rn(h1, cy.w1));
    }
}

}  // namespace dt

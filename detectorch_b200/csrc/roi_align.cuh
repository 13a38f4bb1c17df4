// detectorch_b200 -- RoIAlign forward (caffe2 semantics, no RoI rounding, RoI >= 1x1,
// average of grid_h x grid_w bilinear samples; samples outside [-1,H]x[-1,W] contribute 0).
// Reference: lib/cppcuda_cffi/src/cuda/roi_align_forward_cuda_kernel.cu:30-159 (GPU),
//            lib/cppcuda_cffi/src/cpp/roi_align_cpu_loop.cpp:118-224 (CPU loop = parity oracle).
//
// Two layouts:
//  * roi_align_nchw_kernel  : the reference's public layout (features NCHW, out [R,C,ph,pw]).
//    One CTA per RoI; the separable 1-D sample tables (y taps / x taps) are built once per RoI in
//    shared memory and shared by all channels; threads sweep the RoI's contiguous C*ph*pw output
//    run so stores are fully coalesced.  The fp32 expression order of the reference CPU loop is
//    reproduced with explicit _rn intrinsics (no FMA contraction) => bit-identical to the oracle.
//  * roi_align_nhwc_kernel  : internal layout of the fused detector (features NHWC, multi-level,
//    out [R,ph,pw,C]); every tap is one 128-bit load of 4 channels, stores are 128-bit.
#pragma once
#include "common.cuh"

namespace dt {

struct AxisTap {      // one 1-D bilinear sample along an axis
    int lo, hi;       // cell indices
    float wl, wh;     // weight of lo / hi cell (hy / ly in the reference's naming)
    int valid;        // 0 -> sample is outside [-1, extent] and contributes nothing
};

// reference bilinear_interpolate() :30-80, one axis at a time (the test and the clamps are separable)
__device__ __forceinline__ AxisTap axis_tap(float v, int extent) {
    AxisTap t;
    t.valid = !(v < -1.0f || v > (float)extent);
    if (v <= 0.f) v = 0.f;
    int lo = (int)v;
    int hi;
    if (lo >= extent - 1) { hi = lo = extent - 1; v = (float)lo; } else { hi = lo + 1; }
    const float l = __fsub_rn(v, (float)lo);
    t.lo = lo; t.hi = hi; t.wh = l; t.wl = __fsub_rn(1.f, l);
    return t;
}

struct RoiGeom {
    float start_w, start_h, bin_w, bin_h;
    int grid_w, grid_h, batch;
};

__device__ __forceinline__ RoiGeom roi_geom(const float* r, int roi_cols, float scale, int ph, int pw, int sampling_ratio) {
    RoiGeom g;
    g.batch = 0;
    if (roi_cols == 5) { g.batch = (int)r[0]; ++r; }
    g.start_w = __fmul_rn(r[0], scale); g.start_h = __fmul_rn(r[1], scale);
    const float end_w = __fmul_rn(r[2], scale), end_h = __fmul_rn(r[3], scale);
    const float rw = fmaxf(__fsub_rn(end_w, g.start_w), 1.f), rh = fmaxf(__fsub_rn(end_h, g.start_h), 1.f);
    g.bin_h = __fdiv_rn(rh, (float)ph); g.bin_w = __fdiv_rn(rw, (float)pw);
    g.grid_h = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(__fdiv_rn(rh, (float)ph));
    g.grid_w = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(__fdiv_rn(rw, (float)pw));
    return g;
}

// sample coordinate: start + p*bin + (i + .5f)*bin/grid, evaluated left to right in fp32 (:140-147)
__device__ __forceinline__ float sample_coord(float start, int p, float bin, int i, int grid) {
    return __fadd_rn(__fadd_rn(start, __fmul_rn((float)p, bin)), __fdiv_rn(__fmul_rn((float)i + .5f, bin), (float)grid));
}

static constexpr int kMaxAxisSamples = 512;   // pooled * grid per axis held in smem (14 * 36 fits)

// ---------------------------------------------------------------------------------- NCHW (public layout)
static __global__ void __launch_bounds__(256) roi_align_nchw_kernel(const float* __restrict__ feat, const float* __restrict__ rois,
                                                            long long num_rois, int roi_cols, int C, int H, int W, int PH, int PW,
                                                            float scale, int sampling_ratio, float* __restrict__ out) {
    __shared__ AxisTap ytab[kMaxAxisSamples];
    __shared__ AxisTap xtab[kMaxAxisSamples];
    for (long long n = blockIdx.x; n < num_rois; n += gridDim.x) {
        const RoiGeom g = roi_geom(rois + n * roi_cols, roi_cols, scale, PH, PW, sampling_ratio);
        const int ny = PH * g.grid_h, nx = PW * g.grid_w;
        const bool tabled = (ny <= kMaxAxisSamples) && (nx <= kMaxAxisSamples);
        __syncthreads();   // previous RoI's table no longer in use
        if (tabled) {
            for (int i = threadIdx.x; i < ny + nx; i += blockDim.x) {
                if (i < ny) ytab[i] = axis_tap(sample_coord(g.start_h, i / g.grid_h, g.bin_h, i % g.grid_h, g.grid_h), H);
                else { const int k = i - ny; xtab[k] = axis_tap(sample_coord(g.start_w, k / g.grid_w, g.bin_w, k % g.grid_w, g.grid_w), W); }
            }
        }
        __syncthreads();
        const float count = (float)(g.grid_h * g.grid_w);
        const int per_roi = C * PH * PW;
        const float* fb = feat + (size_t)g.batch * C * H * W;
        float* ob = out + (size_t)n * per_roi;
        for (int o = threadIdx.x; o < per_roi; o += blockDim.x) {
            const int pw = o % PW;
            const int ph = (o / PW) % PH;
            const int c = o / (PW * PH);
            const float* plane = fb + (size_t)c * H * W;
            float acc = 0.f;
            for (int iy = 0; iy < g.grid_h; ++iy) {
                const AxisTap ty = tabled ? ytab[ph * g.grid_h + iy] : axis_tap(sample_coord(g.start_h, ph, g.bin_h, iy, g.grid_h), H);
                const float* r0 = plane + (size_t)ty.lo * W;
                const float* r1 = plane + (size_t)ty.hi * W;
                for (int ix = 0; ix < g.grid_w; ++ix) {
                    const AxisTap tx = tabled ? xtab[pw * g.grid_w + ix] : axis_tap(sample_coord(g.start_w, pw, g.bin_w, ix, g.grid_w), W);
                    if (ty.valid && tx.valid) {
                        // val = w1*v1 + w2*v2 + w3*v3 + w4*v4, left to right, then acc += val  (cpu_loop.cpp:207-212)
                        const float w1 = __fmul_rn(ty.wl, tx.wl), w2 = __fmul_rn(ty.wl, tx.wh);
                        const float w3 = __fmul_rn(ty.wh, tx.wl), w4 = __fmul_rn(ty.wh, tx.wh);
                        float v = __fmul_rn(w1, __ldg(r0 + tx.lo));
                        v = __fadd_rn(v, __fmul_rn(w2, __ldg(r0 + tx.hi)));
                        v = __fadd_rn(v, __fmul_rn(w3, __ldg(r1 + tx.lo)));
                        v = __fadd_rn(v, __fmul_rn(w4, __ldg(r1 + tx.hi)));
                        acc = __fadd_rn(acc, v);
                    }
                }
            }
            ob[o] = __fdiv_rn(acc, count);
        }
    }
}

// ---------------------------------------------------------------------------------- NHWC multi-level (internal layout)
struct RoiLevels {
    const float* feat[5];   // NHWC maps, finest first
    int H[5], W[5];
    float scale[5];
    int num_levels;
    // per-image sizes (image_info): the bounds of a RoI of image b are b's extent at the level's stride, not the canvas map.  Null = off.
    const float* im_info = nullptr;
    int stride[5] = {0, 0, 0, 0, 0};
};

// rois [R,5] (batch,x1,y1,x2,y2); level[R] (index into lv, or nullptr -> level 0); out [R,PH,PW,C].
// grid: one CTA per RoI (grid-stride). C % 4 == 0.
static __global__ void __launch_bounds__(256) roi_align_nhwc_kernel(RoiLevels lv, const float* __restrict__ rois, const int* __restrict__ level,
                                                            const int* __restrict__ num_rois_dev, int max_rois, int C, int PH, int PW,
                                                            int sampling_ratio, float* __restrict__ out) {
    __shared__ AxisTap ytab[kMaxAxisSamples];
    __shared__ AxisTap xtab[kMaxAxisSamples];
    const int num_rois = num_rois_dev ? min(*num_rois_dev, max_rois) : max_rois;
    const int C4 = C >> 2;
    for (int n = blockIdx.x; n < max_rois; n += gridDim.x) {
        float4* ob = reinterpret_cast<float4*>(out + (size_t)n * PH * PW * C);
        const int per_roi = PH * PW * C4;
        if (n >= num_rois) {    // padded slot: defined (zero) output
            for (int o = threadIdx.x; o < per_roi; o += blockDim.x) ob[o] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        const int l = level ? level[n] : 0;
        const int H = lv.H[l], W = lv.W[l];
        const RoiGeom g = roi_geom(rois + (size_t)n * 5, 5, lv.scale[l], PH, PW, sampling_ratio);
        const ImageInfo ext = image_info(lv.im_info, g.batch, lv.stride[l], H, W);     // sample bounds (H, W stay the row pitch)
        const int ny = PH * g.grid_h, nx = PW * g.grid_w;
        const bool tabled = (ny <= kMaxAxisSamples) && (nx <= kMaxAxisSamples);
        __syncthreads();
        if (tabled) {
            for (int i = threadIdx.x; i < ny + nx; i += blockDim.x) {
                if (i < ny) ytab[i] = axis_tap(sample_coord(g.start_h, i / g.grid_h, g.bin_h, i % g.grid_h, g.grid_h), ext.h);
                else { const int k = i - ny; xtab[k] = axis_tap(sample_coord(g.start_w, k / g.grid_w, g.bin_w, k % g.grid_w, g.grid_w), ext.w); }
            }
        }
        __syncthreads();
        const float count = (float)(g.grid_h * g.grid_w);
        const float4* fb = reinterpret_cast<const float4*>(lv.feat[l] + (size_t)g.batch * H * W * C);
        if (tabled && g.grid_h == 2 && g.grid_w == 2) {
            // sampling_ratio == 2 (every FPN RoIAlign): all 16 tap loads of a bin are issued before any arithmetic
            // (memory-level parallelism), then combined in exactly the reference order.
            for (int o = threadIdx.x; o < per_roi; o += blockDim.x) {
                const int c4 = o % C4;
                const int bin = o / C4;
                const int pw = bin % PW, ph = bin / PW;
                AxisTap ty[2], tx[2];
                ty[0] = ytab[ph * 2]; ty[1] = ytab[ph * 2 + 1];
                tx[0] = xtab[pw * 2]; tx[1] = xtab[pw * 2 + 1];
                float4 v[2][2][4];
#pragma unroll
                for (int iy = 0; iy < 2; ++iy)
#pragma unroll
                    for (int ix = 0; ix < 2; ++ix) {
                        v[iy][ix][0] = __ldg(fb + ((size_t)ty[iy].lo * W + tx[ix].lo) * C4 + c4);
                        v[iy][ix][1] = __ldg(fb + ((size_t)ty[iy].lo * W + tx[ix].hi) * C4 + c4);
                        v[iy][ix][2] = __ldg(fb + ((size_t)ty[iy].hi * W + tx[ix].lo) * C4 + c4);
                        v[iy][ix][3] = __ldg(fb + ((size_t)ty[iy].hi * W + tx[ix].hi) * C4 + c4);
                    }
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int iy = 0; iy < 2; ++iy)
#pragma unroll
                    for (int ix = 0; ix < 2; ++ix) {
                        if (ty[iy].valid && tx[ix].valid) {
                            const float w1 = __fmul_rn(ty[iy].wl, tx[ix].wl), w2 = __fmul_rn(ty[iy].wl, tx[ix].wh);
                            const float w3 = __fmul_rn(ty[iy].wh, tx[ix].wl), w4 = __fmul_rn(ty[iy].wh, tx[ix].wh);
#define DT_TAP(f)                                                                                                     \
    acc.f = __fadd_rn(acc.f, __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w1, v[iy][ix][0].f), __fmul_rn(w2, v[iy][ix][1].f)), \
                                                   __fmul_rn(w3, v[iy][ix][2].f)), __fmul_rn(w4, v[iy][ix][3].f)));
                            DT_TAP(x) DT_TAP(y) DT_TAP(z) DT_TAP(w)
#undef DT_TAP
                        }
                    }
                ob[o] = make_float4(__fdiv_rn(acc.x, count), __fdiv_rn(acc.y, count), __fdiv_rn(acc.z, count), __fdiv_rn(acc.w, count));
            }
            continue;
        }
        for (int o = threadIdx.x; o < per_roi; o += blockDim.x) {
            const int c4 = o % C4;
            const int bin = o / C4;
            const int pw = bin % PW, ph = bin / PW;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int iy = 0; iy < g.grid_h; ++iy) {
                const AxisTap ty = tabled ? ytab[ph * g.grid_h + iy] : axis_tap(sample_coord(g.start_h, ph, g.bin_h, iy, g.grid_h), ext.h);
                for (int ix = 0; ix < g.grid_w; ++ix) {
                    const AxisTap tx = tabled ? xtab[pw * g.grid_w + ix] : axis_tap(sample_coord(g.start_w, pw, g.bin_w, ix, g.grid_w), ext.w);
                    if (ty.valid && tx.valid) {
                        const float w1 = __fmul_rn(ty.wl, tx.wl), w2 = __fmul_rn(ty.wl, tx.wh);
                        const float w3 = __fmul_rn(ty.wh, tx.wl), w4 = __fmul_rn(ty.wh, tx.wh);
                        const float4 v1 = __ldg(fb + ((size_t)ty.lo * W + tx.lo) * C4 + c4);
                        const float4 v2 = __ldg(fb + ((size_t)ty.lo * W + tx.hi) * C4 + c4);
                        const float4 v3 = __ldg(fb + ((size_t)ty.hi * W + tx.lo) * C4 + c4);
                        const float4 v4 = __ldg(fb + ((size_t)ty.hi * W + tx.hi) * C4 + c4);
#define DT_TAP(f)                                                                                       \
    acc.f = __fadd_rn(acc.f, __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w1, v1.f), __fmul_rn(w2, v2.f)), \
                                                   __fmul_rn(w3, v3.f)), __fmul_rn(w4, v4.f)));
                        DT_TAP(x) DT_TAP(y) DT_TAP(z) DT_TAP(w)
#undef DT_TAP
                    }
                }
            }
            ob[o] = make_float4(__fdiv_rn(acc.x, count), __fdiv_rn(acc.y, count), __fdiv_rn(acc.z, count), __fdiv_rn(acc.w, count));
        }
    }
}

// ================================================================================== fast path (sampling_ratio == 2)
// Bilinear RoIAlign with a product sample grid is separable:  out[ph][pw] = 1/4 * sum_r sum_c Wy[ph][r] * Wx[pw][c] * F[r][c],
// where for each bin row (column) the <= 4 distinct tap rows (columns) of its two samples carry the summed weights.
// The tables are built once per RoI and shared by all channels; duplicate taps (small RoIs: both samples in the same
// cell) are merged, so a bin costs nr*nc <= 16 (typically 4..9) 128-bit loads + FMAs instead of 16 loads + 28 un-fused
// flops per channel.  Results differ from the exact kernels only by fp32 re-association (~1e-7 relative; parity bar 1e-4).
struct AxisBin {
    int idx[4];
    float w[4];     // summed tap weights, pre-multiplied by 0.5 (0.5 * 0.5 = the 1/4 sample average, exact)
    int n;
};

__device__ __forceinline__ AxisBin axis_bin2(float start, int p, float bin, int extent) {
    AxisBin b;
    b.n = 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const AxisTap t = axis_tap(sample_coord(start, p, bin, i, 2), extent);
        if (!t.valid) continue;
        const int id[2] = {t.lo, t.hi};
        const float wt[2] = {0.5f * t.wl, 0.5f * t.wh};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            if (wt[k] == 0.f) continue;
            int j = 0;
            for (; j < b.n; ++j)
                if (b.idx[j] == id[k]) { b.w[j] += wt[k]; break; }
            if (j == b.n) { b.idx[b.n] = id[k]; b.w[b.n] = wt[k]; ++b.n; }
        }
    }
    for (int j = b.n; j < 4; ++j) { b.idx[j] = 0; b.w[j] = 0.f; }
    return b;
}

static constexpr int kMaxPooled = 16;     // pooled_height / pooled_width supported by the fast path (7 and 14 in practice)

// NHWC features (multi-level), out [R, PH, PW, C]; one CTA per RoI (grid-stride), threads over (bin, 4-channel group)
static __global__ void __launch_bounds__(256) roi_align_fast_nhwc_kernel(RoiLevels lv, const float* __restrict__ rois, const int* __restrict__ level,
                                                                         int max_rois, int C, int PH, int PW, float* __restrict__ out) {
    __shared__ AxisBin ytab[kMaxPooled];
    __shared__ AxisBin xtab[kMaxPooled];
    const int C4 = C >> 2;
    for (int n = blockIdx.x; n < max_rois; n += gridDim.x) {
        const int l = level ? level[n] : 0;
        const int H = lv.H[l], W = lv.W[l];
        const RoiGeom g = roi_geom(rois + (size_t)n * 5, 5, lv.scale[l], PH, PW, 2);
        const ImageInfo ext = image_info(lv.im_info, g.batch, lv.stride[l], H, W);     // sample bounds (H, W stay the row pitch)
        __syncthreads();
        if (threadIdx.x < PH) ytab[threadIdx.x] = axis_bin2(g.start_h, threadIdx.x, g.bin_h, ext.h);
        else if (threadIdx.x >= 32 && threadIdx.x < 32 + PW) xtab[threadIdx.x - 32] = axis_bin2(g.start_w, threadIdx.x - 32, g.bin_w, ext.w);
        __syncthreads();
        const float4* fb = reinterpret_cast<const float4*>(lv.feat[l] + (size_t)g.batch * H * W * C);
        float4* ob = reinterpret_cast<float4*>(out + (size_t)n * PH * PW * C);
        const int per_roi = PH * PW * C4;
        for (int o = threadIdx.x; o < per_roi; o += blockDim.x) {
            const int c4 = o % C4;
            const int bin = o / C4;
            const AxisBin& by = ytab[bin / PW];
            const AxisBin& bx = xtab[bin % PW];
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < by.n; ++r) {
                const float4* rowp = fb + (size_t)by.idx[r] * W * C4 + c4;
                const float wy = by.w[r];
                for (int c = 0; c < bx.n; ++c) {
                    const float4 v = __ldg(rowp + (size_t)bx.idx[c] * C4);
                    const float w = wy * bx.w[c];
                    acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
                }
            }
            ob[o] = acc;
        }
    }
}

// NHWC features [B,H,W,C] (one level) -> the reference's public output layout [R, C, PH, PW].  One CTA per RoI; a slab of CS
// channels x (PH*PW) bins of a RoI is one contiguous run of the output: it is assembled in shared memory and written with a
// single bulk asynchronous copy (cp.async.bulk), so the HBM write stream never goes through the LSU.
static __global__ void __launch_bounds__(256) roi_align_fast_nchw_out_kernel(const float* __restrict__ feat, const float* __restrict__ rois,
                                                                             long long num_rois, int roi_cols, int C, int CS, int H, int W, int PH,
                                                                             int PW, float scale, float* __restrict__ out) {
    extern __shared__ __align__(128) uint8_t roi_smem[];
    float* tile = reinterpret_cast<float*>(roi_smem);             // [CS][PH*PW]
    __shared__ AxisBin ytab[kMaxPooled];
    __shared__ AxisBin xtab[kMaxPooled];
    const int C4 = C >> 2, bins = PH * PW, CS4 = CS >> 2;
    const uint32_t tile_bytes = (uint32_t)(CS * bins * 4);
    for (long long n = blockIdx.x; n < num_rois; n += gridDim.x) {
        const RoiGeom g = roi_geom(rois + n * roi_cols, roi_cols, scale, PH, PW, 2);
        __syncthreads();
        if (threadIdx.x < PH) ytab[threadIdx.x] = axis_bin2(g.start_h, threadIdx.x, g.bin_h, H);
        else if (threadIdx.x >= 32 && threadIdx.x < 32 + PW) xtab[threadIdx.x - 32] = axis_bin2(g.start_w, threadIdx.x - 32, g.bin_w, W);
        const float4* fbase = reinterpret_cast<const float4*>(feat + (size_t)g.batch * H * W * C);
        for (int c0 = 0; c0 < C; c0 += CS) {
            // the previous bulk copy must have finished reading the tile before it is overwritten
            if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            __syncthreads();
            const float4* fb = fbase + (c0 >> 2);
            for (int o = threadIdx.x; o < bins * CS4; o += blockDim.x) {
                const int c4 = o % CS4;
                const int bin = o / CS4;
                const AxisBin& by = ytab[bin / PW];
                const AxisBin& bx = xtab[bin % PW];
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int r = 0; r < by.n; ++r) {
                    const float4* rowp = fb + (size_t)by.idx[r] * W * C4 + c4;
                    const float wy = by.w[r];
                    for (int c = 0; c < bx.n; ++c) {
                        const float4 v = __ldg(rowp + (size_t)bx.idx[c] * C4);
                        const float w = wy * bx.w[c];
                        acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
                    }
                }
                float* t = tile + (size_t)(c4 * 4) * bins + bin;
                t[0] = acc.x; t[bins] = acc.y; t[2 * bins] = acc.z; t[3 * bins] = acc.w;
            }
            fence_proxy_async_smem();
            __syncthreads();
            if (threadIdx.x == 0) {
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(out + ((size_t)n * C + c0) * bins), "r"(smem_u32(tile)), "r"(tile_bytes) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ---------------------------------------------------------------------------------- shared-memory-resident map variant
// When a slab of kSlabC channels of the whole [H,W] map fits in shared memory (H*W*48 B + tables <= 227 KB: any map up to
// ~5000 cells, e.g. the 50x68 stride-16 map of the microbench), the gathers never leave the SM: a CTA loads one 8-channel
// slab as two planes of float4 (channels 0-3 / 4-7) indexed by the pixel number with its low 3 bits XOR-ed with bits 3..5
// (the 128-bit tap loads of a quarter-warp then fall in different bank groups for the common bin strides 1, 2, 4, 8), then
// sweeps a chunk of RoIs.  The per-RoI AxisBin tables are computed once by roi_tables_kernel (they are shared by all
// C/8 slabs), each warp copies the tables of a group of RoIs into its private shared-memory area (no block barriers), lanes
// run over (RoI, bin) with the 8 channels in registers, and the stores of a warp cover 32 consecutive bins of one channel
// plane (coalesced).  Arithmetic and summation order are those of roi_align_fast_nhwc_kernel => identical results.
struct __align__(16) AxisBinPacked {
    float w[4];
    unsigned short idx[4];   // x taps: column; y taps: row * W (pixel index of the row start)
    int n;
    int batch;               // entry 0 of a RoI: batch index (-1: skip)
};
static constexpr int kSlabC = 8;
__host__ __device__ __forceinline__ int slab_swizzle(int p) { return p ^ ((p >> 3) & 7); }

static __global__ void __launch_bounds__(256) roi_tables_kernel(const float* __restrict__ rois, long long num_rois, int roi_cols, float scale, int H,
                                                                int W, int PH, int PW, int batch, AxisBinPacked* __restrict__ tab) {
    const int ents = PH + PW;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= num_rois * ents) return;
    const long long n = t / ents;
    const int e = (int)(t % ents);
    const RoiGeom g = roi_geom(rois + n * roi_cols, roi_cols, scale, PH, PW, 2);
    const AxisBin b = e < PH ? axis_bin2(g.start_h, e, g.bin_h, H) : axis_bin2(g.start_w, e - PH, g.bin_w, W);
    AxisBinPacked o;
#pragma unroll
    for (int j = 0; j < 4; ++j) { o.w[j] = b.w[j]; o.idx[j] = (unsigned short)(e < PH ? b.idx[j] * W : b.idx[j]); }
    o.n = b.n;
    o.batch = (g.batch >= 0 && g.batch < batch) ? g.batch : -1;
    tab[t] = o;
}

template <int PH, int PW, bool kBatched>
static __global__ void __launch_bounds__(768, 1) roi_align_smem_map_kernel(const float* __restrict__ feat, const AxisBinPacked* __restrict__ tab,
                                                                          long long num_rois, int C, int HW, int num_items, int num_chunks,
                                                                          int group, float* __restrict__ out) {
    extern __shared__ __align__(128) uint8_t roi_smem[];
    constexpr int ENTS = PH + PW, BINS = PH * PW;
    float* map = reinterpret_cast<float*>(roi_smem);                                              // [2][HW8] float4, swizzled
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int HW8 = (HW + 7) & ~7;
    const float4* map4 = reinterpret_cast<const float4*>(map);
    const size_t map_bytes = (size_t)HW8 * kSlabC * 4;
    uint4* wtab = reinterpret_cast<uint4*>(roi_smem + map_bytes) + (size_t)warp * group * ENTS * 2;  // this warp's [group][ENTS] tables
    const int slabs_per_image = C / kSlabC;
    const long long chunk_len = (num_rois + num_chunks - 1) / num_chunks;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int chunk = item % num_chunks;
        const int slab = item / num_chunks;               // (image, channel slab)
        const int image = slab / slabs_per_image;
        const int c0 = (slab % slabs_per_image) * kSlabC;
        __syncthreads();                                  // everyone is done with the previous slab
        const float* src = feat + ((size_t)image * C + c0) * HW;
        for (int i = threadIdx.x; i < kSlabC * HW; i += blockDim.x) {
            const int c = i / HW, p = i - c * HW;
            map[((size_t)(c >> 2) * HW8 + slab_swizzle(p)) * 4 + (c & 3)] = __ldg(src + i);
        }
        __syncthreads();
        const long long r_begin = chunk * chunk_len;
        const long long r_end = r_begin + chunk_len < num_rois ? r_begin + chunk_len : num_rois;
        for (long long g0 = r_begin + (long long)warp * group; g0 < r_end; g0 += (long long)nwarps * group) {
            const int nr = (int)(r_end - g0 < group ? r_end - g0 : group);
            __syncwarp();
            // weights and (indices, n, batch) of an entry go to two separate arrays: consecutive entries are then consecutive
            // 16-byte units (conflict-free for the 7 or 14 x-entries a quarter-warp reads)
            const uint4* gsrc = reinterpret_cast<const uint4*>(tab + g0 * ENTS);
            for (int i = lane; i < nr * ENTS * 2; i += 32) wtab[(i & 1) * group * ENTS + (i >> 1)] = __ldg(gsrc + i);
            __syncwarp();
            const uint4* wmeta = wtab + group * ENTS;
            for (int t = lane; t < nr * BINS; t += 32) {
                const int rl = t / BINS, bin = t - rl * BINS;
                const int py = bin / PW, px = bin - py * PW;
                const int iy = rl * ENTS + py, ix = rl * ENTS + PH + px;
                const uint4 ymeta = wmeta[iy], xmeta = wmeta[ix];
                if (kBatched && (int)wmeta[rl * ENTS].w != image) continue;
                const float4 wy4 = *reinterpret_cast<const float4*>(wtab + iy);
                const float4 wx4 = *reinterpret_cast<const float4*>(wtab + ix);
                const float wy[4] = {wy4.x, wy4.y, wy4.z, wy4.w}, wx[4] = {wx4.x, wx4.y, wx4.z, wx4.w};
                const int yi[4] = {(int)(ymeta.x & 0xffff), (int)(ymeta.x >> 16), (int)(ymeta.y & 0xffff), (int)(ymeta.y >> 16)};
                const int xi[4] = {(int)(xmeta.x & 0xffff), (int)(xmeta.x >> 16), (int)(xmeta.y & 0xffff), (int)(xmeta.y >> 16)};
                const int ny = (int)ymeta.z, nx = (int)xmeta.z;
                float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (r < ny) {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            if (c < nx) {
                                const int sp = slab_swizzle(yi[r] + xi[c]);
                                const float4 v0 = map4[sp], v1 = map4[HW8 + sp];
                                const float w = wy[r] * wx[c];
                                a0.x = fmaf(w, v0.x, a0.x); a0.y = fmaf(w, v0.y, a0.y); a0.z = fmaf(w, v0.z, a0.z); a0.w = fmaf(w, v0.w, a0.w);
                                a1.x = fmaf(w, v1.x, a1.x); a1.y = fmaf(w, v1.y, a1.y); a1.z = fmaf(w, v1.z, a1.z); a1.w = fmaf(w, v1.w, a1.w);
                            }
                        }
                    }
                }
                float* o = out + ((size_t)(g0 + rl) * C + c0) * BINS + bin;
                o[0] = a0.x; o[BINS] = a0.y; o[2 * BINS] = a0.z; o[3 * BINS] = a0.w;
                o[4 * BINS] = a1.x; o[5 * BINS] = a1.y; o[6 * BINS] = a1.z; o[7 * BINS] = a1.w;
            }
        }
    }
}

// ---------------------------------------------------------------------------------- backward (training-side caller of b1-b4)
// d(features) of RoIAlign: every pooled gradient element is scattered to the 4 cells of each of its samples with the bilinear
// weights / sample count.  Same atomic scatter as the reference kernel (lib/cppcuda_cffi/src/cuda/roi_align_backward_cuda_kernel.cu
// :100-207): fp32 atomics, so the summation order (and the last bits) vary from run to run exactly as they do there.  One CTA per
// RoI; the 1-D sample tables are built once per RoI and shared by all channels; a warp reads a contiguous run of top_diff.
static __global__ void __launch_bounds__(256) roi_align_backward_nchw_kernel(const float* __restrict__ top_diff, const float* __restrict__ rois,
                                                                             long long num_rois, int roi_cols, int C, int H, int W, int PH, int PW,
                                                                             float scale, int sampling_ratio, float* __restrict__ bottom_diff) {
    __shared__ AxisTap ytab[kMaxAxisSamples];
    __shared__ AxisTap xtab[kMaxAxisSamples];
    for (long long n = blockIdx.x; n < num_rois; n += gridDim.x) {
        const RoiGeom g = roi_geom(rois + n * roi_cols, roi_cols, scale, PH, PW, sampling_ratio);
        const bool tabled = PH * g.grid_h <= kMaxAxisSamples && PW * g.grid_w <= kMaxAxisSamples;
        __syncthreads();
        if (tabled) {
            for (int i = threadIdx.x; i < PH * g.grid_h; i += blockDim.x)
                ytab[i] = axis_tap(sample_coord(g.start_h, i / g.grid_h, g.bin_h, i % g.grid_h, g.grid_h), H);
            for (int i = threadIdx.x; i < PW * g.grid_w; i += blockDim.x)
                xtab[i] = axis_tap(sample_coord(g.start_w, i / g.grid_w, g.bin_w, i % g.grid_w, g.grid_w), W);
        }
        __syncthreads();
        const float count = (float)(g.grid_h * g.grid_w);
        const float* td = top_diff + (size_t)n * C * PH * PW;
        float* bd = bottom_diff + (size_t)g.batch * C * H * W;
        const int per_roi = C * PH * PW;
        for (int o = threadIdx.x; o < per_roi; o += blockDim.x) {
            const int pw = o % PW, ph = (o / PW) % PH, c = o / (PW * PH);
            const float gtop = td[o];
            float* plane = bd + (size_t)c * H * W;
            for (int iy = 0; iy < g.grid_h; ++iy) {
                const AxisTap ty = tabled ? ytab[ph * g.grid_h + iy] : axis_tap(sample_coord(g.start_h, ph, g.bin_h, iy, g.grid_h), H);
                for (int ix = 0; ix < g.grid_w; ++ix) {
                    const AxisTap tx = tabled ? xtab[pw * g.grid_w + ix] : axis_tap(sample_coord(g.start_w, pw, g.bin_w, ix, g.grid_w), W);
                    if (!(ty.valid && tx.valid)) continue;
                    // g_k = top_diff * w_k / count, evaluated left to right as the reference does (:187-190)
                    atomicAdd(plane + ty.lo * W + tx.lo, __fdiv_rn(__fmul_rn(gtop, __fmul_rn(ty.wl, tx.wl)), count));
                    atomicAdd(plane + ty.lo * W + tx.hi, __fdiv_rn(__fmul_rn(gtop, __fmul_rn(ty.wl, tx.wh)), count));
                    atomicAdd(plane + ty.hi * W + tx.lo, __fdiv_rn(__fmul_rn(gtop, __fmul_rn(ty.wh, tx.wl)), count));
                    atomicAdd(plane + ty.hi * W + tx.hi, __fdiv_rn(__fmul_rn(gtop, __fmul_rn(ty.wh, tx.wh)), count));
                }
            }
        }
    }
}

}  // namespace dt

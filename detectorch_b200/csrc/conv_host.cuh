// detectorch_b200 -- host side of the wgmma conv/GEMM engine: TMA descriptor construction,
// tile-geometry selection and launch.  No torch types; raw device pointers only.
#pragma once
#include <cudaTypedefs.h>
#include <stdlib.h>
#include <string.h>

#include "conv_wgmma.cuh"

namespace dt {

// cuTensorMapEncodeTiled is a driver entry point; fetch it through the runtime so that the
// library links against cudart only (libcuda is resolved by the driver at load time).
inline PFN_cuTensorMapEncodeTiled_v12000 get_tmap_encode() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
        if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) {
            fprintf(stderr, "[detectorch_b200] cuTensorMapEncodeTiled unavailable (%s)\n", cudaGetErrorString(e));
            return nullptr;
        }
        fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
    }
    return fn;
}

// 4D fp32 tensor map {d0 (contiguous), d1, d2, d3} with byte strides s1,s2,s3, SWIZZLE_128B
inline bool make_tmap_4d(CUtensorMap* tm, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t s1,
                         uint64_t s2, uint64_t s3, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3, uint32_t e1 = 1,
                         uint32_t e2 = 1) {
    auto fn = get_tmap_encode();
    if (!fn) return false;
    cuuint64_t dims[4] = {d0, d1, d2, d3};
    cuuint64_t strides[3] = {s1, s2, s3};
    cuuint32_t box[4] = {b0, b1, b2, b3};
    cuuint32_t estr[4] = {1, e1, e2, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr,
                "[detectorch_b200] cuTensorMapEncodeTiled(4d) failed: %d dims=(%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu) "
                "box=(%u,%u,%u,%u) estr=(%u,%u)\n",
                (int)r, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)d3,
                (unsigned long long)s1, (unsigned long long)s2, (unsigned long long)s3, b0, b1, b2, b3, e1, e2);
        return false;
    }
    return true;
}

inline bool make_tmap_2d(CUtensorMap* tm, const void* base, uint64_t d0, uint64_t d1, uint64_t s1, uint32_t b0, uint32_t b1) {
    auto fn = get_tmap_encode();
    if (!fn) return false;
    cuuint64_t dims[2] = {d0, d1};
    cuuint64_t strides[1] = {s1};
    cuuint32_t box[2] = {b0, b1};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "[detectorch_b200] cuTensorMapEncodeTiled(2d) failed: %d dims=(%llu,%llu) stride=%llu box=(%u,%u)\n", (int)r,
                (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)s1, b0, b1);
        return false;
    }
    return true;
}

// 2D fp16 weight map {K (contiguous), rows}, box {32 elements = 64 bytes, rows}, SWIZZLE_64B (KIND_F16X3)
inline bool make_tmap_2d_f16(CUtensorMap* tm, const void* base, uint64_t d0, uint64_t d1, uint64_t s1, uint32_t b0, uint32_t b1) {
    auto fn = get_tmap_encode();
    if (!fn) return false;
    cuuint64_t dims[2] = {d0, d1};
    cuuint64_t strides[1] = {s1};
    cuuint32_t box[2] = {b0, b1};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "[detectorch_b200] cuTensorMapEncodeTiled(2d f16) failed: %d dims=(%llu,%llu) stride=%llu box=(%u,%u)\n", (int)r,
                (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)s1, b0, b1);
        return false;
    }
    return true;
}

// 4D fp16 plane map {C (contiguous), W, H, N}, box {32 channels = 64 bytes, ...}, SWIZZLE_64B (activations handed over as hi/lo planes)
inline bool make_tmap_4d_f16(CUtensorMap* tm, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t s1, uint64_t s2,
                             uint64_t s3, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3, uint32_t e1 = 1, uint32_t e2 = 1) {
    auto fn = get_tmap_encode();
    if (!fn) return false;
    cuuint64_t dims[4] = {d0, d1, d2, d3};
    cuuint64_t strides[3] = {s1, s2, s3};
    cuuint32_t box[4] = {b0, b1, b2, b3};
    cuuint32_t estr[4] = {1, e1, e2, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "[detectorch_b200] cuTensorMapEncodeTiled(4d f16) failed: %d dims=(%llu,%llu,%llu,%llu) box=(%u,%u,%u,%u)\n", (int)r,
                (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)d3, b0, b1, b2, b3);
        return false;
    }
    return true;
}

// A conv layer instance: everything needed to (re)launch it.  Built once per (layer, shape).
struct ConvLayer {
    ConvParams p;
    int block_n;
    int nmain = 1;      // rotating main-term accumulators (3 = shorter truncating accumulation chains; 64-wide tiles)
    int kind = KIND_TF32X3;
    dim3 grid;
    bool valid = false;
};

// Logical description of one convolution over NHWC fp32 tensors.
struct ConvSpec {
    const float* x; int N, H, W, Cin;          // input  [N,H,W,Cin], Cin % 32 == 0
    int x_pix_stride;                          // floats between consecutive pixels of x (>= Cin; lets x be a channel slice)
    const void* w_hi; const void* w_lo;        // [Cout_rows][kh*kw*Cin] K-major: fp32 (w, w - trunc_tf32(w)) or fp16 (hi, lo) for KIND_F16X3
    int kind;                                  // ConvKind
    int* range_flag;                           // KIND_F16X3: device flag raised when an activation does not fit fp16
    int Cout;                                  // output channels, multiple of 4
    int kh, kw, pad, stride;
    const float* scale; const float* shift;    // [Cout]
    float* y; int y_pix_stride;                // output [N,Ho,Wo,*], y_pix_stride floats between pixels (>= Cout)
    // optional output remap (transposed conv): pixel (n,h,w) is written at y + ((n*Hy + h*ys + yo)*Wy + w*ys + xo)*y_pix_stride
    int out_h, out_w, out_step, out_y0, out_x0;   // out_step==0 -> plain [N,Ho,Wo]
    const float* residual; int res_pix_stride;    // RES_TILE: same geometry as the (plain) output
    // RES_STAGED: the convolution whose result is the residual, run by the same launch (phase 1; its x, N, H, W, Cin, x_pix_stride,
    // weights, filter geometry, taps, scale and shift are read; the output, kind and passes are this spec's).  It must give the same
    // output extents and, by conv_tile, the same tile shape; its input is fp32.
    const ConvSpec* phase1;
    const float* up_src; int up_h, up_w;          // RES_UPSAMPLE2X
    int res_mode, relu, sigmoid_ch, passes;
    // fp16 hi/lo plane hand-over between two KIND_F16X3 layers (dense channel stride only): x / y then point at the HIGH plane and
    // x_lo / y_lo at the LOW plane, each [N,H,W,C] fp16
    const void* x_lo; void* y_lo;
    int tap0, ntaps;                              // K-split: only filter taps [tap0, tap0+ntaps) (ntaps == 0: all kh*kw)
    int force_block_n;                            // 0 = auto (64 or 128)
    int precise;                                  // 64-wide tiles with 3 rotating main-term accumulators (shorter accumulation chains)
    int im_stride;                                // image-shaped output at this stride: pixels outside each image can be zeroed (ConvParams::im_info)
};

inline void choose_box(int Wo, int Ho, int N, int max_w, int* wbox, int* hbox, int* nbox) {
    long best_tiles = -1;
    int bw = 1, bh = 1, bn = 1;
    for (int w = 1; w <= Wo && w <= 128 && w <= max_w; ++w) {
        for (int h = 1; h <= Ho && w * h <= 128; ++h) {
            int n = 128 / (w * h);
            if (n > N) n = N;
            if (n < 1) n = 1;
            long tiles = (long)ceil_div(Wo, w) * ceil_div(Ho, h) * ceil_div(N, n);
            if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && w > bw)) {
                best_tiles = tiles; bw = w; bh = h; bn = n;
            }
        }
    }
    *wbox = bw; *hbox = bh; *nbox = bn;
}

// Persistent launch geometry: work items = M-tiles x N-tiles; one CTA per SM, each looping over items blockIdx.x, + gridDim.x, ...
inline void finish_grid(ConvLayer* L, int n_tiles) {
    ConvParams& p = L->p;
    p.m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
    p.n_tiles = n_tiles;
    const int items = p.m_tiles * p.n_tiles;
    L->grid = dim3((unsigned)(items < num_sms() ? items : num_sms()), 1, 1);
    L->valid = true;
}

// Tile width and rotating main-term accumulators of a convolution.
// Tiles are at most 128 channels wide: the main and cross accumulators of a 64 x 128 warpgroup tile are 128 registers per thread,
// which is what the register file leaves with two MMA warpgroups per SM.  A wider request (256) runs as 128-wide tiles.
inline void conv_tile(const ConvSpec& s, int* block_n, int* nmain) {
    int bn = s.force_block_n;
    if (bn == 0 || bn > 128) bn = s.Cout > 64 ? 128 : 64;
    // tf32 k-steps are half as long as fp16 ones: a long-K tf32 layer's accumulation chain is twice as long, and the 3xTF32 engine met the
    // 1e-4 mask-logit bar only with the main term rotated over three accumulators (64-wide tiles)
    if (s.precise || (s.kind != KIND_F16X3 && s.kh * s.kw * (s.Cin / 32) > 16)) bn = 64;
    // 64-wide tiles rotate the main term over 3 accumulators (same register budget as one 128-wide pair) -- except at K <= 256, where
    // one accumulator already is a chain of at most 16 k-blocks
    const int ntaps = s.ntaps > 0 ? s.ntaps : s.kh * s.kw;
    *block_n = bn;
    *nmain = (bn == 64 && (s.precise || ntaps * (s.Cin / 32) > 8)) ? 3 : 1;
}

// The phase-1 spec of a RES_STAGED launch as a launch of its own into the same output (what conv_build checks it against)
inline ConvSpec phase1_as_launch(const ConvSpec& s) {
    ConvSpec t = *s.phase1;
    t.kind = s.kind; t.range_flag = s.range_flag; t.passes = s.passes; t.force_block_n = s.force_block_n; t.precise = s.precise;
    t.y = s.y; t.y_pix_stride = s.y_pix_stride; t.y_lo = nullptr; t.out_step = 0;
    t.res_mode = RES_NONE; t.relu = 0; t.sigmoid_ch = 0; t.im_stride = 0; t.phase1 = nullptr;
    return t;
}

// Whether a RES_STAGED launch can serve the spec: phase 1 has the same tile shape and output extents, fp32 input, and phase 2 writes
// a plain fp32 output.  Equal extents give equal boxes (choose_box) while both strides allow 128-pixel-wide boxes.
inline bool conv_staged_ok(const ConvSpec& s) {
    if (!s.phase1 || s.phase1->x_lo || s.y_lo || s.out_step != 0) return false;
    const ConvSpec t = phase1_as_launch(s);
    int bn, nm, bn1, nm1;
    conv_tile(s, &bn, &nm);
    conv_tile(t, &bn1, &nm1);
    return bn == bn1 && nm == nm1 && t.Cout == s.Cout && t.N == s.N && (t.H + 2 * t.pad - t.kh) / t.stride == (s.H + 2 * s.pad - s.kh) / s.stride &&
           (t.W + 2 * t.pad - t.kw) / t.stride == (s.W + 2 * s.pad - s.kw) / s.stride && 256 / t.stride >= 128 && 256 / s.stride >= 128;
}

inline bool conv_build(const ConvSpec& s, ConvLayer* L) {
    memset(&L->p, 0, sizeof(ConvParams));
    ConvParams& p = L->p;
    if (s.Cin % 32 != 0 || s.Cout % 4 != 0) {
        fprintf(stderr, "[detectorch_b200] conv_build: Cin must be a multiple of 32 and Cout of 4 (got %d, %d)\n", s.Cin, s.Cout);
        return false;
    }
    const int Ho = (s.H + 2 * s.pad - s.kh) / s.stride + 1;
    const int Wo = (s.W + 2 * s.pad - s.kw) / s.stride + 1;
    int wbox, hbox, nbox;
    choose_box(Wo, Ho, s.N, 256 / s.stride, &wbox, &hbox, &nbox);
    int bn, nmain;
    conv_tile(s, &bn, &nmain);
    if (bn != 64 && bn != 128) { fprintf(stderr, "[detectorch_b200] conv_build: unsupported tile width %d\n", bn); return false; }
    L->block_n = bn;
    const int K = s.kh * s.kw * s.Cin;
    const uint64_t xs = (uint64_t)s.x_pix_stride * 4;
    if (s.x_lo) {
        if (s.kind != KIND_F16X3 || s.x_pix_stride != s.Cin) { fprintf(stderr, "[detectorch_b200] conv_build: fp16 input planes need the f16 kind and a dense layout\n"); return false; }
        const uint64_t hs = (uint64_t)s.Cin * 2;
        if (!make_tmap_4d_f16(&p.tm_a, s.x, s.Cin, s.W, s.H, s.N, hs, hs * s.W, hs * s.W * s.H, 32, wbox * s.stride, hbox * s.stride, nbox, s.stride, s.stride) ||
            !make_tmap_4d_f16(&p.tm_a2, s.x_lo, s.Cin, s.W, s.H, s.N, hs, hs * s.W, hs * s.W * s.H, 32, wbox * s.stride, hbox * s.stride, nbox, s.stride, s.stride))
            return false;
        p.a_planes = 1;
    } else if (!make_tmap_4d(&p.tm_a, s.x, s.Cin, s.W, s.H, s.N, xs, xs * s.W, xs * s.W * s.H, 32, wbox * s.stride, hbox * s.stride, nbox,
                             s.stride, s.stride))
        return false;
    if (s.kind == KIND_F16X3) {
        if (!make_tmap_2d_f16(&p.tm_bhi, s.w_hi, K, s.Cout, (uint64_t)K * 2, 32, bn)) return false;
        if (!make_tmap_2d_f16(&p.tm_blo, s.w_lo ? s.w_lo : s.w_hi, K, s.Cout, (uint64_t)K * 2, 32, bn)) return false;
    } else {
        if (!make_tmap_2d(&p.tm_bhi, s.w_hi, K, s.Cout, (uint64_t)K * 4, 32, bn)) return false;
        if (!make_tmap_2d(&p.tm_blo, s.w_lo ? s.w_lo : s.w_hi, K, s.Cout, (uint64_t)K * 4, 32, bn)) return false;
    }
    L->kind = s.kind == KIND_F16X3 ? KIND_F16X3 : KIND_TF32X3;
    p.range_flag = s.range_flag;
    const uint64_t ys = (uint64_t)s.y_pix_stride * 4;
    if (s.y_lo) {
        if (s.kind != KIND_F16X3 || s.out_step != 0 || s.y_pix_stride != s.Cout || s.res_mode != RES_NONE || (s.Cout % 32) != 0) {
            fprintf(stderr, "[detectorch_b200] conv_build: fp16 output planes need the f16 kind, a dense layout, Cout %% 32 == 0 and no residual\n");
            return false;
        }
        const uint64_t hs = (uint64_t)s.Cout * 2;
        if (!make_tmap_4d_f16(&p.tm_d, s.y, s.Cout, Wo, Ho, s.N, hs, hs * Wo, hs * Wo * Ho, 32, wbox, hbox, nbox) ||
            !make_tmap_4d_f16(&p.tm_d2, s.y_lo, s.Cout, Wo, Ho, s.N, hs, hs * Wo, hs * Wo * Ho, 32, wbox, hbox, nbox))
            return false;
        p.out_planes = 1;
    } else if (s.out_step == 0) {
        if (!make_tmap_4d(&p.tm_d, s.y, s.Cout, Wo, Ho, s.N, ys, ys * Wo, ys * Wo * Ho, 32, wbox, hbox, nbox)) return false;
    } else {
        // strided scatter view: logical (w,h) -> physical (w*step + x0, h*step + y0) of an [N,out_h,out_w] map
        const float* base = s.y + ((size_t)s.out_y0 * s.out_w + s.out_x0) * s.y_pix_stride;
        if (!make_tmap_4d(&p.tm_d, base, s.Cout, Wo, Ho, s.N, ys * s.out_step, ys * s.out_w * s.out_step, ys * s.out_w * s.out_h, 32,
                          wbox, hbox, nbox))
            return false;
    }
    if (s.res_mode == RES_TILE) {
        const uint64_t rs = (uint64_t)s.res_pix_stride * 4;
        if (!make_tmap_4d(&p.tm_r, s.residual, s.Cout, Wo, Ho, s.N, rs, rs * Wo, rs * Wo * Ho, 32, wbox, hbox, nbox)) return false;
    }
    p.scale = s.scale; p.shift = s.shift;
    p.up_src = s.up_src; p.up_h = s.up_h; p.up_w = s.up_w;
    p.cin_blocks = s.Cin / 32;
    p.kh = s.kh; p.kw = s.kw; p.pad_w = p.pad_h = s.pad; p.stride_w = p.stride_h = s.stride;
    p.tap0 = s.ntaps > 0 ? s.tap0 : 0; p.ntaps = s.ntaps > 0 ? s.ntaps : s.kh * s.kw;
    if (p.tap0 < 0 || p.tap0 + p.ntaps > s.kh * s.kw) { fprintf(stderr, "[detectorch_b200] conv_build: bad tap range\n"); return false; }
    p.tiles_w = ceil_div(Wo, wbox); p.tiles_h = ceil_div(Ho, hbox); p.tiles_n = ceil_div(s.N, nbox);
    p.wbox = wbox; p.hbox = hbox; p.nbox = nbox;
    p.wo = Wo; p.ho = Ho; p.nimg = s.N;
    p.cout = s.Cout;
    p.a_tile_bytes = wbox * hbox * nbox * 128;
    p.relu = s.relu; p.sigmoid_ch = s.sigmoid_ch; p.res_mode = s.res_mode;
    p.passes = s.passes == 1 ? 1 : 3;
    p.im_stride = s.out_step == 0 ? s.im_stride : 0;
    L->nmain = nmain;
    if (s.res_mode == RES_STAGED) {
        // phase 1 is built as a launch of its own into the same output; its operands then move into this launch
        ConvLayer L1;
        if (!conv_staged_ok(s) || !conv_build(phase1_as_launch(s), &L1) || L1.p.wbox != wbox || L1.p.hbox != hbox || L1.p.nbox != nbox) {
            fprintf(stderr, "[detectorch_b200] conv_build: the two phases need the same output, tile shape and box, fp32 phase-1 input and a "
                            "plain fp32 output\n");
            return false;
        }
        p.tm_a1 = L1.p.tm_a; p.tm_bhi1 = L1.p.tm_bhi; p.tm_blo1 = L1.p.tm_blo;
        p.scale1 = L1.p.scale; p.shift1 = L1.p.shift;
        p.cin_blocks1 = L1.p.cin_blocks; p.kw1 = L1.p.kw; p.tap01 = L1.p.tap0; p.ntaps1 = L1.p.ntaps;
        p.pad1 = L1.p.pad_w; p.stride1 = L1.p.stride_w;
    }
    finish_grid(L, ceil_div(s.Cout, bn));
    return true;
}

// The 7x7 stride-2 stem (3 input channels) as an implicit GEMM without an im2col buffer: the image is repacked once as
// zero-bordered NHWC4 [B, Hp, Wp, 4]; for filter row ky the 7 taps x 4 channels of an output pixel are 28 CONTIGUOUS floats
// starting at padded pixel 2*ow, so a TMA descriptor whose "pixel" dimension has an OVERLAPPING stride of 8 floats
// (2 pixels) delivers, per ky, one 32-float K-block per output pixel straight into the swizzled A tile (last 4 floats
// hit zero weights).  K = 7 x 32.  H uses elementStride 2.
inline bool conv_build_stem(const float* x4, int B, int Hp, int Wp, int H1, int W1, const void* w_hi, const void* w_lo, const float* scale,
                            const float* shift, float* y, int passes, ConvLayer* L, int kind = KIND_TF32X3, int* range_flag = nullptr) {
    memset(&L->p, 0, sizeof(ConvParams));
    ConvParams& p = L->p;
    int wbox, hbox, nbox;
    choose_box(W1, H1, B, 256, &wbox, &hbox, &nbox);
    const int bn = 64;
    L->block_n = bn;
    if (kind == KIND_F16X3) {
        // x4 holds two fp16 planes [B, Hp, Wp, 4] back to back (hi, lo): same overlapping-stride window, 16 bytes (2 pixels) per step
        if (Wp & 1) { fprintf(stderr, "[detectorch_b200] conv_build_stem: the fp16 planes need an even padded width (got %d)\n", Wp); return false; }
        const __half* xh = reinterpret_cast<const __half*>(x4);
        const __half* xl = xh + (size_t)B * Hp * Wp * 4;
        const uint64_t rowh = (uint64_t)Wp * 8;
        if (!make_tmap_4d_f16(&p.tm_a, xh, 32, W1, Hp, B, 16, rowh, rowh * Hp, 32, wbox, hbox * 2, nbox, 1, 2) ||
            !make_tmap_4d_f16(&p.tm_a2, xl, 32, W1, Hp, B, 16, rowh, rowh * Hp, 32, wbox, hbox * 2, nbox, 1, 2))
            return false;
        p.a_planes = 1;
        if (!make_tmap_2d_f16(&p.tm_bhi, w_hi, 224, 64, 224 * 2, 32, bn)) return false;
        if (!make_tmap_2d_f16(&p.tm_blo, w_lo, 224, 64, 224 * 2, 32, bn)) return false;
    } else {
        const uint64_t row = (uint64_t)Wp * 16;
        if (!make_tmap_4d(&p.tm_a, x4, 32, W1, Hp, B, 32, row, row * Hp, 32, wbox, hbox * 2, nbox, 1, 2)) return false;
        if (!make_tmap_2d(&p.tm_bhi, w_hi, 224, 64, 224 * 4, 32, bn)) return false;
        if (!make_tmap_2d(&p.tm_blo, w_lo, 224, 64, 224 * 4, 32, bn)) return false;
    }
    L->kind = kind == KIND_F16X3 ? KIND_F16X3 : KIND_TF32X3;
    p.range_flag = range_flag;
    const uint64_t ys = 64 * 4;
    if (!make_tmap_4d(&p.tm_d, y, 64, W1, H1, B, ys, ys * W1, ys * W1 * H1, 32, wbox, hbox, nbox)) return false;
    p.scale = scale; p.shift = shift;
    p.cin_blocks = 1; p.kh = 7; p.kw = 1; p.tap0 = 0; p.ntaps = 7;
    p.pad_w = 0; p.pad_h = 0; p.stride_w = 1; p.stride_h = 2;
    p.tiles_w = ceil_div(W1, wbox); p.tiles_h = ceil_div(H1, hbox); p.tiles_n = ceil_div(B, nbox);
    p.wbox = wbox; p.hbox = hbox; p.nbox = nbox;
    p.wo = W1; p.ho = H1; p.nimg = B; p.cout = 64;
    p.a_tile_bytes = wbox * hbox * nbox * 128;
    p.relu = 1; p.sigmoid_ch = 0; p.res_mode = RES_NONE; p.passes = passes == 1 ? 1 : 3;
    L->nmain = 1;       // K = 7 k-blocks: one main accumulator (see conv_build)
    finish_grid(L, 1);
    return true;
}

template <int BN, int NM, int KIND, bool MASK, bool STAGED>
inline cudaError_t conv_launch_cfg(const ConvLayer& L, cudaStream_t stream) {
    using Cfg = ConvCfg<BN, NM, KIND>;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e =
            cudaFuncSetAttribute(conv_wgmma_kernel<BN, NM, KIND, MASK, STAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    conv_wgmma_kernel<BN, NM, KIND, MASK, STAGED><<<L.grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(L.p);
    return cudaGetLastError();
}

template <int KIND, bool MASK, bool STAGED>
inline cudaError_t conv_launch_tile(const ConvLayer& L, cudaStream_t stream) {
    if (L.block_n == 64)
        return L.nmain == 3 ? conv_launch_cfg<64, 3, KIND, MASK, STAGED>(L, stream) : conv_launch_cfg<64, 1, KIND, MASK, STAGED>(L, stream);
    if (L.block_n == 128 && L.nmain == 1) return conv_launch_cfg<128, 1, KIND, MASK, STAGED>(L, stream);
    return cudaErrorInvalidValue;
}

template <int KIND, bool MASK>
inline cudaError_t conv_launch_kind(const ConvLayer& L, cudaStream_t stream) {
    return L.p.res_mode == RES_STAGED ? conv_launch_tile<KIND, MASK, true>(L, stream) : conv_launch_tile<KIND, MASK, false>(L, stream);
}

inline cudaError_t conv_launch(const ConvLayer& L, cudaStream_t stream) {
    if (!L.valid) return cudaErrorInvalidValue;
    if (L.p.im_info)
        return L.kind == KIND_F16X3 ? conv_launch_kind<KIND_F16X3, true>(L, stream) : conv_launch_kind<KIND_TF32X3, true>(L, stream);
    return L.kind == KIND_F16X3 ? conv_launch_kind<KIND_F16X3, false>(L, stream) : conv_launch_kind<KIND_TF32X3, false>(L, stream);
}

}  // namespace dt

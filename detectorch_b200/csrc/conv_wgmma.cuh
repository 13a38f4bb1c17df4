// detectorch_b200 -- implicit-GEMM convolution / GEMM on Hopper warpgroup MMAs (wgmma, sm_90a).
//
// Replaces every Conv2d / Linear / ConvTranspose2d that the reference runs through
// torch+cuDNN/cuBLAS (reference lib/model/detector.py:17-27,58-59,71-74,89-90,119-121,
// 170-183,212-214; SURVEY.md 2.2 K1/K3/K4/K9/K11).
//
// Data layout: activations are NHWC fp32 in HBM (pixel-major rows of C channels), weights are
// [Cout][kh][kw][Cin] (K-major rows), both fetched by TMA into swizzled shared-memory tiles;
// accumulators live in registers of the two MMA warpgroups.
//
// Precision: the parity contract is fp32 (1e-4, BASELINE.json north_star), but the tensor core has
// no fp32-input MMA.  Both kinds therefore run an error-compensated three-term product
//     D = A_h*B_h + (A_l*B_h + A_h*B_l)
// with the main term and the two cross terms (~2^-11 of the main term) in separate accumulators.
//   KIND_TF32X3: A_h / B_h are the fp32 words themselves (the tensor core reads the top 19 bits), A_l = A - trunc_tf32(A) is
//                written next to the A tile by the MMA warpgroups, B_l is precomputed once per weight tensor.
//   KIND_F16X3 (the engine default, twice the tf32 rate): A_h = fp16(A), A_l = fp16(A - A_h) (22 mantissa bits, like the two tf32
//                pieces); B_h / B_l likewise, precomputed and pre-scaled by a power of two so that B_l stays a normal fp16 number
//                (the epilogue scale undoes it exactly).  The fp32 A tile arrives by TMA and each MMA warpgroup splits its own 64 rows
//                into two 64-byte-row (SWIZZLE_64B) fp16 tiles -- unless the producing layer already wrote the activation as two fp16
//                planes (a_planes / out_planes), in which case TMA delivers the operand tiles directly.  fp16 has a 5-bit exponent:
//                |A| >= 65504 raises a device flag (the engine then reports it; the tf32 kind has no such limit).
// `passes` == 1 runs the plain single-pass product (speed-of-light reference; not fp32-accurate).
//
// Tile: BLOCK_M = 128 output pixels (a wbox x hbox x nbox box of the NHWC output, so the same TMA box geometry loads A for any
// filter tap and stores D, with hardware zero-fill doing the padding and hardware clipping doing the edge masking),
// BLOCK_N = 64 or 128 output channels (two 64 x BLOCK_N register accumulators per MMA warpgroup, plus two more main-term
// accumulators in the NMAIN == 3 form), BLOCK_K = 32 channels of one filter tap per pipeline stage.
//
// Execution model: persistent CTAs (one per SM), 384 threads =
//   warpgroup 0    TMA producer (one thread; the warpgroup gives its registers up to the MMA warpgroups)
//   warpgroups 1-2 MMA + epilogue, rows [0, 64) and [64, 128) of the tile: operand split, wgmma, then scale/shift [+residual]
//                  [ReLU|sigmoid] -> swizzled staging area -> TMA store.  The producer runs ahead into the next tile while a tile
//                  drains, and the stores of a tile overlap the main loop of the next.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace dt {

enum ConvResidualMode { RES_NONE = 0, RES_TILE = 1, RES_UPSAMPLE2X = 2 };
enum ConvKind { KIND_TF32X3 = 0, KIND_F16X3 = 1 };

struct ConvParams {
    CUtensorMap tm_a;      // 4D {C, W, H, N} over the NHWC input (elementStrides carry the conv stride)
    CUtensorMap tm_bhi;    // 2D {K, Cout} weights, box = BLOCK_N rows
    CUtensorMap tm_blo;    // 2D {K, Cout} low parts of the weights
    CUtensorMap tm_d;      // 4D {Cout, Wo, Ho, N} over the NHWC output, box {32, wbox, hbox, nbox}
    CUtensorMap tm_r;      // 4D residual, same geometry as tm_d (RES_TILE only)
    CUtensorMap tm_a2;     // a_planes: the fp16 LOW plane of the input (tm_a is then the fp16 HIGH plane), SWIZZLE_64B boxes of 32 channels
    CUtensorMap tm_d2;     // out_planes: the fp16 LOW plane of the output (tm_d the HIGH plane), SWIZZLE_64B boxes of 32 channels
    const float* scale;    // [Cout] per-channel scale (folded BN gain, or 1)
    const float* shift;    // [Cout] per-channel shift (folded BN bias, or conv bias)
    const float* up_src;   // RES_UPSAMPLE2X: coarser NHWC map [N, up_h, up_w, Cout]
    int up_h, up_w;
    int cin_blocks;        // Cin / 32
    int kh, kw;
    int tap0, ntaps;       // this launch covers filter taps [tap0, tap0 + ntaps) of the kh*kw (a K-split partial convolution; default all)
    int pad_w, pad_h, stride_w, stride_h;   // A-load coordinate = tile origin * stride + tap - pad, per axis
    int tiles_w, tiles_h, tiles_n;
    int m_tiles, n_tiles;  // work items = m_tiles * n_tiles, the N-tile varying fastest
    int wbox, hbox, nbox;
    int wo, ho, nimg;      // output extents (for RES_UPSAMPLE2X bounds)
    int cout;              // true Cout (channels >= cout are never stored: TMA clips)
    int a_tile_bytes;      // wbox*hbox*nbox*128
    int relu;
    int sigmoid_ch;        // channels [0, sigmoid_ch) get a sigmoid (RPN objectness), after bias
    int res_mode;
    int passes;            // 3 = error-compensated three-term product (default), 1 = single pass
    int a_planes;          // KIND_F16X3: the input already is a pair of fp16 planes (hi, lo) written by the producing layer
    int out_planes;        // KIND_F16X3: write the output as a pair of fp16 planes (hi = fp16(y), lo = fp16(y - hi)) instead of fp32
    int* range_flag;       // KIND_F16X3: set to 1 when an activation does not fit fp16 (|x| >= 65504 or NaN); may be null
    int pdl;               // launched with programmatic stream serialization: release the next launch early, wait for the previous one
};

template <int BLOCK_N, int NMAIN, int KIND>
struct ConvCfg {
    static_assert(BLOCK_N == 64 || BLOCK_N == 128, "tile width");
    static_assert(NMAIN == 1 || (NMAIN == 3 && BLOCK_N == 64), "rotating main accumulators: 64-wide tiles only (register budget)");
    static constexpr int BLOCK_M = 128;
    static constexpr int A_BYTES = BLOCK_M * 128;                     // 16 KB: the fp32 A tile as TMA delivers it
    static constexpr int B_ROW_BYTES = KIND == KIND_F16X3 ? 64 : 128; // 32 k-elements per row
    static constexpr int B_BYTES = BLOCK_N * B_ROW_BYTES;
    // tf32: A | A_lo (16 KB each); f16: A (fp32 as delivered) | A_h | A_l (8 KB each; with a_planes TMA fills A_h | A_l).  Then B_h | B_l.
    static constexpr int A_STAGE_BYTES = 2 * A_BYTES;
    static constexpr int STAGE_BYTES = A_STAGE_BYTES + 2 * B_BYTES;
    // epilogue staging: one 16 KB swizzled 128 x 32-channel chunk per 32 output channels (the layout of a tm_d box)
    static constexpr int NCHUNK = BLOCK_N / 32;
    static constexpr int EPI_BYTES = NCHUNK * A_BYTES;
    static constexpr int SMEM_LIMIT = 232448;                         // 227 KB per block on H100
    static constexpr int STAGES_FIT = (SMEM_LIMIT - 1024 - 256 - EPI_BYTES) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;
    static_assert(STAGES >= 2, "pipeline too shallow");
    static constexpr int PIPE_BYTES = STAGES * STAGE_BYTES;
    static constexpr int NUM_BARS = 2 * STAGES + 1;
    static constexpr int SMEM_BYTES = PIPE_BYTES + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static constexpr int THREADS = 384;
    static constexpr int R = BLOCK_N / 2;                             // accumulator registers per thread (64 x BLOCK_N per warpgroup)
    static constexpr int KSTEPS = KIND == KIND_F16X3 ? 2 : 4;         // instructions per 32-element k-block (32 bytes of a row each)
    static_assert(SMEM_BYTES <= SMEM_LIMIT, "exceeds the 227 KB shared-memory limit");
    static_assert(8 * NUM_BARS <= 256, "barrier area");
};

template <int BLOCK_N, int KIND>
__device__ __forceinline__ void conv_mma(float (&d)[BLOCK_N / 2], uint64_t da, uint64_t db) {
    if constexpr (KIND == KIND_F16X3) {
        if constexpr (BLOCK_N == 64) wgmma_f16_n64(d, da, db, 1u); else wgmma_f16_n128(d, da, db, 1u);
    } else {
        if constexpr (BLOCK_N == 64) wgmma_tf32_n64(d, da, db, 1u); else wgmma_tf32_n128(d, da, db, 1u);
    }
}

template <int BLOCK_N, int NMAIN, int KIND>
__global__ void __launch_bounds__(384, 1) conv_wgmma_kernel(const __grid_constant__ ConvParams p) {
    using Cfg = ConvCfg<BLOCK_N, NMAIN, KIND>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int R = Cfg::R;
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment is required by SWIZZLE_128B (TMA and wgmma descriptors)
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t epi_base = smem_base + Cfg::PIPE_BYTES;
    uint8_t* epi_gen = smem_gen + Cfg::PIPE_BYTES;
    const uint32_t bar_base = epi_base + Cfg::EPI_BYTES;
    auto bar_full = [&](int s) { return bar_base + 8u * s; };              // TMA bytes of stage s landed
    auto bar_empty = [&](int s) { return bar_base + 8u * (STAGES + s); };  // the 8 MMA warps are done reading stage s
    const uint32_t bar_res = bar_base + 8u * (2 * STAGES);                 // residual chunks of a tile landed in the staging area

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;
    const int num_kb = p.ntaps * p.cin_blocks;           // pipeline steps per tile: one k-block = 32 channels of one filter tap
    const int num_tiles = p.m_tiles * p.n_tiles;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.tm_a);
        tma_prefetch_desc(&p.tm_bhi);
        if (p.passes == 3) tma_prefetch_desc(&p.tm_blo);
        tma_prefetch_desc(&p.tm_d);
        if (p.res_mode == RES_TILE) tma_prefetch_desc(&p.tm_r);
        if (p.a_planes) tma_prefetch_desc(&p.tm_a2);
        if (p.out_planes) tma_prefetch_desc(&p.tm_d2);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(bar_full(s), 1);
            mbar_init(bar_empty(s), 8);
        }
        mbar_init(bar_res, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (p.pdl) {
        // Everything above touched no global data: with PDL it overlaps the tail of the previous launch.  The next launch in the
        // stream may become resident as soon as every CTA of this grid got here (it then parks in its own griddep_wait).
        griddep_launch_dependents();
        griddep_wait();
    }

    // work item -> tile coordinates.  The N-tile varies fastest so that consecutive items re-read the same A tile from L2.
    auto tile_of = [&](int item, int& w0, int& h0, int& n0img, int& n0) {
        const int nt = item % p.n_tiles;
        int t = item / p.n_tiles;
        const int tw = t % p.tiles_w; t /= p.tiles_w;
        const int th = t % p.tiles_h; t /= p.tiles_h;
        w0 = tw * p.wbox; h0 = th * p.hbox; n0img = t * p.nbox; n0 = nt * BLOCK_N;
    };

    if (wg == 0) {
        // ================================================================ TMA producer
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {
            const uint32_t tx_bytes = (uint32_t)p.a_tile_bytes + (p.passes == 3 ? 2u : 1u) * Cfg::B_BYTES;
            uint32_t it = 0;
            for (int item = blockIdx.x; item < num_tiles; item += gridDim.x) {
                int w0, h0, n0img, n0;
                tile_of(item, w0, h0, n0img, n0);
                for (int kb = 0; kb < num_kb; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(bar_empty(s), ((it / STAGES) & 1u) ^ 1u);
                    const int tap_l = kb / p.cin_blocks;
                    const int cb = kb - tap_l * p.cin_blocks;
                    const int tap = p.tap0 + tap_l;
                    const int kbg = tap * p.cin_blocks + cb;        // k-block index into the full weight row
                    const int fy = tap / p.kw, fx = tap - fy * p.kw;
                    const int xw = w0 * p.stride_w + fx - p.pad_w, xh = h0 * p.stride_h + fy - p.pad_h;
                    const uint32_t st = smem_base + s * Cfg::STAGE_BYTES;
                    mbar_arrive_expect_tx(bar_full(s), tx_bytes);
                    if (KIND == KIND_F16X3 && p.a_planes) {
                        // fp16 planes: the two operand tiles land where the split would have written them
                        tma_load_4d(st + Cfg::A_BYTES, &p.tm_a, bar_full(s), cb * 32, xw, xh, n0img);
                        tma_load_4d(st + Cfg::A_BYTES + Cfg::A_BYTES / 2, &p.tm_a2, bar_full(s), cb * 32, xw, xh, n0img);
                    } else {
                        tma_load_4d(st, &p.tm_a, bar_full(s), cb * 32, xw, xh, n0img);
                    }
                    tma_load_2d(st + Cfg::A_STAGE_BYTES, &p.tm_bhi, bar_full(s), kbg * 32, n0);
                    if (p.passes == 3) tma_load_2d(st + Cfg::A_STAGE_BYTES + Cfg::B_BYTES, &p.tm_blo, bar_full(s), kbg * 32, n0);
                }
            }
        }
        return;
    }

    // ==================================================================== MMA + epilogue warpgroups
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                  // rows [64 cw, 64 cw + 64) of the tile
    const int t = threadIdx.x & 127;        // thread within the warpgroup
    const int ct = threadIdx.x - 128;       // thread within the two MMA warpgroups
    float acc[NMAIN][R];
    float accx[R];
    uint32_t it = 0, tcount = 0;
    for (int item = blockIdx.x; item < num_tiles; item += gridDim.x, ++tcount) {
        int w0, h0, n0img, n0;
        tile_of(item, w0, h0, n0img, n0);
#pragma unroll
        for (int i = 0; i < R; ++i) {
            accx[i] = 0.f;
#pragma unroll
            for (int a = 0; a < NMAIN; ++a) acc[a][i] = 0.f;
        }
        int prev_s = -1;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
            const int s = it % STAGES;
            mbar_wait(bar_full(s), (it / STAGES) & 1u);
            const uint32_t st = smem_base + s * Cfg::STAGE_BYTES;
            uint8_t* st_gen = smem_gen + s * Cfg::STAGE_BYTES;
            if constexpr (KIND == KIND_F16X3) {
                if (!p.a_planes) {
                    // A_h = fp16(A), A_l = fp16(A - A_h): thread -> (row, two 8-channel groups); two 16-byte pieces of the 128B-swizzled
                    // fp32 row in, one 16-byte piece of each 64B-swizzled fp16 row out, per group
                    const int r = 64 * cw + (t & 63);
                    uint8_t* ah = st_gen + Cfg::A_BYTES;
                    uint8_t* al = ah + Cfg::A_BYTES / 2;
                    bool bad = false;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int c8 = (t >> 6) * 2 + i;
                        const float4 v0 = *reinterpret_cast<const float4*>(st_gen + r * 128 + (((2 * c8) ^ (r & 7)) << 4));
                        const float4 v1 = *reinterpret_cast<const float4*>(st_gen + r * 128 + (((2 * c8 + 1) ^ (r & 7)) << 4));
                        const float f[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
                        __half2 hh[4], ll[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const __half x0 = __float2half_rn(f[2 * j]), x1 = __float2half_rn(f[2 * j + 1]);
                            bad = bad || !(fabsf(f[2 * j]) < 65504.f) || !(fabsf(f[2 * j + 1]) < 65504.f);
                            hh[j] = __halves2half2(x0, x1);
                            ll[j] = __halves2half2(__float2half_rn(f[2 * j] - __half2float(x0)), __float2half_rn(f[2 * j + 1] - __half2float(x1)));
                        }
                        const int off = r * 64 + ((c8 ^ ((r >> 1) & 3)) << 4);
                        *reinterpret_cast<uint4*>(ah + off) = *reinterpret_cast<const uint4*>(hh);
                        if (p.passes == 3) *reinterpret_cast<uint4*>(al + off) = *reinterpret_cast<const uint4*>(ll);
                    }
                    // rows past the TMA box (boxes smaller than 128 pixels) hold stale data: their accumulator rows are never stored, and
                    // they must not trip the range flag
                    if (bad && r * 128 < p.a_tile_bytes && p.range_flag) *p.range_flag = 1;
                    fence_proxy_async_smem();      // generic-proxy writes -> visible to the tensor core (async proxy)
                    named_bar_sync(2 + cw, 128);
                }
            } else {
                if (p.passes == 3) {
                    // A_lo = A - trunc_tf32(A), element-wise, so the swizzled placement is preserved verbatim
                    const float4* a = reinterpret_cast<const float4*>(st_gen) + 512 * cw;
                    float4* alo = reinterpret_cast<float4*>(st_gen + Cfg::A_BYTES) + 512 * cw;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float4 v = a[t + i * 128];
                        float4 o;
                        o.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u);
                        o.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
                        o.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u);
                        o.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
                        alo[t + i * 128] = o;
                    }
                    fence_proxy_async_smem();
                    named_bar_sync(2 + cw, 128);
                }
            }
            uint64_t da, dal, dbh, dbl;      // "hi" A, "lo" A, "hi" B, "lo" B
            if constexpr (KIND == KIND_F16X3) {
                da = gmma_desc_sw64(st + Cfg::A_BYTES + cw * 64 * 64);
                dal = gmma_desc_sw64(st + Cfg::A_BYTES + Cfg::A_BYTES / 2 + cw * 64 * 64);
                dbh = gmma_desc_sw64(st + Cfg::A_STAGE_BYTES);
                dbl = gmma_desc_sw64(st + Cfg::A_STAGE_BYTES + Cfg::B_BYTES);
            } else {
                da = gmma_desc_sw128(st + cw * 64 * 128);
                dal = gmma_desc_sw128(st + Cfg::A_BYTES + cw * 64 * 128);
                dbh = gmma_desc_sw128(st + Cfg::A_STAGE_BYTES);
                dbl = gmma_desc_sw128(st + Cfg::A_STAGE_BYTES + Cfg::B_BYTES);
            }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < Cfg::KSTEPS; ++k) {
                const uint64_t koff = (uint64_t)(k * 32 >> 4);
                if (p.passes == 3) {
                    conv_mma<BLOCK_N, KIND>(accx, dal + koff, dbh + koff);
                    conv_mma<BLOCK_N, KIND>(accx, da + koff, dbl + koff);
                }
                // The tensor core accumulates in fp32 with truncation, so every accumulate step costs up to 1 ulp of the running sum.
                // NMAIN == 3 rotates the main term over three accumulators by k-block (summed with RN adds in the epilogue): shorter chains.
                if constexpr (NMAIN == 1) {
                    conv_mma<BLOCK_N, KIND>(acc[0], da + koff, dbh + koff);
                } else {
                    const int sel = kb % 3;
                    if (sel == 0) conv_mma<BLOCK_N, KIND>(acc[0], da + koff, dbh + koff);
                    else if (sel == 1) conv_mma<BLOCK_N, KIND>(acc[NMAIN > 1 ? 1 : 0], da + koff, dbh + koff);
                    else conv_mma<BLOCK_N, KIND>(acc[NMAIN > 2 ? 2 : 0], da + koff, dbh + koff);
                }
            }
            wgmma_commit();
            // the MMAs of the previous k-block have retired: its stage goes back to the producer
            wgmma_wait<1>();
            if (prev_s >= 0 && lane == 0) mbar_arrive(bar_empty(prev_s));
            prev_s = s;
        }
        wgmma_wait<0>();
        if (prev_s >= 0 && lane == 0) mbar_arrive(bar_empty(prev_s));
        reg_fence(accx);
#pragma unroll
        for (int a = 0; a < NMAIN; ++a) reg_fence(acc[a]);

        // ---------------------------------------------------------------- epilogue
        int nlive = (p.cout - n0 + 31) / 32;       // chunks past the true Cout are neither computed nor stored
        nlive = nlive > Cfg::NCHUNK ? Cfg::NCHUNK : nlive;
        if (ct == 0) {
            tma_store_wait_read0();                // the previous tile's stores have read the staging area
            if (p.res_mode == RES_TILE) {
                mbar_arrive_expect_tx(bar_res, (uint32_t)(nlive * p.a_tile_bytes));
                for (int c = 0; c < nlive; ++c) tma_load_4d(epi_base + c * Cfg::A_BYTES, &p.tm_r, bar_res, n0 + c * 32, w0, h0, n0img);
            }
        }
        named_bar_sync(1, 256);
        if (p.res_mode == RES_TILE) mbar_wait(bar_res, tcount & 1u);
        // accumulator fragment of m64nN: thread (warp w, lane l) holds rows 16 (w % 4) + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1)
        const int rbase = 64 * cw + 16 * (warp & 3) + (lane >> 2);
        const int cq = 2 * (lane & 3);
        bool bad = false;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int row = rbase + 8 * hr;
            const float* up_row = nullptr;
            if (p.res_mode == RES_UPSAMPLE2X) {
                int r = row;
                const int pw_ = r % p.wbox; r /= p.wbox;
                const int ph_ = r % p.hbox; r /= p.hbox;
                const int pn_ = r;
                if (pn_ < p.nbox && w0 + pw_ < p.wo && h0 + ph_ < p.ho && n0img + pn_ < p.nimg) {
                    const int uy = min((h0 + ph_) >> 1, p.up_h - 1), ux = min((w0 + pw_) >> 1, p.up_w - 1);
                    up_row = p.up_src + (((size_t)(n0img + pn_) * p.up_h + uy) * p.up_w + ux) * (size_t)p.cout;
                }
            }
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
                const int col = 8 * j + cq;
                const int ch = n0 + col;
                const int c = j >> 2;               // 32-channel chunk
                if (c >= nlive) continue;
                const int i0 = 4 * j + 2 * hr;
                float v0 = accx[i0], v1 = accx[i0 + 1];
                if (p.passes != 3) { v0 = 0.f; v1 = 0.f; }
#pragma unroll
                for (int a = 0; a < NMAIN; ++a) { v0 += acc[a][i0]; v1 += acc[a][i0 + 1]; }
                float2 sc = make_float2(1.f, 1.f), sh = make_float2(0.f, 0.f);
                if (ch < p.cout) {                  // cout % 4 == 0 and ch is even: ch + 1 < cout too
                    sc = __ldg(reinterpret_cast<const float2*>(p.scale + ch));
                    sh = __ldg(reinterpret_cast<const float2*>(p.shift + ch));
                }
                float o0 = fmaf(v0, sc.x, sh.x), o1 = fmaf(v1, sc.y, sh.y);
                uint8_t* slot = epi_gen + c * Cfg::A_BYTES;
                // SWIZZLE_128B fp32 chunk: 16-byte piece (col % 32) / 4 of the row, XOR (row mod 8)
                const int off32 = row * 128 + (((((col & 31) >> 2)) ^ (row & 7)) << 4) + ((col & 3) << 2);
                if (p.res_mode == RES_TILE) {
                    const float2 r2 = *reinterpret_cast<const float2*>(slot + off32);
                    o0 += r2.x; o1 += r2.y;
                } else if (p.res_mode == RES_UPSAMPLE2X) {
                    if (up_row != nullptr && ch < p.cout) {
                        const float2 u = __ldg(reinterpret_cast<const float2*>(up_row + ch));
                        o0 += u.x; o1 += u.y;
                    }
                }
                if (p.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                // torch.sigmoid on CPU evaluates 1/(1+exp(-x)); expf/div are IEEE-rounded here
                if (ch < p.sigmoid_ch) o0 = 1.f / (1.f + expf(-o0));
                if (ch + 1 < p.sigmoid_ch) o1 = 1.f / (1.f + expf(-o1));
                if (KIND == KIND_F16X3 && p.out_planes) {
                    // two 64-byte-row fp16 tiles in the chunk (hi | lo), SWIZZLE_64B: 16-byte piece (col % 32) / 8 XOR ((row / 2) mod 4)
                    const __half2 h = __floats2half2_rn(o0, o1);
                    const float2 hf = __half22float2(h);
                    const __half2 l = __floats2half2_rn(o0 - hf.x, o1 - hf.y);
                    bad = bad || ((!(fabsf(o0) < 65504.f) || !(fabsf(o1) < 65504.f)) && row * 128 < p.a_tile_bytes);
                    const int off16 = row * 64 + ((((col & 31) >> 3) ^ ((row >> 1) & 3)) << 4) + ((col & 7) << 1);
                    *reinterpret_cast<__half2*>(slot + off16) = h;
                    *reinterpret_cast<__half2*>(slot + Cfg::A_BYTES / 2 + off16) = l;
                } else {
                    *reinterpret_cast<float2*>(slot + off32) = make_float2(o0, o1);
                }
            }
        }
        // (out_planes layers have Cout % 32 == 0: every channel of a live chunk is live)
        if (bad && p.range_flag) *p.range_flag = 1;
        fence_proxy_async_smem();
        named_bar_sync(1, 256);
        if (ct == 0) {
            for (int c = 0; c < nlive; ++c) {
                const uint32_t slot = epi_base + c * Cfg::A_BYTES;
                tma_store_4d(&p.tm_d, slot, n0 + c * 32, w0, h0, n0img);
                if (KIND == KIND_F16X3 && p.out_planes) tma_store_4d(&p.tm_d2, slot + Cfg::A_BYTES / 2, n0 + c * 32, w0, h0, n0img);
            }
            tma_store_commit();
        }
    }
    if (ct == 0) tma_store_wait0();      // all output bytes written before the CTA may exit
}

}  // namespace dt

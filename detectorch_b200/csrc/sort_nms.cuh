// detectorch_b200 -- CTA-level building blocks shared by the proposal / detection kernels:
//   * block_radix_sort_desc : stable LSD radix sort of (float key, int value) pairs by DESCENDING key
//     (ties keep ascending input order), one CTA, any n, global ping-pong buffers.
//   * block_rank / block_rank_count : ordered block-wide compaction ranks.
//   * block_nms_sorted      : greedy hard-NMS over boxes already in descending-score order.
//   * nms_mask_kernel + block_nms_walk : the same NMS for large sets (the RPN levels, dt_nms beyond one CTA): the IoU
//     bit-matrix on every SM, then one CTA walks the survivors over it.
//     Reference semantics (lib/utils_cython/cython_nms.pyx:37-87): "+1" widths, fp32 arithmetic in the
//     order  inter / ((area_i + area_j) - inter),  suppression when ovr >= thresh.  All fp32 ops use
//     the _rn intrinsics so nvcc cannot contract them into FMAs: kept ids are bit-exact vs the oracle.
//
// The NMS works in 64-box chunks (one bitmask word per chunk): (a) a warp-ballot 64x64 IoU bit-matrix
// for the chunk, (b) a serial resolve of the chunk against the running `removed` mask, (c) every
// thread tests one later box against the chunk's survivors only (suppressed boxes never suppress).
#pragma once
#include "common.cuh"

namespace dt {

__device__ __forceinline__ uint32_t float_desc_key(float f) {
    // monotone map float -> uint32 ascending, then inverted so that ascending radix order == descending float
    uint32_t b = __float_as_uint(f);
    b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ~b;
}

// Requires blockDim.x == 1024.  keys/vals: n entries in (k0,v0); scratch (k1,v1).  Result ends in (k0,v0)
// (4 passes = even number of ping-pongs).  smem_hist: 32*256 uint32 (32 KB).
static __device__ void block_radix_sort_asc_u32(uint32_t* k0, int* v0, uint32_t* k1, int* v1, int n, uint32_t* smem_hist) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t lt_mask = (1u << lane) - 1u;
    int chunk = (n + 31) / 32;
    chunk = (chunk + 31) & ~31;      // per-warp contiguous range, multiple of 32
    const int beg = warp * chunk;
    const int end = min(beg + chunk, n);
    __shared__ uint32_t warp_sums[32];
    uint32_t* kin = k0; int* vin = v0; uint32_t* kout = k1; int* vout = v1;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = pass * 8;
        for (int i = threadIdx.x; i < 32 * 256; i += blockDim.x) smem_hist[i] = 0;
        __syncthreads();
        // ---- sweep 1: per-warp digit histograms
        for (int i = beg + lane; i - lane < end; i += 32) {
            const bool valid = i < end;
            const unsigned act = __ballot_sync(0xffffffffu, valid);
            if (valid) {
                const uint32_t d = (kin[i] >> shift) & 255u;
                const unsigned m = __match_any_sync(act, d);
                if ((m & lt_mask) == 0) smem_hist[warp * 256 + d] += __popc(m);
            }
            __syncwarp();
        }
        __syncthreads();
        // ---- exclusive scan in (digit-major, warp-minor) order; thread t owns 8 consecutive entries
        {
            const int d = threadIdx.x >> 2, w0 = (threadIdx.x & 3) * 8;
            uint32_t loc[8], sum = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { loc[j] = smem_hist[(w0 + j) * 256 + d]; sum += loc[j]; }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
            if (lane == 31) warp_sums[warp] = incl;
            __syncthreads();
            if (warp == 0) {
                uint32_t ws = warp_sums[lane], wi = ws;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += y; }
                warp_sums[lane] = wi - ws;
            }
            __syncthreads();
            uint32_t run = warp_sums[warp] + incl - sum;
#pragma unroll
            for (int j = 0; j < 8; ++j) { smem_hist[(w0 + j) * 256 + d] = run; run += loc[j]; }
        }
        __syncthreads();
        // ---- sweep 2: stable scatter
        for (int i = beg + lane; i - lane < end; i += 32) {
            const bool valid = i < end;
            const unsigned act = __ballot_sync(0xffffffffu, valid);
            uint32_t key = 0, d = 0; int val = 0; unsigned m = 0; uint32_t base = 0;
            if (valid) {
                key = kin[i]; val = vin[i];
                d = (key >> shift) & 255u;
                m = __match_any_sync(act, d);
                base = smem_hist[warp * 256 + d];
            }
            __syncwarp();
            if (valid) {
                const uint32_t pos = base + __popc(m & lt_mask);
                kout[pos] = key; vout[pos] = val;
                if ((m & lt_mask) == 0) smem_hist[warp * 256 + d] = base + __popc(m);
            }
            __syncwarp();
        }
        __syncthreads();
        uint32_t* tk = kin; kin = kout; kout = tk;
        int* tv = vin; vin = vout; vout = tv;
    }
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

// ---------------------------------------------------------------------------------- NMS
__device__ __forceinline__ float box_area_p1(float4 b) {
    // (x2 - x1 + 1) * (y2 - y1 + 1)   cython_nms.pyx:44
    return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
}
__device__ __forceinline__ bool iou_suppresses(float4 a, float area_a, float4 b, float area_b, float thresh) {
    const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
    const float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
    const float w = fmaxf(0.f, __fadd_rn(__fsub_rn(xx2, xx1), 1.f));
    const float h = fmaxf(0.f, __fadd_rn(__fsub_rn(yy2, yy1), 1.f));
    const float inter = __fmul_rn(w, h);
    const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
    return ovr >= thresh;
}

struct NmsSmem {
    float4 cbox[64];
    float carea[64];
    unsigned long long diag[64];
    float4 kbox[64];
    float karea[64];
    int kcount;
    int total_kept;
};

// boxes: n boxes in descending-score order (global or shared).  removed: ceil(n/64) words (shared or global),
// overwritten.  On return bit j of removed is 1 iff box j is suppressed (bits >= n are 1).
// Returns (to all threads) the number kept.  blockDim.x must be a multiple of 64 and >= 64.
static __device__ int block_nms_sorted(const float4* boxes, int n, float thresh, unsigned long long* removed, NmsSmem* sm) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int nchunks = (n + 63) >> 6;
    for (int i = threadIdx.x; i < nchunks; i += blockDim.x) removed[i] = 0ull;
    if (threadIdx.x == 0) sm->total_kept = 0;
    __syncthreads();
    for (int c = 0; c < nchunks; ++c) {
        const int cbeg = c << 6;
        const int cn = min(64, n - cbeg);
        if (threadIdx.x < 64) {
            float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
            if (threadIdx.x < cn) b = boxes[cbeg + threadIdx.x];
            sm->cbox[threadIdx.x] = b;
            sm->carea[threadIdx.x] = box_area_p1(b);
        }
        __syncthreads();
        // (a) chunk-local bit-matrix: diag[i] bit j (j > i) set if box i suppresses box j
        for (int i = warp; i < 64; i += nwarps) {
            const float4 bi = sm->cbox[i];
            const float ai = sm->carea[i];
            const bool s0 = (lane > i) && (lane < cn) && (i < cn) && iou_suppresses(bi, ai, sm->cbox[lane], sm->carea[lane], thresh);
            const bool s1 = (lane + 32 > i) && (lane + 32 < cn) && (i < cn) &&
                            iou_suppresses(bi, ai, sm->cbox[lane + 32], sm->carea[lane + 32], thresh);
            const unsigned lo = __ballot_sync(0xffffffffu, s0), hi = __ballot_sync(0xffffffffu, s1);
            if (lane == 0) sm->diag[i] = (unsigned long long)lo | ((unsigned long long)hi << 32);
        }
        __syncthreads();
        // (b) serial resolve of this chunk: one thread walks the survivors (the only truly sequential part of greedy NMS: a 64-bit mask and
        // one dependent shared-memory read per kept box); the survivors' boxes are then compacted by 64 threads in parallel
        if (threadIdx.x == 0) {
            const unsigned long long valid = (cn == 64) ? ~0ull : ((1ull << cn) - 1ull);
            unsigned long long alive = ~removed[c] & valid, kept = 0ull;
            int kc = 0, tot = sm->total_kept;
            while (alive) {
                const int b = __ffsll((long long)alive) - 1;
                kept |= 1ull << b;
                ++kc; ++tot;
                alive &= ~sm->diag[b];
                alive &= ~(1ull << b);
            }
            removed[c] = ~kept;
            sm->kcount = kc;
            sm->total_kept = tot;
        }
        __syncthreads();
        if (threadIdx.x < 64) {
            const unsigned long long kept = ~removed[c];
            if ((kept >> threadIdx.x) & 1ull) {
                const int pos = __popcll(kept & ((1ull << threadIdx.x) - 1ull));       // ascending order, as the serial walk produced it
                sm->kbox[pos] = sm->cbox[threadIdx.x];
                sm->karea[pos] = sm->carea[threadIdx.x];
            }
        }
        __syncthreads();
        const int kc = sm->kcount;
        // (c) later boxes vs this chunk's survivors
        if (kc > 0) {
            for (int j = cbeg + 64 + threadIdx.x; j < n; j += blockDim.x) {
                if ((removed[j >> 6] >> (j & 63)) & 1ull) continue;
                const float4 bj = boxes[j];
                const float aj = box_area_p1(bj);
                bool sup = false;
                for (int k = 0; k < kc && !sup; ++k) sup = iou_suppresses(sm->kbox[k], sm->karea[k], bj, aj, thresh);
                if (sup) atomicOr(&removed[j >> 6], 1ull << (j & 63));
            }
        }
        __syncthreads();
    }
    return sm->total_kept;
}

// ---- large sets: the suppression bit-matrix at full-GPU width (nms_mask_kernel), then one CTA walks it (block_nms_walk)
// grid (nchunks, nchunks, sets), 64 threads.  Set s: counts[s] boxes in descending-score order at boxes + s * set_stride, its matrix at
// mask + s * set_stride * nchunks (row i = nchunks words).  Block (bj, bi) with bj >= bi fills word (i, bj) for the 64 boxes i of
// chunk bi: bit b set <=> box i suppresses box bj*64 + b (only later boxes: index > i)
static __global__ void __launch_bounds__(64) nms_mask_kernel(const float4* __restrict__ boxes, const int* __restrict__ counts, long long set_stride,
                                                             int nchunks, float thresh, unsigned long long* __restrict__ mask) {
    const int bj = blockIdx.x, bi = blockIdx.y, s = blockIdx.z;
    if (bj < bi) return;
    const int n = counts[s];
    if (bi * 64 >= n || bj * 64 >= n) return;
    __shared__ float4 jb[64];
    __shared__ float ja[64];
    boxes += s * set_stride;
    mask += s * set_stride * nchunks;
    const int j0 = bj * 64, i = bi * 64 + threadIdx.x;
    const int jn = min(64, n - j0);
    if ((int)threadIdx.x < jn) { const float4 b = boxes[j0 + threadIdx.x]; jb[threadIdx.x] = b; ja[threadIdx.x] = box_area_p1(b); }
    __syncthreads();
    if (i >= n) return;
    const float4 me = boxes[i];
    const float ma = box_area_p1(me);
    unsigned long long bits = 0ull;
    for (int b = 0; b < jn; ++b)
        if (j0 + b > i && iou_suppresses(me, ma, jb[b], ja[b], thresh)) bits |= 1ull << b;
    mask[(size_t)i * nchunks + bj] = bits;
}

struct NmsWalkSmem {
    unsigned long long diag[64];
    int kept_list[64];
    int kcount;
    int total_kept;
};

// Greedy NMS of one set of n boxes over its nms_mask_kernel matrix (rows of `nchunks` words).  Chunk by chunk, one thread resolves the
// chunk against the running `removed` mask (the only truly sequential part), then the chunk's survivors OR their rows into `removed`.
// removed (shared): ceil(n / 64) words, overwritten; on return bit i is 0 iff box i is kept.  max_keep > 0: keep at most that many (every
// later box is then marked removed).  All threads of the block must call.
static __device__ __forceinline__ void block_nms_walk(const unsigned long long* mask, int n, int nchunks, int max_keep, unsigned long long* removed, NmsWalkSmem* sm) {
    const int nc = (n + 63) >> 6;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) removed[i] = 0ull;
    if (threadIdx.x == 0) sm->total_kept = 0;
    __syncthreads();
    for (int c = 0; c < nc; ++c) {
        const int cn = min(64, n - c * 64);
        if ((int)threadIdx.x < cn) sm->diag[threadIdx.x] = mask[(size_t)(c * 64 + threadIdx.x) * nchunks + c];
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned long long valid = (cn == 64) ? ~0ull : ((1ull << cn) - 1ull);
            unsigned long long alive = ~removed[c] & valid, kept = 0ull;
            int kc = 0, tot = sm->total_kept;
            while (alive) {
                const int t = __ffsll((long long)alive) - 1;
                if (max_keep > 0 && tot >= max_keep) break;
                kept |= 1ull << t;
                sm->kept_list[kc++] = c * 64 + t;
                ++tot;
                alive &= ~sm->diag[t];
                alive &= ~(1ull << t);
            }
            removed[c] = ~kept;
            sm->kcount = kc;
            sm->total_kept = tot;
        }
        __syncthreads();
        if (max_keep > 0 && sm->total_kept >= max_keep) {
            for (int i = c + 1 + threadIdx.x; i < nc; i += blockDim.x) removed[i] = ~0ull;
            __syncthreads();
            break;
        }
        // the survivors of this chunk suppress later boxes: OR their matrix rows into `removed`.  Thread t takes word c + 1 + t % words
        // (and every blockDim-th after it) and, when fewer words than threads remain, every groups-th survivor from t / words: the block
        // stays busy both on the few words of an RPN level and on the thousands of a large dt_nms set.
        const int kc = sm->kcount, words = nc - c - 1;
        if (words > 0) {
            const int groups = max(1, (int)blockDim.x / words), g = (int)threadIdx.x / words;
            if (g < groups)
                for (int wd = c + 1 + (int)threadIdx.x % words; wd < nc; wd += blockDim.x) {
                    unsigned long long acc = 0ull;
#pragma unroll 4
                    for (int k = g; k < kc; k += groups) acc |= mask[(size_t)sm->kept_list[k] * nchunks + wd];
                    if (groups == 1) removed[wd] |= acc;          // the word's only writer
                    else if (acc) atomicOr(&removed[wd], acc);
                }
        }
        __syncthreads();
    }
}

}  // namespace dt

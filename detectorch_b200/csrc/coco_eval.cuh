// detectorch_b200 -- COCO box and mask evaluation on the device: pycocotools' COCOeval (iouType 'bbox' / 'segm', default thresholds)
// restated kernel by kernel so that precision, recall and scores come out bit for bit as COCOeval.evaluate() + accumulate() give them.
//
//   coco_gt_kernel        one CTA per annotation: polygon -> RLE (maskApi rleFrPoly: x5 upsampling, edge walk, y-boundary points,
//                         sort, run lengths) and union of the parts (rleMerge); uncompressed RLE copied; compressed RLE decoded;
//                         rleToBbox of the result.  Runs once per ground-truth set.
//   coco_det_rle_kernel   one thread per detection: rleFrString of its compressed string, maskUtils.area, rleToBbox.
//   coco_pair_kernel      one CTA per (category, image) pair with detections: stable score sort cut to 100 (computeIoU), the IoU
//                         matrix (bbIou / rleIou, double), then one thread per (area range, IoU threshold) runs evaluateImg's greedy
//                         matching and writes a 2-bit state (matched, ignored) per detection.
//   coco_rank_*           accumulate()'s stable sort by -score of each category's kept detections, concatenated in image order:
//                         a stable segmented sort (CUB) of descending score keys per category, then one scan of the maxDets cut
//                         flags places each detection in the list of every cut it survives.
//   coco_accum_kernel     one thread per (category, area, maxDets, threshold): cumulative tp / fp, recall, the right-to-left
//                         precision envelope and searchsorted(rc, recThrs, 'left'), in float64 as numpy computes them.
//
// Every product that feeds a sum is an explicit __dmul_rn / __dadd_rn: the C code it restates is compiled without contraction.
// Pairs are ordered category-major, image-minor (COCOeval's evalImgs order), so a category's kept detections are one contiguous
// range in image order, which is the concatenation accumulate() sorts.
#pragma once
#include <cstdint>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cuda_runtime.h>

namespace dt {

constexpr int kCocoAreas = 4, kCocoThrs = 10, kCocoRecThrs = 101, kCocoMaxDets = 3, kCocoKeep = 100;
constexpr int kCocoStates = kCocoAreas * kCocoThrs;   // per kept detection: one state byte per (area range, threshold)
// params block (double): area ranges [4][2], IoU thresholds already clipped to 1 - 1e-10 [10], recall thresholds [101]
constexpr int kCocoParAreas = 0, kCocoParThrs = 8, kCocoParRec = 18, kCocoParams = 119;
// annotation table (int64 per annotation): kind, h, w, first part, number of parts, output offset
constexpr int kCocoAnnCols = 6;
enum { kCocoPoly = 0, kCocoCounts = 1, kCocoString = 2 };
// part table (int64 per part): first element (xy pair / count / char), number of elements, int32 workspace offset, upsampled points
// of a polygon (maskApi's m after the edge walk; the host counts it from the same rounding).  A polygon part of k points and m
// upsampled points takes k + 4 m + 3 ints of workspace.
constexpr int kCocoPartCols = 4;
// ground truth in pair order: f64 [box x y w h, area, rle box x y w h]; i64 [rle offset, rle length, h, w, iscrowd, id != 0]
constexpr int kCocoGtF = 9, kCocoGtI = 6;
// detections in pair order: f64 [score, box x y w h]; i64 [char offset, char count, h, w]
constexpr int kCocoDetF = 5, kCocoDetI = 4;
// active pair table (int64): pair index (category * images + image), first detection, D, first gt, G, first kept slot, first IoU
constexpr int kCocoPairCols = 7;

// x86 cvttsd2si: truncation, and INT_MIN for NaN or out of range (what the host build of maskApi.c does with (int) of a double)
__host__ __device__ __forceinline__ int coco_trunc(double v) {
    return (v >= -2147483648.0 && v < 2147483648.0) ? (int)v : (int)0x80000000;
}

__device__ __forceinline__ uint32_t coco_umin(uint32_t a, uint32_t b) { return a < b ? a : b; }
__device__ __forceinline__ uint32_t coco_umax(uint32_t a, uint32_t b) { return a > b ? a : b; }

// maskApi rleToBbox of one RLE (uint arithmetic as in C)
__device__ void coco_rle_box(const uint32_t* cnts, int64_t m, uint32_t h, uint32_t w, double* bb) {
    m = (m / 2) * 2;
    if (m == 0) { bb[0] = bb[1] = bb[2] = bb[3] = 0; return; }
    uint32_t xs = w, ys = h, xe = 0, ye = 0, cc = 0;
    for (int64_t j = 0; j < m; j++) {
        cc += cnts[j];
        const uint32_t t = cc - (uint32_t)(j % 2), y = t % h, x = (t - y) / h;
        xs = coco_umin(xs, x); xe = coco_umax(xe, x); ys = coco_umin(ys, y); ye = coco_umax(ye, y);
    }
    bb[0] = xs; bb[2] = (double)(uint32_t)(xe - xs + 1);
    bb[1] = ys; bb[3] = (double)(uint32_t)(ye - ys + 1);
}

// maskApi bbIou of one (detection, gt) pair, xywh
__device__ __forceinline__ double coco_bb_iou(const double* D, const double* G, bool crowd) {
    const double ga = __dmul_rn(G[2], G[3]), da = __dmul_rn(D[2], D[3]);
    const double w = __dsub_rn(fmin(__dadd_rn(D[2], D[0]), __dadd_rn(G[2], G[0])), fmax(D[0], G[0]));
    if (w <= 0) return 0;
    const double h = __dsub_rn(fmin(__dadd_rn(D[3], D[1]), __dadd_rn(G[3], G[1])), fmax(D[1], G[1]));
    if (h <= 0) return 0;
    const double i = __dmul_rn(w, h), u = crowd ? da : __dsub_rn(__dadd_rn(da, ga), i);
    return __ddiv_rn(i, u);
}

// maskApi rleIou of one pair: box IoU first, the run merge only where the boxes overlap
__device__ double coco_rle_iou(const uint32_t* dc, int64_t dm, const double* dbox, int64_t dh, int64_t dw, const uint32_t* gc, int64_t gm,
                               const double* gbox, int64_t gh, int64_t gw, bool crowd) {
    const double o = coco_bb_iou(dbox, gbox, crowd);
    if (!(o > 0)) return o;
    if (dh != gh || dw != gw) return -1;
    uint32_t ca = dc[0], cb = gc[0], c, ct = 1, i = 0, u = 0;
    int64_t a = 1, b = 1;
    bool va = false, vb = false;
    while (ct > 0) {
        c = coco_umin(ca, cb);
        if (va || vb) { u += c; if (va && vb) i += c; }
        ct = 0;
        ca -= c; if (!ca && a < dm) { ca = dc[a++]; va = !va; } ct += ca;
        cb -= c; if (!cb && b < gm) { cb = gc[b++]; vb = !vb; } ct += cb;
    }
    if (i == 0) u = 1;
    else if (crowd) { u = 0; for (int64_t j = 1; j < dm; j += 2) u += dc[j]; }
    return __ddiv_rn((double)i, (double)u);
}

// maskApi rleFrString of one string: returns the number of counts written to cnts
__device__ int64_t coco_rle_from_string(const char* s, int64_t len, uint32_t* cnts) {
    int64_t m = 0, p = 0;
    while (p < len) {
        long long x = 0;
        int k = 0, more = 1;
        while (more) {
            const int c = s[p] - 48;
            x |= (long long)(int)((c & 0x1f) << (5 * k));
            more = c & 0x20; p++; k++;
            if (!more && (c & 0x10)) x |= (long long)(int)(0xffffffffu << (5 * k));
        }
        if (m > 2) x += (long long)cnts[m - 2];
        cnts[m++] = (uint32_t)x;
    }
    return m;
}

// maskApi rleMerge step (union) of A and B into out: returns the number of counts
__device__ int64_t coco_rle_union(const uint32_t* A, int64_t am, const uint32_t* B, int64_t bm, uint32_t* out) {
    uint32_t ca = A[0], cb = B[0], c, cc = 0, ct = 1;
    int v = 0, va = 0, vb = 0, vp;
    int64_t a = 1, b = 1, m = 0;
    while (ct > 0) {
        c = coco_umin(ca, cb); cc += c; ct = 0;
        ca -= c; if (!ca && a < am) { ca = A[a++]; va = !va; } ct += ca;
        cb -= c; if (!cb && b < bm) { cb = B[b++]; vb = !vb; } ct += cb;
        vp = v; v = va || vb;
        if (v != vp || ct == 0) { out[m++] = cc; cc = 0; }
    }
    return m;
}

__device__ __forceinline__ int coco_up(double v) { return coco_trunc(__dadd_rn(__dmul_rn(5.0, v), .5)); }

// rleFrPoly of one polygon of k points, cooperatively by the CTA.  ws: the part's int32 workspace (k + 4 m_up + 3 ints, m_up the
// number of upsampled boundary points); thread 0 gets the part's run lengths at *out (inside ws) and their number in *out_m.
__device__ void coco_poly_rle(const double* xy, int k, uint32_t h, uint32_t w, int* ws, int64_t m_up, uint32_t** out, int64_t* out_m) {
    __shared__ int s_n;
    int* eoff = ws;                          // k + 1 edge offsets into the upsampled points
    int* u = eoff + k + 1;
    int* v = u + m_up;
    uint32_t* a = reinterpret_cast<uint32_t*>(v + m_up);   // y-boundary points, then h * w      (m_up + 1)
    uint32_t* srt = a + m_up + 1;                           // sorted, then differenced and packed (m_up + 1)
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) {
        int o = 0;
        for (int j = 0; j < k; j++) {
            eoff[j] = o;
            const int j1 = j + 1 < k ? j + 1 : 0;
            const int dx = abs(coco_up(xy[2 * j1]) - coco_up(xy[2 * j])), dy = abs(coco_up(xy[2 * j1 + 1]) - coco_up(xy[2 * j + 1]));
            o += (int)coco_umax((uint32_t)dx, (uint32_t)dy) + 1;
        }
        eoff[k] = o;
        s_n = 0;
    }
    __syncthreads();
    const int m = eoff[k];
    for (int i = tid; i < m; i += nt) {
        int lo = 0, hi = k - 1;              // the edge j with eoff[j] <= i < eoff[j + 1]
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (eoff[mid] <= i) lo = mid; else hi = mid - 1; }
        const int j = lo, d = i - eoff[j], j1 = j + 1 < k ? j + 1 : 0;
        int xs = coco_up(xy[2 * j]), xe = coco_up(xy[2 * j1]), ys = coco_up(xy[2 * j + 1]), ye = coco_up(xy[2 * j1 + 1]);
        const int dx = abs(xe - xs), dy = abs(ys - ye);
        const bool flip = (dx >= dy && xs > xe) || (dx < dy && ys > ye);
        if (flip) { int t = xs; xs = xe; xe = t; t = ys; ys = ye; ye = t; }
        const double s = dx >= dy ? __ddiv_rn((double)(ye - ys), (double)dx) : __ddiv_rn((double)(xe - xs), (double)dy);
        if (dx >= dy) {
            const int t = flip ? dx - d : d;
            u[i] = t + xs; v[i] = coco_trunc(__dadd_rn(__dadd_rn((double)ys, __dmul_rn(s, (double)t)), .5));
        } else {
            const int t = flip ? dy - d : d;
            v[i] = t + ys; u[i] = coco_trunc(__dadd_rn(__dadd_rn((double)xs, __dmul_rn(s, (double)t)), .5));
        }
    }
    __syncthreads();
    // y-boundary points and downsampling; their order does not matter (they are sorted next)
    for (int j = 1 + tid; j < m; j += nt) {
        if (u[j] == u[j - 1]) continue;
        double xd = (double)(u[j] < u[j - 1] ? u[j] : u[j] - 1);
        xd = (xd + .5) / 5.0 - .5;
        if (floor(xd) != xd || xd < 0 || xd > (double)(w - 1)) continue;
        double yd = (double)(v[j] < v[j - 1] ? v[j] : v[j - 1]);
        yd = (yd + .5) / 5.0 - .5;
        if (yd < 0) yd = 0; else if (yd > (double)h) yd = h;
        yd = ceil(yd);
        a[atomicAdd(&s_n, 1)] = (uint32_t)((int)xd * (int)h + (int)yd);
    }
    __syncthreads();
    const int n = s_n + 1;
    if (tid == 0) a[n - 1] = h * w;
    __syncthreads();
    for (int i = tid; i < n; i += nt) {      // rank sort (equal values keep their index order: the sorted multiset is unique)
        const uint32_t x = a[i];
        int r = 0;
        for (int j = 0; j < n; j++) r += (a[j] < x) || (a[j] == x && j < i);
        srt[r] = x;
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t p = 0;
        for (int j = 0; j < n; j++) { const uint32_t t = srt[j]; srt[j] -= p; p = t; }
        int j = 0, mm = 0;
        srt[mm++] = srt[j++];
        while (j < n) {
            if (srt[j] > 0) srt[mm++] = srt[j++];
            else { j++; if (j < n) srt[mm - 1] += srt[j++]; }
        }
        *out = srt; *out_m = mm;
    }
    __syncthreads();
}

// one CTA per annotation.  out_cnts / tmp_cnts: same layout, capacity per annotation = the distance to the next one's offset
__global__ void coco_gt_kernel(const int64_t* __restrict__ ann, const int64_t* __restrict__ parts, const double* __restrict__ xy,
                               const uint32_t* __restrict__ ucounts, const char* __restrict__ chars, int* __restrict__ ws,
                               uint32_t* __restrict__ out_cnts, uint32_t* __restrict__ tmp_cnts, int64_t* __restrict__ out_len,
                               double* __restrict__ out_box) {
    const int64_t* A = ann + (int64_t)blockIdx.x * kCocoAnnCols;
    const int kind = (int)A[0], np_ = (int)A[4];
    const uint32_t h = (uint32_t)A[1], w = (uint32_t)A[2];
    const int64_t p0 = A[3], off = A[5];
    uint32_t* out = out_cnts + off;
    uint32_t* tmp = tmp_cnts + off;
    __shared__ int64_t s_m;
    if (kind == kCocoPoly) {
        for (int p = 0; p < np_; p++) {
            const int64_t* P = parts + (p0 + p) * kCocoPartCols;
            uint32_t* r; int64_t rm;
            coco_poly_rle(xy + 2 * P[0], (int)P[1], h, w, ws + P[2], P[3], &r, &rm);
            if (threadIdx.x == 0) {
                if (p == 0) { for (int64_t j = 0; j < rm; j++) out[j] = r[j]; s_m = rm; }
                else {
                    const int64_t mm = coco_rle_union(out, s_m, r, rm, tmp);
                    for (int64_t j = 0; j < mm; j++) out[j] = tmp[j];
                    s_m = mm;
                }
            }
            __syncthreads();
        }
    } else if (threadIdx.x == 0) {
        const int64_t* P = parts + p0 * kCocoPartCols;
        if (kind == kCocoCounts) {
            for (int64_t j = 0; j < P[1]; j++) out[j] = ucounts[P[0] + j];
            s_m = P[1];
        } else {
            s_m = coco_rle_from_string(chars + P[0], P[1], out);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        out_len[blockIdx.x] = s_m;
        coco_rle_box(out, s_m, h, w, out_box + 4 * (int64_t)blockIdx.x);
    }
}

// one thread per detection: decoded counts at the detection's char offset (a count takes at least one char)
__global__ void coco_det_rle_kernel(int64_t n, const int64_t* __restrict__ det_i, const char* __restrict__ chars, uint32_t* __restrict__ cnts,
                                    int64_t* __restrict__ det_m, double* __restrict__ det_area, double* __restrict__ det_box) {
    const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n) return;
    const int64_t* I = det_i + d * kCocoDetI;
    uint32_t* c = cnts + I[0];
    const int64_t m = coco_rle_from_string(chars + I[0], I[1], c);
    uint32_t area = 0;
    for (int64_t j = 1; j < m; j += 2) area += c[j];
    det_m[d] = m;
    det_area[d] = (double)area;
    coco_rle_box(c, m, (uint32_t)I[2], (uint32_t)I[3], det_box + 4 * d);
}

// one thread per detection string: bad[d] = 1 when rleFrString's uint32 counts of it do not sum to h * w.  rleIou walks two masks'
// runs until both end, so a mask whose runs cover another number of pixels than its partner's never ends (in maskApi as here); the
// host refuses such results before dt_coco_eval.  Same decode as coco_rle_from_string, keeping only the last two counts.
__global__ void coco_det_check_kernel(int64_t n, const int64_t* __restrict__ det_i, const char* __restrict__ chars, uint8_t* __restrict__ bad) {
    const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n) return;
    const int64_t* I = det_i + d * kCocoDetI;
    const char* s = chars + I[0];
    const int64_t len = I[1];
    int64_t m = 0, p = 0;
    uint32_t c2 = 0, c1 = 0;                 // counts m - 2 and m - 1
    uint64_t tot = 0;
    while (p < len) {
        long long x = 0;
        int k = 0, more = 1;
        while (more) {
            const int c = s[p] - 48;
            x |= (long long)(int)((c & 0x1f) << (5 * k));
            more = c & 0x20; p++; k++;
            if (!more && (c & 0x10)) x |= (long long)(int)(0xffffffffu << (5 * k));
        }
        if (m > 2) x += (long long)c2;
        const uint32_t cnt = (uint32_t)x;
        tot += cnt;
        c2 = c1; c1 = cnt; m++;
    }
    bad[d] = tot != (uint64_t)I[2] * (uint64_t)I[3];
}

inline cudaError_t coco_det_check_launch(int64_t n, const int64_t* det_i, const char* chars, uint8_t* bad, cudaStream_t st) {
    coco_det_check_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, det_i, chars, bad);
    return cudaGetLastError();
}

struct CocoEvalArgs {
    int segm, num_images;
    int use_area;             // det_area holds each detection's area (segm: the RLE area; else the caller's), not w h
    const int64_t* pairs;
    const double* det_f; const int64_t* det_i;
    const uint32_t* det_cnts; const int64_t* det_m; const double* det_area; const double* det_rbox;
    const double* gt_f; const int64_t* gt_i; const uint32_t* gt_cnts;
    const double* par;
    int* kept_det;            // [kept] detection index of each kept slot
    int* kept_rank;           // [kept] rank within its pair
    double* kept_score;       // [kept]
    uint8_t* state;           // [kept][40] bit 0 matched (to a gt of non-zero id), bit 1 ignored
    double* iou;              // [sum D' G]
    uint8_t* gtm;             // [gts][40]
};

__device__ __forceinline__ bool coco_out(double area, const double* rng) { return area < rng[0] || area > rng[1]; }

// one CTA per (category, image) pair that has detections
__global__ void coco_pair_kernel(CocoEvalArgs p) {
    const int64_t* T = p.pairs + (int64_t)blockIdx.x * kCocoPairCols;
    const int64_t d0 = T[1], D = T[2], g0 = T[3], G = T[4], k0 = T[5], i0 = T[6];
    const int64_t Dk = D < kCocoKeep ? D : kCocoKeep;
    const int tid = threadIdx.x, nt = blockDim.x;
    // computeIoU: np.argsort(-score, kind='mergesort'), cut to maxDets[-1]
    for (int64_t i = tid; i < D; i += nt) {
        const double s = p.det_f[(d0 + i) * kCocoDetF];
        int64_t r = 0;
        for (int64_t j = 0; j < D; j++) {
            const double sj = p.det_f[(d0 + j) * kCocoDetF];
            r += (sj > s) || (sj == s && j < i);
        }
        if (r < kCocoKeep) { p.kept_det[k0 + r] = (int)(d0 + i); p.kept_rank[k0 + r] = (int)r; p.kept_score[k0 + r] = s; }
    }
    __syncthreads();
    for (int64_t e = tid; e < Dk * G; e += nt) {
        const int64_t dr = e / G, g = e % G, d = p.kept_det[k0 + dr], gi = g0 + g;
        const bool crowd = p.gt_i[gi * kCocoGtI + 4] != 0;
        double o;
        if (p.segm) {
            const int64_t* DI = p.det_i + d * kCocoDetI;
            const int64_t* GI = p.gt_i + gi * kCocoGtI;
            o = coco_rle_iou(p.det_cnts + DI[0], p.det_m[d], p.det_rbox + 4 * d, DI[2], DI[3], p.gt_cnts + GI[0], GI[1], p.gt_f + gi * kCocoGtF + 5,
                             GI[2], GI[3], crowd);
        } else {
            o = coco_bb_iou(p.det_f + d * kCocoDetF + 1, p.gt_f + gi * kCocoGtF, crowd);
        }
        p.iou[i0 + dr * G + g] = o;
    }
    __syncthreads();
    // evaluateImg per (area range, threshold): gts ignore-last (stable), greedy matching in score order
    for (int c = tid; c < kCocoStates; c += nt) {
        const int ar = c / kCocoThrs, t = c % kCocoThrs;
        const double* rng = p.par + kCocoParAreas + 2 * ar;
        uint8_t* gm = p.gtm + g0 * kCocoStates + (int64_t)c * G;
        for (int64_t g = 0; g < G; g++) gm[g] = 0;
        for (int64_t dr = 0; dr < Dk; dr++) {
            double best = p.par[kCocoParThrs + t];
            int64_t m = -1;
            bool m_ig = false;
            for (int pass = 0; pass < 2; pass++) {
                for (int64_t g = 0; g < G; g++) {
                    const int64_t* GI = p.gt_i + (g0 + g) * kCocoGtI;
                    const bool ig = GI[4] != 0 || coco_out(p.gt_f[(g0 + g) * kCocoGtF + 4], rng);
                    if ((int)ig != pass) continue;
                    if (gm[g] && !GI[4]) continue;
                    if (m > -1 && !m_ig && ig) goto matched;
                    const double o = p.iou[i0 + dr * G + g];
                    if (o < best) continue;
                    best = o; m = g; m_ig = ig;
                }
            }
        matched:
            bool hit = false, dig = false;
            if (m > -1) {
                dig = m_ig;
                hit = p.gt_i[(g0 + m) * kCocoGtI + 5] != 0;
                gm[m] = 1;
            }
            const int64_t d = p.kept_det[k0 + dr];
            const double area = p.use_area ? p.det_area[d] : __dmul_rn(p.det_f[d * kCocoDetF + 3], p.det_f[d * kCocoDetF + 4]);
            if (!hit && coco_out(area, rng)) dig = true;
            p.state[(k0 + dr) * kCocoStates + c] = (uint8_t)((hit ? 1 : 0) | (dig ? 2 : 0));
        }
    }
}

// accumulate(): each kept detection's position in the stable -score sort of its category, per maxDets cut (order_off [3][K + 1]: start
// of category k's list for cut m; cat_kept [K + 1]: the category's kept slots).  The key sorts ascending as -score does (-0.0 and 0.0
// equal, as numpy compares them) and the slot index is the value, so a stable sort of each category's slots keeps the concatenation
// order among equal scores.
__global__ void coco_rank_keys_kernel(int64_t kept, const double* __restrict__ kept_score, uint64_t* __restrict__ keys, int* __restrict__ vals) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= kept) return;
    const double s = kept_score[e];
    const uint64_t u = s == 0.0 ? 0ull : (uint64_t)__double_as_longlong(s);
    const uint64_t asc = (u >> 63) ? ~u : (u | (1ull << 63));
    keys[e] = ~asc;
    vals[e] = (int)e;
}

// flags[m * kept + i] = 1 when the i-th slot of the sorted order is inside maxDets cut m.  Their exclusive scan over the three cuts in a
// row is each surviving slot's index in order[] (cut-major, then category, then sort order: order_off's layout).
__global__ void coco_rank_flags_kernel(int64_t kept, const int* __restrict__ sorted, const int* __restrict__ kept_rank, int* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kept) return;
    const int r = kept_rank[sorted[i]];
    flags[i] = r < 1; flags[kept + i] = r < 10; flags[2 * kept + i] = r < kCocoKeep;
}

__global__ void coco_rank_scatter_kernel(int64_t kept, const int* __restrict__ sorted, const int* __restrict__ flags,
                                         const int* __restrict__ pos, int* __restrict__ order) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kCocoMaxDets * kept) return;
    if (flags[i]) order[pos[i]] = sorted[i % kept];
}

// bytes of CUB temporary storage for the sort of `kept` slots in K categories and the scan of 3 kept flags
inline size_t coco_rank_temp_bytes(int64_t kept, int K) {
    size_t sort_b = 0, scan_b = 0;
    cub::DeviceSegmentedSort::StableSortPairs(nullptr, sort_b, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr, (int*)nullptr,
                                              (int)kept, K, (const int64_t*)nullptr, (const int64_t*)nullptr);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int*)nullptr, (int*)nullptr, (int64_t)kCocoMaxDets * kept);
    return sort_b > scan_b ? sort_b : scan_b;
}

// one thread per (category, area range, maxDets, threshold).  precision / scores [T, R, K, A, M], recall [T, K, A, M]
__global__ void coco_accum_kernel(int K, const int64_t* __restrict__ cat_gt, const double* __restrict__ gt_f, const int64_t* __restrict__ gt_i,
                                  const int64_t* __restrict__ order_off, const int* __restrict__ order, const double* __restrict__ kept_score,
                                  const uint8_t* __restrict__ state, const double* __restrict__ par, double* __restrict__ precision,
                                  double* __restrict__ recall, double* __restrict__ scores) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= K * kCocoAreas * kCocoMaxDets * kCocoThrs) return;
    const int t = idx % kCocoThrs, m = (idx / kCocoThrs) % kCocoMaxDets, a = (idx / (kCocoThrs * kCocoMaxDets)) % kCocoAreas;
    const int k = idx / (kCocoThrs * kCocoMaxDets * kCocoAreas);
    const int A = kCocoAreas, M = kCocoMaxDets, R = kCocoRecThrs;
    const double* rng = par + kCocoParAreas + 2 * a;
    const double* rec = par + kCocoParRec;
    const int64_t cell = ((int64_t)k * A + a) * M + m;
    double* prec = precision + (int64_t)t * R * K * A * M + cell;     // + r * K * A * M
    double* sco = scores + (int64_t)t * R * K * A * M + cell;
    const int64_t rstride = (int64_t)K * A * M;
    int64_t npig = 0;
    for (int64_t g = cat_gt[k]; g < cat_gt[k + 1]; g++) npig += !(gt_i[g * kCocoGtI + 4] != 0 || coco_out(gt_f[g * kCocoGtF + 4], rng));
    if (npig == 0) {
        for (int r = 0; r < R; r++) { prec[r * rstride] = -1; sco[r * rstride] = -1; }
        recall[(int64_t)t * K * A * M + cell] = -1;
        return;
    }
    const int* list = order + order_off[m * (K + 1) + k];
    const int64_t nd = order_off[m * (K + 1) + k + 1] - order_off[m * (K + 1) + k];
    const int sc = a * kCocoThrs + t;
    int64_t tp = 0, fp = 0;
    for (int64_t i = 0; i < nd; i++) {
        const uint8_t st = state[(int64_t)list[i] * kCocoStates + sc];
        if (!(st & 2)) { if (st & 1) tp++; else fp++; }
    }
    const double np_ = (double)npig, eps = 2.220446049250313e-16;   // np.spacing(1)
    recall[(int64_t)t * K * A * M + cell] = nd ? __ddiv_rn((double)tp, np_) : 0.0;
    int r = R - 1;
    const double rc_last = nd ? __ddiv_rn((double)tp, np_) : 0.0;
    // searchsorted(rc, recThrs, 'left') == nd: precision and score stay 0
    while (r >= 0 && (nd == 0 || rec[r] > rc_last)) { prec[r * rstride] = 0; sco[r * rstride] = 0; r--; }
    double env = 0;
    for (int64_t i = nd - 1; i >= 0; i--) {
        const double pr = __ddiv_rn((double)tp, __dadd_rn(__dadd_rn((double)fp, (double)tp), eps));
        env = (i == nd - 1 || !(env > pr)) ? pr : env;     // pr[i-1] = pr[i] if pr[i] > pr[i-1]
        const uint8_t st = state[(int64_t)list[i] * kCocoStates + sc];
        if (!(st & 2)) { if (st & 1) tp--; else fp--; }
        const double rc_prev = __ddiv_rn((double)tp, np_);
        const double s = kept_score[list[i]];
        while (r >= 0 && (i == 0 || rec[r] > rc_prev)) { prec[r * rstride] = env; sco[r * rstride] = s; r--; }
    }
}

// workspace of dt_coco_eval, 256-byte aligned pieces
// (the rank sort's pieces come last, so the earlier offsets do not depend on the number of categories)
struct CocoEvalWs {
    size_t det_cnts, det_m, det_area, det_rbox, kept_det, kept_rank, kept_score, state, iou, gtm, order, total;
    size_t rank_keys, rank_keys_out, rank_vals, rank_sorted, rank_flags, rank_pos, rank_temp, rank_temp_bytes, total_with_rank;
};
inline CocoEvalWs coco_eval_ws(int64_t n_det, int64_t n_chars, int64_t kept, int64_t n_iou, int64_t n_gt, int64_t n_order, int K = 0) {
    CocoEvalWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 255) / 256 * 256; return at; };
    w.det_cnts = take(4 * (size_t)n_chars);
    w.det_m = take(8 * (size_t)n_det);
    w.det_area = take(8 * (size_t)n_det);
    w.det_rbox = take(32 * (size_t)n_det);
    w.kept_det = take(4 * (size_t)kept);
    w.kept_rank = take(4 * (size_t)kept);
    w.kept_score = take(8 * (size_t)kept);
    w.state = take((size_t)kCocoStates * kept);
    w.iou = take(8 * (size_t)n_iou);
    w.gtm = take((size_t)kCocoStates * n_gt);
    w.order = take(4 * (size_t)n_order);
    w.total = o;
    w.rank_keys = take(8 * (size_t)kept);
    w.rank_keys_out = take(8 * (size_t)kept);
    w.rank_vals = take(4 * (size_t)kept);
    w.rank_sorted = take(4 * (size_t)kept);
    w.rank_flags = take(4 * (size_t)kCocoMaxDets * kept);
    w.rank_pos = take(4 * (size_t)kCocoMaxDets * kept);
    w.rank_temp_bytes = kept > 0 && K > 0 ? coco_rank_temp_bytes(kept, K) : 0;
    w.rank_temp = take(w.rank_temp_bytes);
    w.total_with_rank = o;
    return w;
}

inline cudaError_t coco_gt_launch(int n_ann, const int64_t* ann, const int64_t* parts, const double* xy, const uint32_t* ucounts,
                                  const char* chars, int* ws, uint32_t* out_cnts, uint32_t* tmp_cnts, int64_t* out_len, double* out_box,
                                  cudaStream_t st) {
    coco_gt_kernel<<<n_ann, 128, 0, st>>>(ann, parts, xy, ucounts, chars, ws, out_cnts, tmp_cnts, out_len, out_box);
    return cudaGetLastError();
}

// accumulate()'s lists for the three maxDets cuts (order[], laid out by order_off) from the kept slots of dt_coco_eval's workspace
inline cudaError_t coco_rank_launch(int64_t kept, int K, const int64_t* cat_kept, const int* kept_rank, const double* kept_score, int* order,
                                    uint8_t* ws, const CocoEvalWs& L, cudaStream_t st) {
    uint64_t* keys = reinterpret_cast<uint64_t*>(ws + L.rank_keys);
    uint64_t* keys_out = reinterpret_cast<uint64_t*>(ws + L.rank_keys_out);
    int* vals = reinterpret_cast<int*>(ws + L.rank_vals);
    int* sorted = reinterpret_cast<int*>(ws + L.rank_sorted);
    int* flags = reinterpret_cast<int*>(ws + L.rank_flags);
    int* pos = reinterpret_cast<int*>(ws + L.rank_pos);
    size_t temp = L.rank_temp_bytes;
    coco_rank_keys_kernel<<<(unsigned)((kept + 255) / 256), 256, 0, st>>>(kept, kept_score, keys, vals);
    cudaError_t e = cub::DeviceSegmentedSort::StableSortPairs(ws + L.rank_temp, temp, keys, keys_out, vals, sorted, (int)kept, K, cat_kept,
                                                              cat_kept + 1, st);
    if (e != cudaSuccess) return e;
    coco_rank_flags_kernel<<<(unsigned)((kept + 255) / 256), 256, 0, st>>>(kept, sorted, kept_rank, flags);
    temp = L.rank_temp_bytes;
    e = cub::DeviceScan::ExclusiveSum(ws + L.rank_temp, temp, flags, pos, (int64_t)kCocoMaxDets * kept, st);
    if (e != cudaSuccess) return e;
    coco_rank_scatter_kernel<<<(unsigned)((kCocoMaxDets * kept + 255) / 256), 256, 0, st>>>(kept, sorted, flags, pos, order);
    return cudaGetLastError();
}

inline cudaError_t coco_eval_launch(int segm, int num_images, int K, int n_active, const int64_t* pairs, const int64_t* cat_gt,
                                    const int64_t* cat_kept, const int64_t* order_off, int64_t n_det, const double* det_f,
                                    const int64_t* det_i, const char* det_chars, int64_t n_chars, int64_t kept, int64_t n_iou, int64_t n_gt,
                                    int64_t n_order, const double* gt_f, const int64_t* gt_i, const uint32_t* gt_cnts, const double* par,
                                    double* precision, double* recall, double* scores, double* ious, void* workspace, cudaStream_t st,
                                    const double* det_area = nullptr) {
    const CocoEvalWs L = coco_eval_ws(n_det, n_chars, kept, n_iou, n_gt, n_order, K);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    double* rle_area = reinterpret_cast<double*>(ws + L.det_area);
    CocoEvalArgs p;
    p.segm = segm; p.num_images = num_images; p.pairs = pairs;
    p.use_area = segm || det_area != nullptr;
    p.det_f = det_f; p.det_i = det_i;
    p.det_cnts = reinterpret_cast<uint32_t*>(ws + L.det_cnts); p.det_m = reinterpret_cast<int64_t*>(ws + L.det_m);
    p.det_area = det_area ? det_area : rle_area; p.det_rbox = reinterpret_cast<double*>(ws + L.det_rbox);
    p.gt_f = gt_f; p.gt_i = gt_i; p.gt_cnts = gt_cnts; p.par = par;
    p.kept_det = reinterpret_cast<int*>(ws + L.kept_det); p.kept_rank = reinterpret_cast<int*>(ws + L.kept_rank);
    p.kept_score = reinterpret_cast<double*>(ws + L.kept_score); p.state = ws + L.state;
    p.iou = ious ? ious : reinterpret_cast<double*>(ws + L.iou); p.gtm = ws + L.gtm;
    int* order = reinterpret_cast<int*>(ws + L.order);
    if (segm && n_det > 0) {
        coco_det_rle_kernel<<<(unsigned)((n_det + 127) / 128), 128, 0, st>>>(n_det, det_i, det_chars, const_cast<uint32_t*>(p.det_cnts), const_cast<int64_t*>(p.det_m), rle_area, const_cast<double*>(p.det_rbox));
    }
    if (n_active > 0) {
        coco_pair_kernel<<<n_active, 128, 0, st>>>(p);
    }
    if (kept > 0) {
        cudaError_t e = coco_rank_launch(kept, K, cat_kept, p.kept_rank, p.kept_score, order, ws, L, st);
        if (e != cudaSuccess) return e;
    }
    const int cells = K * kCocoAreas * kCocoMaxDets * kCocoThrs;
    if (cells > 0) {
        coco_accum_kernel<<<(cells + 127) / 128, 128, 0, st>>>(K, cat_gt, gt_f, gt_i, order_off, order, p.kept_score, p.state, par, precision, recall, scores);
    }
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ device-resident results
// utils.coco_eval.DeviceResults keeps detect() batches on the device as raw records, one per (image, slot) of each batch, in the order
// they were added.  At evaluate() they are flattened into the det_f / det_i / pairs / cat_kept / order_off tables of dt_coco_eval, in
// the order the host conversion gives them: by key = k * I + i (category index k, image index i), slot order inside a key.
//
//   coco_results_append_kernel   one thread per (image, slot) of a batch: the record, the slot's rank inside its class in the image,
//                                and the batch_results checks (class in 1..num_classes-1, slots grouped by class) as an error flag.
//   coco_results_count_kernel    one thread per record: the last record of each (image, class) group writes the group's size to its
//                                (category, image) bin; records of live slots with non-finite values set a flag.
//   coco_results_bins_kernel     one thread per bin: D, D > 0, min(D, 10), min(D, 100) and min(D, 100) G for the scans (torch.cumsum).
//   coco_results_scatter_kernel  one thread per record: its det_f / det_i row at its bin's start + its rank (a counting sort).
//   coco_results_pairs_kernel    one thread per bin: the pair row of a non-empty bin at its rank among them; one thread per category:
//                                cat_kept and order_off from the scans at the category's first bin.
// Each (category, image) bin is filled by one class of one image (category ids are distinct), so no two groups share a bin and the
// only atomics are the integer error flags.
//
// Subsets and class-agnostic evaluation (COCOeval's imgIds, catIds, useCats) only change the maps: cls_k takes a class to its category
// slot or -1, ord_i an image ordinal to its image index or -1 (records mapped to -1 take no part).  With `per` category slots per pair
// (useCats = 0: the evaluated categories, in COCOeval's concatenation order; otherwise 1) the records are counted in per * P fine bins,
// fine bin = image * per + slot (per > 1) or slot * I + image (per = 1), and pair p holds fine bins p * per .. p * per + per - 1 in a row,
// so its detections come in concatenation order.
// record: f32 [x1, y1, x2, y2, score]; i64 [image ordinal (-1: dead slot), class, rank in class, char offset, char count, h, w]
constexpr int kCocoRecF = 5, kCocoRecI = 7;
// the bin scans, int64 [5][K I] inclusive: D, D > 0 (= min(D, 1)), min(D, 10), min(D, 100), min(D, 100) G
constexpr int kCocoScanRows = 5;

__device__ __forceinline__ int64_t coco_lower_bound(const int64_t* a, int64_t n, int64_t v, bool upper) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < v || (upper && a[mid] == v)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// images [B, 3] int64: ordinal, h, w; str_offs [B cap + 1] the batch's string offsets (NULL without masks), placed at char_base.
// err[0] |= 1 and err[1] = min ordinal of an image whose live classes are outside 1..num_classes-1 or not grouped.
__global__ void coco_results_append_kernel(int B, int cap, int num_classes, const float* __restrict__ boxes, const float* __restrict__ scores,
                                           const int* __restrict__ classes, const int* __restrict__ counts, const int64_t* __restrict__ images,
                                           const int64_t* __restrict__ str_offs, int64_t char_base, float* __restrict__ rec_f,
                                           int64_t* __restrict__ rec_i, int* __restrict__ err) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)B * cap) return;
    const int b = (int)(e / cap), d = (int)(e % cap);
    const int n = min(max(counts[b], 0), cap);
    int64_t* R = rec_i + e * kCocoRecI;
    float* F = rec_f + e * kCocoRecF;
    if (d >= n) {
        R[0] = -1;
        for (int j = 1; j < kCocoRecI; j++) R[j] = 0;
        for (int j = 0; j < kCocoRecF; j++) F[j] = 0.f;
        return;
    }
    const int* cl = classes + (int64_t)b * cap;
    const int c = cl[d];
    const int64_t* im = images + 3 * (int64_t)b;
    if (c < 1 || c >= num_classes || (d > 0 && cl[d - 1] > c)) {
        atomicOr(err, 1);
        atomicMin(err + 1, (int)im[0]);
    }
    int r = 0;
    while (r < d && cl[d - 1 - r] == c) r++;
    R[0] = im[0]; R[1] = c; R[2] = r;
    if (str_offs) {
        R[3] = char_base + str_offs[e]; R[4] = str_offs[e + 1] - str_offs[e]; R[5] = im[1]; R[6] = im[2];
    } else {
        R[3] = R[4] = R[5] = R[6] = 0;
    }
    for (int j = 0; j < 4; j++) F[j] = boxes[4 * e + j];
    F[4] = scores[e];
}

// the category index of a record (-1: dead slot, or a class without a category); cls_k [num_cls], ord_i [ordinals] -> gt image index
__device__ __forceinline__ int coco_rec_cat(const int64_t* R, int num_cls, const int* cls_k) {
    const int64_t o = R[0], c = R[1];
    if (o < 0 || c < 0 || c >= num_cls) return -1;
    return cls_k[c];
}

__device__ __forceinline__ int64_t coco_fine_bin(int k, int i, int I, int per) {
    return per > 1 ? (int64_t)i * per + k : (int64_t)k * I + i;
}

__global__ void coco_results_count_kernel(int64_t n, const float* __restrict__ rec_f, const int64_t* __restrict__ rec_i, int num_cls,
                                          const int* __restrict__ cls_k, const int* __restrict__ ord_i, int I, int per, int* __restrict__ bin_cnt,
                                          int* __restrict__ nonfinite) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int64_t* R = rec_i + r * kCocoRecI;
    const int k = coco_rec_cat(R, num_cls, cls_k);
    if (k < 0 || ord_i[R[0]] < 0) return;
    const float* F = rec_f + r * kCocoRecF;
    bool fin = true;
    for (int j = 0; j < kCocoRecF; j++) fin = fin && isfinite(F[j]);
    if (!fin) atomicOr(nonfinite, 1);
    const bool last = r + 1 == n || R[kCocoRecI] != R[0] || R[kCocoRecI + 1] != R[1];
    if (last) bin_cnt[coco_fine_bin(k, ord_i[R[0]], I, per)] = (int)R[2] + 1;
}

__global__ void coco_results_bins_kernel(int64_t nb, int per, const int* __restrict__ bin_cnt, const int64_t* __restrict__ gt_keys, int64_t G,
                                         int64_t* __restrict__ vals) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    int64_t D = 0;
    for (int c = 0; c < per; c++) D += bin_cnt[b * per + c];
    int64_t gn = 0;
    if (D > 0) gn = coco_lower_bound(gt_keys, G, b, true) - coco_lower_bound(gt_keys, G, b, false);
    const int64_t kept = D < kCocoKeep ? D : kCocoKeep;
    vals[b] = D;
    vals[nb + b] = D > 0;
    vals[2 * nb + b] = D < 10 ? D : 10;
    vals[3 * nb + b] = kept;
    vals[4 * nb + b] = kept * gn;
}

// det_f: (score, x1, y1, x2 - x1 + 1, y2 - y1 + 1), each term the double of the stored float, as the host's float64 arithmetic
// det_key: each row's fine bin (its pair when per = 1)
__global__ void coco_results_scatter_kernel(int64_t n, const float* __restrict__ rec_f, const int64_t* __restrict__ rec_i, int num_cls,
                                            const int* __restrict__ cls_k, const int* __restrict__ ord_i, int I, int per,
                                            const int* __restrict__ bin_cnt, const int64_t* __restrict__ scan, int64_t* __restrict__ det_key,
                                            double* __restrict__ det_f, int64_t* __restrict__ det_i) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int64_t* R = rec_i + r * kCocoRecI;
    const int k = coco_rec_cat(R, num_cls, cls_k);
    if (k < 0 || ord_i[R[0]] < 0) return;
    const int64_t key = coco_fine_bin(k, ord_i[R[0]], I, per), b = key / per;
    int64_t pos = (b > 0 ? scan[b - 1] : 0) + R[2];
    for (int64_t f = b * per; f < key; f++) pos += bin_cnt[f];
    const float* F = rec_f + r * kCocoRecF;
    const double x1 = F[0], y1 = F[1], x2 = F[2], y2 = F[3];
    double* D = det_f + pos * kCocoDetF;
    D[0] = (double)F[4]; D[1] = x1; D[2] = y1;
    D[3] = __dadd_rn(__dsub_rn(x2, x1), 1.0); D[4] = __dadd_rn(__dsub_rn(y2, y1), 1.0);
    int64_t* DI = det_i + pos * kCocoDetI;
    DI[0] = R[3]; DI[1] = R[4]; DI[2] = R[5]; DI[3] = R[6];
    det_key[pos] = key;
}

__global__ void coco_results_pairs_kernel(int K, int I, const int64_t* __restrict__ scan, const int64_t* __restrict__ gt_keys, int64_t G,
                                          int64_t* __restrict__ pairs, int64_t* __restrict__ cat_kept, int64_t* __restrict__ order_off) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nb = (int64_t)K * I;
    auto excl = [&](int row, int64_t b) -> int64_t { return b > 0 ? scan[row * nb + b - 1] : 0; };
    if (t < nb) {
        const int64_t d0 = excl(0, t), D = scan[t] - d0;
        if (D > 0) {
            const int64_t g0 = coco_lower_bound(gt_keys, G, t, false), g1 = coco_lower_bound(gt_keys, G, t, true);
            int64_t* P = pairs + excl(1, t) * kCocoPairCols;
            P[0] = t; P[1] = d0; P[2] = D; P[3] = g0; P[4] = g1 - g0; P[5] = excl(3, t); P[6] = excl(4, t);
        }
    }
    if (t <= K) {
        const int64_t b = t * I;                  // category t's first bin; t == K: the totals
        const int64_t T1 = excl(1, nb), T2 = excl(2, nb);
        cat_kept[t] = excl(3, b);
        order_off[t] = excl(1, b);
        order_off[(K + 1) + t] = T1 + excl(2, b);
        order_off[2 * (K + 1) + t] = T1 + T2 + excl(3, b);
    }
}

inline cudaError_t coco_results_append_launch(int B, int cap, int num_classes, const float* boxes, const float* scores, const int* classes,
                                              const int* counts, const int64_t* images, const int64_t* str_offs, int64_t char_base, float* rec_f,
                                              int64_t* rec_i, int* err, cudaStream_t st) {
    const int64_t n = (int64_t)B * cap;
    coco_results_append_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(B, cap, num_classes, boxes, scores, classes, counts, images, str_offs,
                                                                           char_base, rec_f, rec_i, err);
    return cudaGetLastError();
}

inline cudaError_t coco_results_count_launch(int64_t n, const float* rec_f, const int64_t* rec_i, int num_cls, const int* cls_k, const int* ord_i,
                                             int I, int K, int per, const int64_t* gt_keys, int64_t G, int* bin_cnt, int64_t* vals, int* nonfinite,
                                             cudaStream_t st) {
    const int64_t nb = (int64_t)K * I;
    if (n > 0) coco_results_count_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, rec_f, rec_i, num_cls, cls_k, ord_i, I, per, bin_cnt, nonfinite);
    if (nb > 0) coco_results_bins_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, st>>>(nb, per, bin_cnt, gt_keys, G, vals);
    return cudaGetLastError();
}

inline cudaError_t coco_results_write_launch(int64_t n, const float* rec_f, const int64_t* rec_i, int num_cls, const int* cls_k, const int* ord_i,
                                             int I, int K, int per, const int* bin_cnt, const int64_t* scan, const int64_t* gt_keys, int64_t G,
                                             int64_t* det_key, double* det_f, int64_t* det_i, int64_t* pairs, int64_t* cat_kept, int64_t* order_off,
                                             cudaStream_t st) {
    const int64_t nb = (int64_t)K * I, nt = nb > K + 1 ? nb : K + 1;
    if (n > 0) coco_results_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, rec_f, rec_i, num_cls, cls_k, ord_i, I, per, bin_cnt, scan,
                                                                                      det_key, det_f, det_i);
    coco_results_pairs_kernel<<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(K, I, scan, gt_keys, G, pairs, cat_kept, order_off);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ per-image records (evalImgs)
// COCOeval.evaluate() keeps one record per (category, area range, image) whose pair has detections or gts: which gt each detection
// matched at each threshold, which detection each gt matched last, and which of them were ignored.  After dt_coco_eval, from its
// workspace (kept slots, segm areas) and the IoU matrices it kept (never recomputed):
//
//   coco_eval_imgs_kernel   one CTA per pair of a union table (the sorted pair indices of the pairs with detections and of those with
//                           gts): per gt and area range its place in the stable ignore-last order; then one thread per (area range,
//                           threshold) repeats coco_pair_kernel's matching, keeping the indices it matched.
//
// Outputs, with state c = area range * 10 + threshold as in state[]:
//   slot_det [kept]        detection index of each kept slot (for the host's mapping to detection ids and scores)
//   dt_gt [kept][40]       index in its pair (annotation order) of the gt the kept detection matched, -1 for none
//   dt_ig [kept][40]       evaluateImg's dtIgnore
//   gt_dt [gts][40]        rank in its pair of the last kept detection that matched the gt (a crowd gt matches several), -1 for none
//   gt_pos [gts][4]        the gt's position in the area range's ignore-last order;  gt_ig [gts][4] its ignore flag
struct CocoEvalImgsArgs {
    int segm, use_area;       // as CocoEvalArgs
    int64_t n_active, n_gt;
    const int64_t* ukeys; const int64_t* pairs; const int64_t* gt_keys;
    const double* det_f; const double* det_area; const int* kept_det;
    const double* gt_f; const int64_t* gt_i; const double* par; const double* iou;
    int* slot_det; int* dt_gt; uint8_t* dt_ig; int* gt_dt; int* gt_pos; uint8_t* gt_ig;
};

__global__ void coco_eval_imgs_kernel(CocoEvalImgsArgs p) {
    const int64_t key = p.ukeys[blockIdx.x];
    const int64_t g0 = coco_lower_bound(p.gt_keys, p.n_gt, key, false), G = coco_lower_bound(p.gt_keys, p.n_gt, key, true) - g0;
    int64_t lo = 0, hi = p.n_active;                 // the pair's row among the pairs with detections, if it has any
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (p.pairs[mid * kCocoPairCols] < key) lo = mid + 1; else hi = mid;
    }
    const int64_t* T = lo < p.n_active && p.pairs[lo * kCocoPairCols] == key ? p.pairs + lo * kCocoPairCols : nullptr;
    const int64_t D = T ? T[2] : 0, k0 = T ? T[5] : 0, i0 = T ? T[6] : 0;
    const int64_t Dk = D < kCocoKeep ? D : kCocoKeep;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int64_t e = tid; e < G * kCocoStates; e += nt) p.gt_dt[g0 * kCocoStates + e] = -1;
    for (int64_t r = tid; r < Dk; r += nt) p.slot_det[k0 + r] = p.kept_det[k0 + r];
    // gtind = np.argsort(_ignore, kind='mergesort'): the kept gts in annotation order, then the ignored ones
    for (int ar = tid; ar < kCocoAreas; ar += nt) {
        const double* rng = p.par + kCocoParAreas + 2 * ar;
        int64_t n_keep = 0;
        for (int64_t g = 0; g < G; g++) n_keep += !(p.gt_i[(g0 + g) * kCocoGtI + 4] != 0 || coco_out(p.gt_f[(g0 + g) * kCocoGtF + 4], rng));
        int64_t a = 0, b = n_keep;
        for (int64_t g = 0; g < G; g++) {
            const bool ig = p.gt_i[(g0 + g) * kCocoGtI + 4] != 0 || coco_out(p.gt_f[(g0 + g) * kCocoGtF + 4], rng);
            p.gt_pos[(g0 + g) * kCocoAreas + ar] = (int)(ig ? b++ : a++);
            p.gt_ig[(g0 + g) * kCocoAreas + ar] = ig;
        }
    }
    __syncthreads();
    // coco_pair_kernel's matching, step for step; a gt is taken when gt_dt holds a rank (the last one for a crowd gt)
    for (int c = tid; c < kCocoStates; c += nt) {
        const int ar = c / kCocoThrs, t = c % kCocoThrs;
        const double* rng = p.par + kCocoParAreas + 2 * ar;
        int* gm = p.gt_dt + g0 * kCocoStates + c;    // gm[g * kCocoStates]
        for (int64_t dr = 0; dr < Dk; dr++) {
            double best = p.par[kCocoParThrs + t];
            int64_t m = -1;
            bool m_ig = false;
            for (int pass = 0; pass < 2; pass++) {
                for (int64_t g = 0; g < G; g++) {
                    const int64_t* GI = p.gt_i + (g0 + g) * kCocoGtI;
                    const bool ig = GI[4] != 0 || coco_out(p.gt_f[(g0 + g) * kCocoGtF + 4], rng);
                    if ((int)ig != pass) continue;
                    if (gm[g * kCocoStates] >= 0 && !GI[4]) continue;
                    if (m > -1 && !m_ig && ig) goto matched;
                    const double o = p.iou[i0 + dr * G + g];
                    if (o < best) continue;
                    best = o; m = g; m_ig = ig;
                }
            }
        matched:
            bool hit = false, dig = false;
            if (m > -1) {
                dig = m_ig;
                hit = p.gt_i[(g0 + m) * kCocoGtI + 5] != 0;
                gm[m * kCocoStates] = (int)dr;
            }
            const int64_t d = p.kept_det[k0 + dr];
            const double area = p.use_area ? p.det_area[d] : __dmul_rn(p.det_f[d * kCocoDetF + 3], p.det_f[d * kCocoDetF + 4]);
            if (!hit && coco_out(area, rng)) dig = true;
            p.dt_gt[(k0 + dr) * kCocoStates + c] = (int)m;
            p.dt_ig[(k0 + dr) * kCocoStates + c] = dig;
        }
    }
}

// workspace: the one dt_coco_eval has just filled, of the same sizes; ious: the IoU matrices it kept
inline cudaError_t coco_eval_imgs_launch(int segm, int n_union, const int64_t* ukeys, int n_active, const int64_t* pairs, int64_t n_det,
                                         int64_t n_chars, int64_t kept, int64_t n_iou, int64_t n_gt, int64_t n_order, const int64_t* gt_keys,
                                         const double* det_f, const double* gt_f, const int64_t* gt_i, const double* par, const double* ious,
                                         const void* workspace, int* slot_det, int* dt_gt, uint8_t* dt_ig, int* gt_dt, int* gt_pos,
                                         uint8_t* gt_ig, cudaStream_t st, const double* det_area = nullptr) {
    const CocoEvalWs L = coco_eval_ws(n_det, n_chars, kept, n_iou, n_gt, n_order);
    const uint8_t* ws = reinterpret_cast<const uint8_t*>(workspace);
    CocoEvalImgsArgs p;
    p.segm = segm; p.use_area = segm || det_area != nullptr; p.n_active = n_active; p.n_gt = n_gt;
    p.ukeys = ukeys; p.pairs = pairs; p.gt_keys = gt_keys;
    p.det_f = det_f; p.det_area = det_area ? det_area : reinterpret_cast<const double*>(ws + L.det_area); p.kept_det = reinterpret_cast<const int*>(ws + L.kept_det);
    p.gt_f = gt_f; p.gt_i = gt_i; p.par = par; p.iou = ious;
    p.slot_det = slot_det; p.dt_gt = dt_gt; p.dt_ig = dt_ig; p.gt_dt = gt_dt; p.gt_pos = gt_pos; p.gt_ig = gt_ig;
    if (n_union > 0) coco_eval_imgs_kernel<<<n_union, 64, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace dt

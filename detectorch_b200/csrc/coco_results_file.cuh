// detectorch_b200 -- a COCO results json read on the device: the detections pycocotools' COCO.loadRes(file) hands to COCOeval, as
// the tables of dt_coco_eval (utils.coco_eval.load_results).  The file's bytes are uploaded once; everything after runs here, with
// 64-bit offsets throughout.
//
// Structural pass, one thread per byte:
//   cf_quote_kernel      q[i] = 1 for a '"' after an even run of backslashes (an odd run escapes it)
//   CUB scan (xor)       s[i] = q[0] ^ .. ^ q[i]: 1 inside a string, its opening quote included
//   cf_delta_kernel      +1 / -1 for each { [ / } ] outside strings; CUB scan (sum): the depth after each byte
//   cf_classify_kernel   the separators (the top-level '[', its ']' and the ',' at depth 1), counted, and the errors a record cannot see:
//                        a byte >= 0x80, anything but blanks around the one top-level array, a depth below 0 or not back to 0 at the
//                        end, a string still open at the end, a top level closed by '}'
//   CUB select           the separators' positions: record r is the text between separators r and r + 1
// Record pass:
//   cf_record_kernel     one thread per record: a strict JSON state machine over its bytes (json.loads' grammar without NaN and
//                        Infinity; values of unknown keys skipped at any depth up to kCfMaxDepth), the last occurrence of each key kept;
//                        image_id / category_id (integer literals in int64, looked up in the sorted ids of the ground truth), score and
//                        bbox (correctly rounded doubles), the segmentation's compressed RLE (the raw span of 'counts', its decoded
//                        length, 'size').  Errors are bits or-ed into info[1], the first record with one min-ed into info[4].
//   cf_counts_kernel     each record's counts decoded at its offset (the caller's scan of the lengths), with list input's string checks
//   coco_det_check_kernel / coco_det_rle_kernel (coco_eval.cuh): run sums; in the segm branch the RLE area and toBbox
//   cf_columns_kernel    loadRes's area (bbox branch: w h, segm branch: the RLE area) and box (segm branch, no bbox: toBbox); sort keys
//   CUB radix sort       by key = category index * I + image index, stable: file order inside a key; unknown categories last
//   cf_gather_kernel     det_f / det_i / area / loadRes id (1 + file index) in key order, as dt_coco_eval takes them
//
// Numbers: w, the first 19 significant digits, and q, the exponent of the rest (the value lies in [w, w + 1) 10^q, = w 10^q when there
// are no more digits).  w 10^q is bounded below and above by Eisel-Lemire's product with the 128-bit truncated power of five of
// coco_results_pow5.inc (10^q = (t + e) 2^(q - s), 0 <= e < 1); when both bounds round to the same double it is the answer.
// Otherwise (more digits that matter, or a product too close to a halfway point) the double is decided among that one and its
// neighbours by comparing the exact decimal (its first kCfBigDigits significant digits, and whether a nonzero digit follows) with the
// halfway points in big-integer arithmetic.  A halfway point has at most 769 significant digits, so the digits cut off can only
// break a tie.
#pragma once
#include <cstdint>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <cuda_runtime.h>

#include "coco_eval.cuh"
#include "coco_results_pow5.inc"

namespace dt {

__device__ const uint64_t kCfPow5T[] = DT_POW5_T;
__device__ const int16_t kCfPow5S[] = DT_POW5_S;

// error bits (info[1]); utils.coco_eval mirrors them
enum : unsigned {
    kCfSyntax = 1u << 0,         // not JSON
    kCfAscii = 1u << 1,          // a byte >= 0x80
    kCfTop = 1u << 2,            // the top level is not one array
    kCfNotObject = 1u << 3,      // an element that is not an object
    kCfDepth = 1u << 4,          // nesting deeper than kCfMaxDepth inside a record
    kCfNonFinite = 1u << 5,      // a score / bbox number whose double is not finite
    kCfImageId = 1u << 6,        // image_id missing or not an integer literal in int64
    kCfImageUnknown = 1u << 7,   // image_id not an image of the ground truth
    kCfCategoryId = 1u << 8,     // category_id missing or not an integer literal in int64
    kCfScore = 1u << 9,          // score missing or not a number
    kCfRle = 1u << 10,           // a segmentation dict that is not a compressed RLE: string counts, size [h, w] integers, 1 <= h w < 2^32
    kCfCounts = 1u << 11,        // counts outside the RLE alphabet, with a value over 6 chars, or ending inside a value
    kCfSums = 1u << 12,          // counts whose runs do not sum to h w
};
// summary bits (info[2]): some record lacks what a branch or an iou type needs
enum : unsigned { kCfNoBbox = 1u, kCfBadBbox = 2u, kCfNoRle = 4u };
// per-record flags (rec_b)
enum : uint8_t { kCfHasBbox = 1, kCfBboxOk = 2, kCfBboxEmpty = 4, kCfHasRle = 8, kCfHasCaption = 16 };
// info [8] int64: separators, error bits, summary bits, records of unknown categories, first record with an error (the caller sets
// INT64_MAX), top-level '[' count, empty array (1: the one record slot is blank), unused
enum { kCfInfoSeps = 0, kCfInfoErr = 1, kCfInfoSum = 2, kCfInfoDropped = 3, kCfInfoFirst = 4, kCfInfoOpen = 5, kCfInfoEmpty = 6, kCfInfo = 8 };
constexpr int kCfRecF = 5, kCfRecI = 6;   // rec_f: score, bbox x y w h; rec_i: image index, category index (-1), counts begin, end, h, w
constexpr int kCfMaxDepth = 64;
constexpr int kCfLimbs = 128, kCfBigDigits = 780;
constexpr int64_t kCfExpCap = 1000000000;
constexpr uint64_t kCfInf = 0x7ff0000000000000ull;

__device__ __forceinline__ bool cf_ws(int c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
__device__ __forceinline__ bool cf_digit(int c) { return c >= '0' && c <= '9'; }
__device__ __forceinline__ int cf_hex(int c) {
    const int l = c | 0x20;
    return cf_digit(c) ? c - '0' : (l >= 'a' && l <= 'f') ? l - 'a' + 10 : -1;
}

// warp-aggregated or / add into one info word (many records raise the same bit)
__device__ __forceinline__ void cf_or(unsigned long long* a, unsigned v) {
    const unsigned m = __activemask();
    const unsigned r = __reduce_or_sync(m, v);
    if (r && (threadIdx.x & 31) == __ffs(m) - 1) atomicOr(a, (unsigned long long)r);
}
__device__ __forceinline__ void cf_add(unsigned long long* a, unsigned v) {
    const unsigned m = __activemask();
    const unsigned r = __reduce_add_sync(m, v);
    if (r && (threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(a, (unsigned long long)r);
}
__device__ __forceinline__ void cf_fail(unsigned long long* info, unsigned err, int64_t r) {
    atomicOr(info + kCfInfoErr, (unsigned long long)err);
    atomicMin(reinterpret_cast<long long*>(info + kCfInfoFirst), (long long)r);
}

// ------------------------------------------------------------------------------------------------ structural pass
__global__ void cf_quote_kernel(int64_t n, const uint8_t* __restrict__ t, uint8_t* __restrict__ q) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t v = 0;
    if (t[i] == '"') {               // each backslash run is walked by the quote after it only: linear in the file
        int64_t j = i - 1;
        while (j >= 0 && t[j] == '\\') j--;
        v = ((i - 1 - j) & 1) == 0;
    }
    q[i] = v;
}

struct CfXor {
    __device__ __forceinline__ uint8_t operator()(uint8_t a, uint8_t b) const { return a ^ b; }
};

__device__ __forceinline__ int cf_bracket(int c) { return (c == '{' || c == '[') ? 1 : (c == '}' || c == ']') ? -1 : 0; }

__global__ void cf_delta_kernel(int64_t n, const uint8_t* __restrict__ t, const uint8_t* __restrict__ q, const uint8_t* __restrict__ s,
                                int* __restrict__ delta) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    delta[i] = (s[i] | q[i]) ? 0 : cf_bracket(t[i]);
}

__global__ void cf_classify_kernel(int64_t n, const uint8_t* __restrict__ t, const uint8_t* __restrict__ q, const uint8_t* __restrict__ s,
                                   const int* __restrict__ depth, uint8_t* __restrict__ sep, unsigned long long* __restrict__ info) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = t[i];
    const bool out = !(s[i] | q[i]);
    const int d = depth[i], before = d - (out ? cf_bracket(c) : 0);
    unsigned err = 0;
    bool is_sep = false, open = false;
    if (c >= 0x80) err |= kCfAscii;
    if (d < 0) err |= kCfTop;
    if (before == 0 && !(out && cf_ws(c))) {
        if (out && c == '[') is_sep = open = true;
        else err |= kCfTop;
    }
    if (out && before == 1 && d == 0) {
        is_sep = true;
        if (c != ']') err |= kCfTop;
    }
    if (out && before == 1 && c == ',') is_sep = true;
    if (i == n - 1) {
        if (s[i]) err |= kCfSyntax;
        if (d != 0) err |= kCfTop;
    }
    sep[i] = is_sep;
    cf_add(info + kCfInfoSeps, is_sep);
    cf_add(info + kCfInfoOpen, open);
    if (err) atomicOr(info + kCfInfoErr, (unsigned long long)err);
}

// ------------------------------------------------------------------------------------------------ JSON tokens
struct CfText {
    const uint8_t* t;
    int64_t end;
    __device__ __forceinline__ int at(int64_t p) const { return p < end ? t[p] : 0; }   // 0: past the record, valid nowhere
};

__device__ __forceinline__ int64_t cf_skip_ws(const CfText& x, int64_t p) {
    while (cf_ws(x.at(p))) p++;
    return p;
}

// x.at(p) == '"' -> the position after the closing quote (-1: not a JSON string); *units: decoded characters (an escape is one)
__device__ __forceinline__ int64_t cf_string(const CfText& x, int64_t p, int64_t* units) {
    int64_t u = 0;
    p++;
    for (;;) {
        const int c = x.at(p);
        if (c == '"') { *units = u; return p + 1; }
        if (c < 0x20 || c >= 0x80) return -1;
        if (c == '\\') {
            const int e = x.at(p + 1);
            if (e == 'u') {
                if ((cf_hex(x.at(p + 2)) | cf_hex(x.at(p + 3)) | cf_hex(x.at(p + 4)) | cf_hex(x.at(p + 5))) < 0) return -1;
                p += 6;
            } else if (e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't') {
                p += 2;
            } else {
                return -1;
            }
        } else {
            p++;
        }
        u++;
    }
}

// one decoded character of a validated string at p (a \u escape gives its code unit)
__device__ __forceinline__ int cf_unescape(const uint8_t* t, int64_t& p) {
    const int c = t[p];
    if (c != '\\') { p++; return c; }
    const int e = t[p + 1];
    if (e == 'u') {
        const int v = (cf_hex(t[p + 2]) << 12) | (cf_hex(t[p + 3]) << 8) | (cf_hex(t[p + 4]) << 4) | cf_hex(t[p + 5]);
        p += 6;
        return v;
    }
    p += 2;
    return e == 'b' ? 8 : e == 'f' ? 12 : e == 'n' ? 10 : e == 'r' ? 13 : e == 't' ? 9 : e;
}

// does the validated string content [b, e) decode to lit?
template <int N>
__device__ bool cf_key_is(const uint8_t* t, int64_t b, int64_t e, const char (&lit)[N]) {
    int i = 0;
    while (b < e) {
        const int c = cf_unescape(t, b);
        if (i >= N - 1 || c != lit[i]) return false;
        i++;
    }
    return i == N - 1;
}

// a key: its string, blanks, ':', blanks -> the position of the value (-1: syntax error); [*kb, *ke): the key's raw content
__device__ __forceinline__ int64_t cf_key(const CfText& x, int64_t p, int64_t* kb, int64_t* ke) {
    if (x.at(p) != '"') return -1;
    int64_t u;
    const int64_t q = cf_string(x, p, &u);
    if (q < 0) return -1;
    *kb = p + 1; *ke = q - 1;
    p = cf_skip_ws(x, q);
    if (x.at(p) != ':') return -1;
    return cf_skip_ws(x, p + 1);
}

struct CfNumber {
    int64_t int_beg, int_end, frac_beg, frac_end, exp;
    bool neg, is_int;
};

// at a '-' or a digit: a JSON number -> the position after it (-1: not one)
__device__ __forceinline__ int64_t cf_number(const CfText& x, int64_t p, CfNumber& m) {
    m.neg = x.at(p) == '-';
    if (m.neg) p++;
    const int c = x.at(p);
    if (!cf_digit(c)) return -1;
    m.int_beg = p;
    if (c == '0') p++;
    else while (cf_digit(x.at(p))) p++;
    m.int_end = m.frac_beg = m.frac_end = p;
    m.is_int = true;
    m.exp = 0;
    if (x.at(p) == '.') {
        p++;
        if (!cf_digit(x.at(p))) return -1;
        m.frac_beg = p;
        while (cf_digit(x.at(p))) p++;
        m.frac_end = p;
        m.is_int = false;
    }
    if ((x.at(p) | 0x20) == 'e') {
        m.is_int = false;
        p++;
        const bool en = x.at(p) == '-';
        if (en || x.at(p) == '+') p++;
        if (!cf_digit(x.at(p))) return -1;
        int64_t e = 0;
        for (; cf_digit(x.at(p)); p++)
            if (e < kCfExpCap) e = e * 10 + (x.at(p) - '0');
        m.exp = en ? -e : e;
    }
    return p;
}

// the k-th digit of the integer part followed by the fraction
__device__ __forceinline__ int cf_digit_at(const uint8_t* t, const CfNumber& m, int64_t k) {
    const int64_t ni = m.int_end - m.int_beg;
    return t[k < ni ? m.int_beg + k : m.frac_beg + (k - ni)] - '0';
}

// an integer literal in int64
__device__ __forceinline__ bool cf_int64(const uint8_t* t, const CfNumber& m, int64_t* v) {
    const int64_t n = m.int_end - m.int_beg;
    if (!m.is_int || n > 19) return false;
    uint64_t u = 0;
    for (int64_t k = 0; k < n; k++) u = u * 10 + (uint64_t)(t[m.int_beg + k] - '0');
    if (u > (m.neg ? (1ull << 63) : (1ull << 63) - 1)) return false;
    *v = m.neg ? (int64_t)(0ull - u) : (int64_t)u;
    return true;
}

// ------------------------------------------------------------------------------------------------ decimal -> double
// Bits of the double nearest to z 2^e0, z = m' t (+ m' for the upper bound), m' = m normalised to 64 bits, t = 5^q's table entry:
// the lower (upper) bound of m 10^q, rounded to nearest, ties to even; kCfInf past the largest double.
__device__ __forceinline__ uint64_t cf_round(uint64_t m, int q, bool upper) {
    const int lz = __clzll(m);
    const uint64_t w = m << lz;
    const int qi = q - DT_POW5_Q_MIN;
    const uint64_t th = kCfPow5T[2 * qi], tl = kCfPow5T[2 * qi + 1];
    uint64_t z0 = w * tl, z1 = __umul64hi(w, tl), z2 = __umul64hi(w, th);
    const uint64_t a = w * th;
    z1 += a;
    z2 += z1 < a;
    if (upper) {
        z0 += w;
        if (z0 < w && ++z1 == 0) z2++;
    }
    const int msb = 191 - __clzll(z2);                // z >= 2^190
    const int e0 = q - (int)kCfPow5S[qi] - lz;
    int u = msb + e0 - 52;                            // the result's unit: 2^u
    if (u < -1074) u = -1074;
    const int sh = u - e0 - 128;                      // >= 10: the unit is a bit of z2 or above
    uint64_t mant, rb, sticky;
    if (sh >= 65) { mant = 0; rb = 0; sticky = 1; }
    else if (sh == 64) { mant = 0; rb = z2 >> 63; sticky = (z2 << 1) | z1 | z0; }
    else { mant = z2 >> sh; rb = (z2 >> (sh - 1)) & 1; sticky = (z2 & ((1ull << (sh - 1)) - 1)) | z1 | z0; }
    if (rb && (sticky || (mant & 1))) mant++;
    if (mant == (1ull << 53)) { mant >>= 1; u++; }
    if (mant < (1ull << 52)) return mant;             // subnormal or zero (u is -1074)
    const int E = u + 1075;
    if (E >= 2047) return kCfInf;
    return ((uint64_t)E << 52) | (mant & ((1ull << 52) - 1));
}

struct CfBig {
    uint32_t v[kCfLimbs];
    int n;                                            // limbs in use, no leading zero limb
};

__device__ void cf_big_mul(CfBig& a, uint32_t m, uint32_t add) {
    uint64_t c = add;
    for (int i = 0; i < a.n; i++) {
        const uint64_t x = (uint64_t)a.v[i] * m + c;
        a.v[i] = (uint32_t)x;
        c = x >> 32;
    }
    if (c && a.n < kCfLimbs) a.v[a.n++] = (uint32_t)c;
}

__device__ void cf_big_pow5(CfBig& a, int64_t e) {
    for (; e >= 13; e -= 13) cf_big_mul(a, 1220703125u, 0);
    uint32_t p = 1;
    for (; e > 0; e--) p *= 5;
    cf_big_mul(a, p, 0);
}

__device__ void cf_big_shl(CfBig& a, int64_t s) {
    if (a.n == 0) return;
    const int w = (int)(s >> 5), b = (int)(s & 31);
    const int n = min(a.n + w + 1, kCfLimbs);
    for (int i = n - 1; i >= 0; i--) {
        const int j = i - w;
        const uint32_t hi = (j >= 0 && j < a.n) ? a.v[j] : 0u, lo = (j >= 1 && j - 1 < a.n) ? a.v[j - 1] : 0u;
        a.v[i] = b ? (hi << b) | (lo >> (32 - b)) : hi;
    }
    a.n = n;
    while (a.n > 0 && a.v[a.n - 1] == 0) a.n--;
}

__device__ int cf_big_cmp(const CfBig& a, const CfBig& b) {
    if (a.n != b.n) return a.n < b.n ? -1 : 1;
    for (int i = a.n - 1; i >= 0; i--)
        if (a.v[i] != b.v[i]) return a.v[i] < b.v[i] ? -1 : 1;
    return 0;
}

// the sign of D 10^e - h, D the nd digits from digit f, h the halfway point between the double of bits b, c 2^k, and the next one up:
// (2 c + 1) 2^(k - 1); with sticky (nonzero digits after the nd) a tie counts as above
__device__ int cf_cmp_half(const uint8_t* t, const CfNumber& m, int64_t f, int64_t nd, int64_t e, bool sticky, uint64_t b, CfBig& L, CfBig& R) {
    const int E = (int)(b >> 52);
    const uint64_t c = (b & ((1ull << 52) - 1)) | (E ? 1ull << 52 : 0);
    const int64_t k2 = (E ? E - 1075 : -1074) - 1;
    L.n = 0;
    for (int64_t k = f; k < f + nd;) {
        uint32_t chunk = 0, mul = 1;
        for (int j = 0; j < 9 && k < f + nd; j++, k++) { chunk = chunk * 10 + (uint32_t)cf_digit_at(t, m, k); mul *= 10; }
        cf_big_mul(L, mul, chunk);
    }
    const uint64_t h = 2 * c + 1;
    R.v[0] = (uint32_t)h; R.v[1] = (uint32_t)(h >> 32); R.n = (h >> 32) ? 2 : 1;
    if (e >= 0) cf_big_pow5(L, e); else cf_big_pow5(R, -e);
    if (e >= k2) cf_big_shl(L, e - k2); else cf_big_shl(R, k2 - e);
    const int r = cf_big_cmp(L, R);
    return r == 0 && sticky ? 1 : r;
}

// the correctly rounded double of digits f .. f + ns - 1 times 10^e10, from a candidate b within a few units of it
__device__ uint64_t cf_decide(const uint8_t* t, CfNumber m, int64_t f, int64_t ns, int64_t e10, uint64_t b) {
    CfBig L, R;
    const int64_t nd = ns < kCfBigDigits ? ns : kCfBigDigits;
    const int64_t e = e10 + (ns - nd);
    const bool sticky = ns > nd;
    for (int it = 0; it < 8; it++) {
        if (b > 0) {
            const int c = cf_cmp_half(t, m, f, nd, e, sticky, b - 1, L, R);
            if (c < 0) { b--; continue; }
            if (c == 0) return ((b - 1) & 1) ? b : b - 1;
        }
        if (b < kCfInf) {
            const int c = cf_cmp_half(t, m, f, nd, e, sticky, b, L, R);
            if (c > 0) { b++; continue; }
            if (c == 0) return (b & 1) ? b + 1 : b;
        }
        break;
    }
    return b;
}

// the double json.loads gives a number (float(text); an integer literal's exact value, converted the same way) -> its bits;
// *finite = false when that is not finite (float() overflows).  Without kExact, a number the bounds leave open sets *open and gets a
// candidate within a unit (cf_exact_kernel decides it).
template <bool kExact>
__device__ __forceinline__ uint64_t cf_to_double(const uint8_t* t, const CfNumber& m, bool* finite, bool* open) {
    const int64_t ni = m.int_end - m.int_beg, nd = ni + (m.frac_end - m.frac_beg);
    *finite = true;
    int64_t f = 0;
    while (f < nd && cf_digit_at(t, m, f) == 0) f++;
    if (f == nd) return (m.neg && !m.is_int) ? 1ull << 63 : 0;     // the integer -0 is int 0
    const uint64_t sign = m.neg ? 1ull << 63 : 0;
    int64_t l = nd - 1;
    while (cf_digit_at(t, m, l) == 0) l--;
    const int64_t ns = l - f + 1, e10 = m.exp + (ni - 1 - l);          // value = digits f..l 10^e10
    const int64_t n19 = ns < 19 ? ns : 19, q = e10 + (ns - n19);
    uint64_t w = 0;
    for (int64_t k = f; k < f + n19; k++) w = w * 10 + (uint64_t)cf_digit_at(t, m, k);
    if (q > DT_POW5_Q_MAX) { *finite = false; return sign | kCfInf; }   // >= 10^309
    if (q < DT_POW5_Q_MIN) return sign;                                   // < 10^-323, below half the least subnormal
    const uint64_t lo = cf_round(w, (int)q, false), hi = cf_round(ns > 19 ? w + 1 : w, (int)q, true);
    uint64_t b = lo;
    if (lo != hi) {
        if (kExact) b = cf_decide(t, m, f, ns, e10, lo);
        else *open = true;
    }
    if (b >= kCfInf && (kExact || lo == hi)) *finite = false;
    return sign | b;
}

// ------------------------------------------------------------------------------------------------ record pass
// any JSON value at p -> the position after it; -1: syntax error, -2: nested deeper than kCfMaxDepth
__device__ __forceinline__ int64_t cf_skip_value(const CfText& x, int64_t p) {
    uint64_t stack = 0;                               // bit d: the container at depth d + 1 is an object
    int depth = 0;
    for (;;) {
        const int c = x.at(p);
        bool closed = false;
        if (c == '{' || c == '[') {
            if (depth == kCfMaxDepth) return -2;
            const bool obj = c == '{';
            stack = obj ? stack | (1ull << depth) : stack & ~(1ull << depth);
            depth++;
            p = cf_skip_ws(x, p + 1);
            if (x.at(p) == (obj ? '}' : ']')) {
                p++;
                depth--;
                closed = true;
            } else {
                if (obj) {
                    int64_t kb, ke;
                    p = cf_key(x, p, &kb, &ke);
                    if (p < 0) return -1;
                }
                continue;
            }
        }
        if (!closed) {
            if (c == '"') {
                int64_t u;
                p = cf_string(x, p, &u);
            } else if (c == '-' || cf_digit(c)) {
                CfNumber m;
                p = cf_number(x, p, m);
            } else if (c == 't' && x.at(p + 1) == 'r' && x.at(p + 2) == 'u' && x.at(p + 3) == 'e') {
                p += 4;
            } else if (c == 'f' && x.at(p + 1) == 'a' && x.at(p + 2) == 'l' && x.at(p + 3) == 's' && x.at(p + 4) == 'e') {
                p += 5;
            } else if (c == 'n' && x.at(p + 1) == 'u' && x.at(p + 2) == 'l' && x.at(p + 3) == 'l') {
                p += 4;
            } else {
                return -1;
            }
            if (p < 0) return -1;
        }
        // after a value: close containers or move to the next element
        for (;;) {
            if (depth == 0) return p;
            p = cf_skip_ws(x, p);
            const int d = x.at(p);
            const bool obj = (stack >> (depth - 1)) & 1;
            if (d == ',') {
                p = cf_skip_ws(x, p + 1);
                if (obj) {
                    int64_t kb, ke;
                    p = cf_key(x, p, &kb, &ke);
                    if (p < 0) return -1;
                }
                break;
            }
            if (d != (obj ? '}' : ']')) return -1;
            p++;
            depth--;
        }
    }
}

// an array of numbers at p ('[') -> the position after it (< 0 as cf_skip_value); *n elements, *ok all numbers (and integer literals
// in int64 when ints), the first `keep` converted into out (doubles) or iout (ints)
template <bool kInts>
__device__ __forceinline__ int64_t cf_number_array(const CfText& x, int64_t p, int keep, double* out, int64_t* iout, int* n, bool* ok, bool* nonfinite,
                                   int64_t* open_at) {
    *n = 0; *ok = true;
    p = cf_skip_ws(x, p + 1);
    if (x.at(p) == ']') return p + 1;
    for (;;) {
        const int c = x.at(p);
        if (c == '-' || cf_digit(c)) {
            CfNumber m;
            p = cf_number(x, p, m);
            if (p < 0) return -1;
            if (kInts) {
                int64_t v = 0;
                if (!cf_int64(x.t, m, &v)) *ok = false;
                if (*n < keep) iout[*n] = v;
            } else {
                bool fin, open = false;
                const uint64_t b = cf_to_double<false>(x.t, m, &fin, &open);
                if (!fin) *nonfinite = true;
                if (*n < keep) {
                    out[*n] = __longlong_as_double((long long)b);
                    open_at[*n] = open ? m.int_beg - m.neg : -1;
                }
            }
        } else {
            *ok = false;
            p = cf_skip_value(x, p);
            if (p < 0) return p;
        }
        (*n)++;
        p = cf_skip_ws(x, p);
        if (x.at(p) == ',') { p = cf_skip_ws(x, p + 1); continue; }
        if (x.at(p) == ']') return p + 1;
        return -1;
    }
}

struct CfRecord {
    int img_state, cat_state, score_state, seg_state;    // 0 missing, 1 valid, 2 not valid (seg_state 2: a dict that is not an RLE)
    int64_t img, cat, cb, ce, cn, h, w;
    double score, box[4];
    int64_t open_at[5];       // where the score / bbox numbers the bounds left open start (-1: decided)
    uint8_t flags;
    bool nonfinite;
};

// a segmentation dict at p ('{') -> the position after it; sets the record's RLE fields when it is a compressed RLE
__device__ __forceinline__ int64_t cf_segmentation(const CfText& x, int64_t p, CfRecord& R) {
    int cs = 0, ss = 0;
    int64_t b0 = 0, e0 = 0, n0 = 0, hw[2] = {0, 0};
    p = cf_skip_ws(x, p + 1);
    if (x.at(p) == '}') {
        p++;
    } else {
        for (;;) {
            int64_t kb, ke;
            p = cf_key(x, p, &kb, &ke);
            if (p < 0) return -1;
            const int c = x.at(p);
            if (cf_key_is(x.t, kb, ke, "counts")) {
                if (c == '"') { cs = 1; b0 = p + 1; p = cf_string(x, p, &n0); e0 = p - 1; }
                else { cs = 2; p = cf_skip_value(x, p); }
            } else if (cf_key_is(x.t, kb, ke, "size")) {
                ss = 2;
                if (c == '[') {
                    int n; bool ok, nf = false;
                    p = cf_number_array<true>(x, p, 2, nullptr, hw, &n, &ok, &nf, nullptr);
                    if (p >= 0 && ok && n == 2 && hw[0] >= 1 && hw[1] >= 1 && hw[0] < (1ll << 32) && hw[1] < (1ll << 32) &&
                        (uint64_t)hw[0] * (uint64_t)hw[1] < (1ull << 32))
                        ss = 1;
                } else {
                    p = cf_skip_value(x, p);
                }
            } else {
                p = cf_skip_value(x, p);
            }
            if (p < 0) return p;
            p = cf_skip_ws(x, p);
            if (x.at(p) == ',') { p = cf_skip_ws(x, p + 1); continue; }
            if (x.at(p) == '}') { p++; break; }
            return -1;
        }
    }
    if (cs == 1 && ss == 1) {
        R.seg_state = 1; R.cb = b0; R.ce = e0; R.cn = n0; R.h = hw[0]; R.w = hw[1];
    } else {
        R.seg_state = 2;
    }
    return p;
}

// one record's element text [p, x.end) -> error bits (0: a valid object, fields in R)
__device__ __forceinline__ unsigned cf_parse_record(const CfText& x, int64_t p, CfRecord& R) {
    p = cf_skip_ws(x, p);
    if (x.at(p) != '{') return x.at(p) == 0 ? kCfSyntax : kCfNotObject;
    p = cf_skip_ws(x, p + 1);
    if (x.at(p) == '}') {
        p++;
    } else {
        for (;;) {
            int64_t kb, ke;
            p = cf_key(x, p, &kb, &ke);
            if (p < 0) return kCfSyntax;
            const int c = x.at(p);
            const bool num = c == '-' || cf_digit(c);
            const bool is_img = cf_key_is(x.t, kb, ke, "image_id"), is_cat = !is_img && cf_key_is(x.t, kb, ke, "category_id");
            if (is_img || is_cat) {
                int st = 2;
                int64_t v = 0;
                if (num) {
                    CfNumber m;
                    p = cf_number(x, p, m);
                    if (p >= 0 && cf_int64(x.t, m, &v)) st = 1;
                } else {
                    p = cf_skip_value(x, p);
                }
                if (is_img) { R.img_state = st; R.img = v; } else { R.cat_state = st; R.cat = v; }
            } else if (cf_key_is(x.t, kb, ke, "score")) {
                R.score_state = 2;
                if (num) {
                    CfNumber m;
                    p = cf_number(x, p, m);
                    if (p >= 0) {
                        bool fin, open = false;
                        R.score = __longlong_as_double((long long)cf_to_double<false>(x.t, m, &fin, &open));
                        R.open_at[0] = open ? m.int_beg - m.neg : -1;
                        R.nonfinite |= !fin;
                        R.score_state = 1;
                    }
                } else {
                    p = cf_skip_value(x, p);
                }
            } else if (cf_key_is(x.t, kb, ke, "bbox")) {
                R.flags = (uint8_t)((R.flags & ~(kCfBboxOk | kCfBboxEmpty)) | kCfHasBbox);
                if (c == '[') {
                    int n; bool ok;
                    for (int j = 1; j < 5; j++) R.open_at[j] = -1;
                    p = cf_number_array<false>(x, p, 4, R.box, nullptr, &n, &ok, &R.nonfinite, R.open_at + 1);
                    if (n == 0) R.flags |= kCfBboxEmpty;
                    if (ok && n == 4) R.flags |= kCfBboxOk;
                } else {
                    p = cf_skip_value(x, p);
                }
            } else if (cf_key_is(x.t, kb, ke, "segmentation")) {
                R.seg_state = 0;
                p = c == '{' ? cf_segmentation(x, p, R) : cf_skip_value(x, p);
            } else {
                if (cf_key_is(x.t, kb, ke, "caption")) R.flags |= kCfHasCaption;
                p = cf_skip_value(x, p);
            }
            if (p < 0) return p == -2 ? kCfDepth : kCfSyntax;
            p = cf_skip_ws(x, p);
            if (x.at(p) == ',') { p = cf_skip_ws(x, p + 1); continue; }
            if (x.at(p) == '}') { p++; break; }
            return kCfSyntax;
        }
    }
    if (cf_skip_ws(x, p) != x.end) return kCfSyntax;
    unsigned err = 0;
    if (R.img_state != 1) err |= kCfImageId;
    if (R.cat_state != 1) err |= kCfCategoryId;
    if (R.score_state != 1) err |= kCfScore;
    if (R.seg_state == 2) err |= kCfRle;
    if (R.nonfinite) err |= kCfNonFinite;
    return err;
}

struct CfArgs {
    int64_t R;
    const uint8_t* text;
    const int64_t* sep;
    int num_images, num_cats;
    const int64_t* img_ids;       // sorted json ids
    const int64_t* cat_ids;       // sorted json ids
    double* rec_f;                // [R, kCfRecF]
    int64_t* rec_open;            // [R, kCfRecF] text position of a number left open by the bounds, -1 if none
    int64_t* rec_i;               // [R, kCfRecI]
    int64_t* rec_n;               // [R] decoded counts length (0 without an RLE)
    uint8_t* rec_b;               // [R] flags
    unsigned long long* info;
};

__global__ void __launch_bounds__(128, 4) cf_record_kernel(CfArgs a) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.R) return;
    const CfText x{a.text, a.sep[r + 1]};
    const int64_t p = a.sep[r] + 1;
    CfRecord R;
    R.img_state = R.cat_state = R.score_state = R.seg_state = 0;
    R.img = R.cat = R.cb = R.ce = R.cn = R.h = R.w = 0;
    R.score = R.box[0] = R.box[1] = R.box[2] = R.box[3] = 0;
    R.flags = 0;
    R.nonfinite = false;
    for (int j = 0; j < kCfRecF; j++) R.open_at[j] = -1;
    const bool empty = a.R == 1 && cf_skip_ws(x, p) == x.end;     // "[]": no records
    if (empty) a.info[kCfInfoEmpty] = 1;
    unsigned err = empty ? 0u : cf_parse_record(x, p, R);
    int64_t i = -1, k = -1;
    if (!err && !empty) {
        i = coco_lower_bound(a.img_ids, a.num_images, R.img, false);
        if (i == a.num_images || a.img_ids[i] != R.img) err |= kCfImageUnknown;
        k = coco_lower_bound(a.cat_ids, a.num_cats, R.cat, false);
        if (k == a.num_cats || a.cat_ids[k] != R.cat) k = -1;
    }
    if (err) cf_fail(a.info, err, r);
    if (R.seg_state == 1) R.flags |= kCfHasRle;
    else R.h = R.w = R.cn = 0;
    unsigned sum = 0;
    if (!(R.flags & kCfBboxOk)) sum |= kCfNoBbox;
    if ((R.flags & kCfHasBbox) && !(R.flags & kCfBboxOk)) sum |= kCfBadBbox;
    if (!(R.flags & kCfHasRle)) sum |= kCfNoRle;
    cf_or(a.info + kCfInfoSum, sum);
    cf_add(a.info + kCfInfoDropped, k < 0 && !err && !empty);
    double* F = a.rec_f + r * kCfRecF;
    F[0] = R.score; F[1] = R.box[0]; F[2] = R.box[1]; F[3] = R.box[2]; F[4] = R.box[3];
    int64_t* I = a.rec_i + r * kCfRecI;
    I[0] = i; I[1] = k; I[2] = R.cb; I[3] = R.ce; I[4] = R.h; I[5] = R.w;
    a.rec_n[r] = R.cn;
    a.rec_b[r] = R.flags;
    for (int j = 0; j < kCfRecF; j++) a.rec_open[r * kCfRecF + j] = R.open_at[j];
}

// the numbers cf_record_kernel's bounds left open, decided exactly (big-integer comparisons with the halfway points): one thread per
// (record, score / bbox entry), nearly all of which return at once
__global__ void cf_exact_kernel(int64_t n, const uint8_t* __restrict__ text, int64_t text_len, const int64_t* __restrict__ rec_open,
                                double* __restrict__ rec_f, unsigned long long* __restrict__ info) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n || rec_open[e] < 0) return;
    const CfText x{text, text_len};
    CfNumber m;
    cf_number(x, rec_open[e], m);
    bool fin;
    const uint64_t b = cf_to_double<true>(text, m, &fin, nullptr);
    rec_f[e] = __longlong_as_double((long long)b);
    if (!fin) cf_fail(info, kCfNonFinite, e / kCfRecF);
}

// each record's counts decoded at offs[r] - rec_n[r] (offs: the inclusive scan of rec_n) and checked as list input's strings are
// (utils.coco_eval._check_strings); det_i [R, 4]: char offset, count, h, w (0, 0 without an RLE) in file order
__global__ void cf_counts_kernel(int64_t R, const uint8_t* __restrict__ text, const int64_t* __restrict__ rec_i, const int64_t* __restrict__ rec_n,
                                 const int64_t* __restrict__ offs, char* __restrict__ chars, int64_t* __restrict__ det_i,
                                 unsigned long long* __restrict__ info) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const int64_t n = rec_n[r], o = offs[r] - n;
    const int64_t* I = rec_i + r * kCfRecI;
    int64_t* D = det_i + r * kCocoDetI;
    D[0] = o; D[1] = n; D[2] = I[4]; D[3] = I[5];
    int64_t p = I[2];
    int run = 0, v = 0;
    bool bad = false;
    for (int64_t j = 0; j < n; j++) {
        const int c = cf_unescape(text, p);
        bad |= c < 48 || c > 111;
        chars[o + j] = (char)(c < 0x80 ? c : 0xff);
        v = c - 48;
        if (v & 0x20) bad |= ++run > 5;
        else run = 0;
    }
    bad |= n > 0 && (v & 0x20);
    if (bad) cf_fail(info, kCfCounts, r);
}

// loadRes's area and box of each record (file order) and its sort key; bad: coco_det_check_kernel's run-sum flags
__global__ void cf_columns_kernel(int64_t R, int segm, int num_images, int num_cats, double* __restrict__ rec_f, const int64_t* __restrict__ rec_i,
                                  const uint8_t* __restrict__ rec_b, const uint8_t* __restrict__ bad, const double* __restrict__ rle_area,
                                  const double* __restrict__ rle_box, double* __restrict__ area, int64_t* __restrict__ keys,
                                  int64_t* __restrict__ vals, unsigned long long* __restrict__ info) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    if (bad[r]) cf_fail(info, kCfSums, r);
    double* F = rec_f + r * kCfRecF;
    if (segm) {
        area[r] = rle_area[r];
        if (!(rec_b[r] & kCfHasBbox))
            for (int j = 0; j < 4; j++) F[1 + j] = rle_box[4 * r + j];
    } else {
        area[r] = __dmul_rn(F[3], F[4]);
    }
    const int64_t k = rec_i[r * kCfRecI + 1];
    keys[r] = k >= 0 ? k * num_images + rec_i[r * kCfRecI] : (int64_t)num_cats * num_images;
    vals[r] = r;
}

__global__ void cf_gather_kernel(int64_t N, const int64_t* __restrict__ order, const double* __restrict__ rec_f, const int64_t* __restrict__ det_i_file,
                                 const double* __restrict__ area, double* __restrict__ det_f, int64_t* __restrict__ det_i, double* __restrict__ det_area,
                                 int64_t* __restrict__ det_id) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    const int64_t r = order[p];
    for (int j = 0; j < kCocoDetF; j++) det_f[p * kCocoDetF + j] = rec_f[r * kCfRecF + j];
    for (int j = 0; j < kCocoDetI; j++) det_i[p * kCocoDetI + j] = det_i_file[r * kCocoDetI + j];
    det_area[p] = area[r];
    det_id[p] = r + 1;
}

// ------------------------------------------------------------------------------------------------ launchers
inline size_t cf_take(size_t& o, size_t bytes) {
    const size_t at = o;
    o += (bytes + 255) / 256 * 256;
    return at;
}

struct CfStructWs { size_t q, s, sep, delta, depth, nsel, temp, temp_bytes, total; };
inline CfStructWs cf_struct_ws(int64_t n) {
    CfStructWs w;
    size_t o = 0, a = 0, b = 0, c = 0;
    w.q = cf_take(o, n); w.s = cf_take(o, n); w.sep = cf_take(o, n);
    w.delta = cf_take(o, 4 * (size_t)n); w.depth = cf_take(o, 4 * (size_t)n); w.nsel = cf_take(o, 8);
    cub::DeviceScan::InclusiveScan(nullptr, a, (const uint8_t*)nullptr, (uint8_t*)nullptr, CfXor(), n);
    cub::DeviceScan::InclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, n);
    cub::DeviceSelect::Flagged(nullptr, c, thrust::counting_iterator<int64_t>(0), (const uint8_t*)nullptr, (int64_t*)nullptr, (int64_t*)nullptr, n);
    w.temp_bytes = a > b ? (a > c ? a : c) : (b > c ? b : c);
    w.temp = cf_take(o, w.temp_bytes);
    w.total = o;
    return w;
}

inline unsigned cf_blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

inline cudaError_t cf_struct_launch(int64_t n, const uint8_t* text, uint8_t* ws, unsigned long long* info, cudaStream_t st) {
    const CfStructWs W = cf_struct_ws(n);
    uint8_t *q = ws + W.q, *s = ws + W.s, *sep = ws + W.sep;
    int *delta = reinterpret_cast<int*>(ws + W.delta), *depth = reinterpret_cast<int*>(ws + W.depth);
    cf_quote_kernel<<<cf_blocks(n, 256), 256, 0, st>>>(n, text, q);
    size_t tb = W.temp_bytes;
    cudaError_t e = cub::DeviceScan::InclusiveScan(ws + W.temp, tb, q, s, CfXor(), n, st);
    if (e != cudaSuccess) return e;
    cf_delta_kernel<<<cf_blocks(n, 256), 256, 0, st>>>(n, text, q, s, delta);
    tb = W.temp_bytes;
    e = cub::DeviceScan::InclusiveSum(ws + W.temp, tb, delta, depth, n, st);
    if (e != cudaSuccess) return e;
    cf_classify_kernel<<<cf_blocks(n, 256), 256, 0, st>>>(n, text, q, s, depth, sep, info);
    return cudaGetLastError();
}

inline cudaError_t cf_separators_launch(int64_t n, uint8_t* ws, int64_t* sep_pos, cudaStream_t st) {
    const CfStructWs W = cf_struct_ws(n);
    size_t tb = W.temp_bytes;
    return cub::DeviceSelect::Flagged(ws + W.temp, tb, thrust::counting_iterator<int64_t>(0), ws + W.sep, sep_pos,
                                      reinterpret_cast<int64_t*>(ws + W.nsel), n, st);
}

inline cudaError_t cf_records_launch(const CfArgs& a, int64_t text_len, cudaStream_t st) {
    cf_record_kernel<<<cf_blocks(a.R, 128), 128, 0, st>>>(a);
    cf_exact_kernel<<<cf_blocks(a.R * kCfRecF, 256), 256, 0, st>>>(a.R * kCfRecF, a.text, text_len, a.rec_open, a.rec_f, a.info);
    return cudaGetLastError();
}

struct CfFinishWs { size_t det_i_file, bad, area, keys, keys_out, vals, vals_out, cnts, det_m, rle_area, rle_box, temp, temp_bytes, total; };
inline CfFinishWs cf_finish_ws(int64_t R, int64_t num_chars, int segm) {
    CfFinishWs w;
    size_t o = 0, t = 0;
    w.det_i_file = cf_take(o, 8 * kCocoDetI * (size_t)R); w.bad = cf_take(o, R); w.area = cf_take(o, 8 * (size_t)R);
    w.keys = cf_take(o, 8 * (size_t)R); w.keys_out = cf_take(o, 8 * (size_t)R); w.vals = cf_take(o, 8 * (size_t)R); w.vals_out = cf_take(o, 8 * (size_t)R);
    w.cnts = cf_take(o, segm ? 4 * (size_t)num_chars : 0); w.det_m = cf_take(o, segm ? 8 * (size_t)R : 0);
    w.rle_area = cf_take(o, segm ? 8 * (size_t)R : 0); w.rle_box = cf_take(o, segm ? 32 * (size_t)R : 0);
    cub::DeviceRadixSort::SortPairs(nullptr, t, (const int64_t*)nullptr, (int64_t*)nullptr, (const int64_t*)nullptr, (int64_t*)nullptr, R);
    w.temp_bytes = t;
    w.temp = cf_take(o, t);
    w.total = o;
    return w;
}

// counts decoded and checked, run sums checked, loadRes's area and box, the stable sort by key and the gather of the first N (the
// records of known categories).  chars holds num_chars + 1 bytes: a last '0' ends any value a bad string leaves open, so the checks
// and the decoder never read past the buffer.
inline cudaError_t cf_finish_launch(int64_t R, int segm, const uint8_t* text, const int64_t* rec_i, const int64_t* rec_n, const int64_t* offs,
                                    const uint8_t* rec_b, double* rec_f, int num_images, int num_cats, int64_t num_chars, char* chars,
                                    uint8_t* ws, int64_t N, int64_t* det_key, double* det_f, int64_t* det_i, double* det_area, int64_t* det_id,
                                    unsigned long long* info, cudaStream_t st) {
    const CfFinishWs W = cf_finish_ws(R, num_chars, segm);
    int64_t* det_i_file = reinterpret_cast<int64_t*>(ws + W.det_i_file);
    uint8_t* bad = ws + W.bad;
    double* area = reinterpret_cast<double*>(ws + W.area);
    int64_t *keys = reinterpret_cast<int64_t*>(ws + W.keys), *vals = reinterpret_cast<int64_t*>(ws + W.vals);
    int64_t *vals_out = reinterpret_cast<int64_t*>(ws + W.vals_out);
    double *rle_area = reinterpret_cast<double*>(ws + W.rle_area), *rle_box = reinterpret_cast<double*>(ws + W.rle_box);
    cudaMemsetAsync(chars + num_chars, '0', 1, st);
    cf_counts_kernel<<<cf_blocks(R, 128), 128, 0, st>>>(R, text, rec_i, rec_n, offs, chars, det_i_file, info);
    coco_det_check_kernel<<<cf_blocks(R, 128), 128, 0, st>>>(R, det_i_file, chars, bad);
    if (segm)
        coco_det_rle_kernel<<<cf_blocks(R, 128), 128, 0, st>>>(R, det_i_file, chars, reinterpret_cast<uint32_t*>(ws + W.cnts),
                                                             reinterpret_cast<int64_t*>(ws + W.det_m), rle_area, rle_box);
    cf_columns_kernel<<<cf_blocks(R, 256), 256, 0, st>>>(R, segm, num_images, num_cats, rec_f, rec_i, rec_b, bad, rle_area, rle_box, area, keys,
                                                         vals, info);
    const uint64_t top = (uint64_t)num_cats * (uint64_t)num_images;
    const int end_bit = top ? 64 - __builtin_clzll(top) : 1;
    size_t tb = W.temp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(ws + W.temp, tb, keys, det_key, vals, vals_out, R, 0, end_bit, st);
    if (e != cudaSuccess) return e;
    if (N > 0) cf_gather_kernel<<<cf_blocks(N, 256), 256, 0, st>>>(N, vals_out, rec_f, det_i_file, area, det_f, det_i, det_area, det_id);
    return cudaGetLastError();
}

}  // namespace dt

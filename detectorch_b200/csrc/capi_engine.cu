// detectorch_b200 -- the fused Mask R-CNN (ResNet-50/101 + FPN) inference engine.
//
// One C++ object owns the whole hot path of reference lib/model/detector.py:233-286 (detector.forward),
// lib/utils/result_utils.py:76-168 (postprocess_output) and lib/model/detector.py:99-112 (mask_head.forward):
// a static program of kernel launches over pre-built TMA descriptors, with zero host synchronisation
// (the reference syncs >= 17 times per image, SURVEY.md 3.1).  Memory is supplied by the caller as two
// flat device buffers (weights, workspace) so that the host language (PyTorch here) stays pure plumbing.
#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/detectorch_b200.h"
#include <cuda_fp16.h>

#include "conv_host.cuh"
#include "detect_ops.cuh"
#include "roi_align.cuh"

using namespace dt;

namespace {

constexpr float kBnEps = 1e-5f;
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------- weight packing kernels
// torch conv weight [Cout, Cin, kh, kw] -> K-major [Cout][kh][kw][Cin] at dst row stride K
__global__ void pack_conv_w_kernel(const float* __restrict__ src, int Cout, int Cin, int kh, int kw, float* __restrict__ dst) {
    const long long total = (long long)Cout * Cin * kh * kw;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        long long t = i;
        const int c = (int)(t % Cin); t /= Cin;
        const int x = (int)(t % kw); t /= kw;
        const int y = (int)(t % kh);
        const int o = (int)(t / kh);
        dst[i] = src[(((size_t)o * Cin + c) * kh + y) * kw + x];
    }
}
// rows [Cout][Kin] -> [Cout][Kout] zero padded (stem 147 -> 160, plain copies)
__global__ void pack_rows_kernel(const float* __restrict__ src, int rows, int Kin, int Kout, float* __restrict__ dst) {
    const long long total = (long long)rows * Kout;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % Kout);
        const int r = (int)(i / Kout);
        dst[i] = k < Kin ? src[(size_t)r * Kin + k] : 0.f;
    }
}
// stem [64][3][7][7] -> [64][7 (ky)][32 (kx*4 + c; kx < 7, c < 3; rest 0)]  (fused-window stem, conv_build_stem)
__global__ void pack_stem_window_kernel(const float* __restrict__ src, float* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 64 * 224) return;
    const int j = i % 32, ky = (i / 32) % 7, o = i / 224;
    const int kx = j >> 2, c = j & 3;
    dst[i] = (kx < 7 && c < 3) ? src[((o * 3 + c) * 7 + ky) * 7 + kx] : 0.f;
}
// fc6 [O][C*P] (k = c*P + p) -> [O][P*C] (k = p*C + c)
__global__ void pack_fc6_kernel(const float* __restrict__ src, int O, int C, int P, float* __restrict__ dst) {
    const long long total = (long long)O * C * P;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int p = (int)((i / C) % P);
        const int o = (int)(i / ((long long)C * P));
        dst[i] = src[((size_t)o * C + c) * P + p];
    }
}
// ConvTranspose2d weight [Cin][Cout][2][2] -> 4 K-major matrices [(i*2+j)][Cout][Cin]
__global__ void pack_deconv_kernel(const float* __restrict__ src, int Cin, int Cout, float* __restrict__ dst) {
    const long long total = 4ll * Cin * Cout;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % Cin);
        const int co = (int)((i / Cin) % Cout);
        const int ij = (int)(i / ((long long)Cin * Cout));
        dst[i] = src[((size_t)ci * Cout + co) * 4 + ij];
    }
}
__global__ void bn_scale_kernel(const float* __restrict__ gamma, int n, float* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = gamma[i] / sqrtf(1.f + kBnEps);     // running_var = 1 (detector.py:301)
}
__global__ void copy_kernel(const float* __restrict__ src, long long n, float* __restrict__ dst) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
}
__global__ void fill_kernel(float* __restrict__ dst, long long n, float v) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = v;
}
__global__ void tf32_lo_kernel(const float* __restrict__ w, float* __restrict__ lo, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = w[i];
        lo[i] = v - __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    }
}
// ---- fp16 hi/lo weight halves for the kind::f16 convs (per-matrix power-of-two pre-scale) ----------
struct MatInfo { unsigned int maxbits; float mult; };
__global__ void absmax_kernel(const float* __restrict__ w, long long n, MatInfo* __restrict__ info) {
    unsigned int m = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = max(m, __float_as_uint(w[i]) & 0x7fffffffu);        // non-negative floats order like their bit patterns
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&info->maxbits, m);
}
// multiplier = the power of two that brings max|w| into [2^13, 2^14): the fp16 low half of every weight within 2^-9 of the largest
// one is then a normal number; 1 for an all-zero (or non-finite) matrix
__global__ void matmult_kernel(MatInfo* __restrict__ info, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int e = (int)((info[i].maxbits >> 23) & 255u) - 127;
    int pe = 127 + 13 - e;
    if (info[i].maxbits == 0 || e == 128) pe = 127;
    pe = pe < 1 ? 1 : (pe > 254 ? 254 : pe);
    info[i].mult = __uint_as_float((unsigned int)pe << 23);
}
__global__ void fp16_split_dev_kernel(const float* __restrict__ w, long long n, const MatInfo* __restrict__ info, __half* __restrict__ hi,
                                      __half* __restrict__ lo) {
    const float mult = info->mult;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = w[i] * mult;
        const __half h = __float2half_rn(v);
        hi[i] = h;
        lo[i] = __float2half_rn(v - __half2float(h));
    }
}
__global__ void scale16_kernel(const float* __restrict__ scale, const MatInfo* __restrict__ info, float* __restrict__ dst, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = scale[i] / info->mult;      // division by a power of two: exact
}
inline int grid_for(long long n, int threads = 256) {
    long long g = (n + threads - 1) / threads;
    return (int)(g < 1 ? 1 : (g > num_sms() * 16 ? num_sms() * 16 : g));
}

// ---------------------------------------------------------------------------------- engine
enum ParamKind { PK_CONV_W, PK_STEM_W, PK_FC6_W, PK_ROWS_W, PK_DECONV_W, PK_BN_SCALE, PK_VEC };

struct ParamSlot {
    ParamKind kind;
    size_t off;          // float offset into the weight buffer (hi region for matrices, vector region otherwise)
    int d0, d1, d2, d3;  // kind-specific dims
    int row_off;         // PK_ROWS_W / PK_VEC: destination row / element offset (fused heads)
    int Kout;
    bool loaded = false;
};

struct Buf {
    size_t off = 0;      // byte offset in workspace
    size_t bytes = 0;
    int dims[5] = {0, 0, 0, 0, 0};
    int nd = 0;
    int dtype = 0;       // 0 = float32, 1 = int32
};

struct Op {
    double flops = 0.0;   // algorithmic FLOPs (2*MAC) of this launch, 0 for non-GEMM ops
    int stage;
    int kind;            // 0 conv, 1 custom lambda index
    ConvLayer conv;
    int fn;              // index into engine fns for kind==1
    // kind::f16 convs: scale16 = scale / multiplier(matrix) is (re)derived at finalize time
    const float* scale_src = nullptr;
    float* scale16 = nullptr;
    int scale_n = 0;
    int matrix = -1;
};

struct Engine;
typedef cudaError_t (*StageFn)(Engine*, cudaStream_t);

struct Engine {
    dt_engine_config cfg;
    // weights
    std::map<std::string, ParamSlot> params;
    size_t mat_floats = 0;      // hi-region floats (lo region has the same size)
    size_t vec_floats = 0;
    float* wbase = nullptr;
    // workspace
    std::map<std::string, Buf> bufs;
    size_t ws_bytes = 0;
    uint8_t* ws = nullptr;
    bool bound = false;
    // program
    std::vector<Op> ops;
    std::vector<std::string> errors;
    const float* image = nullptr;
    float scaling_factor = 1.f;
    float orig_h = 0.f, orig_w = 0.f;   // original image size for the final clip (0 = network size / scaling_factor)
    // static geometry
    int H1, W1, H2, W2;                 // stem out, pool out
    int Hp, Wp;                         // padded NHWC4 stem input
    bool stem_fused = true;
    int LH[5], LW[5];                   // P2..P6
    RpnParams rpn;
    CollectParams col;
    DetParams det;
    RoiLevels roi_lv;
    int num_stage_fns = 0;
    std::vector<StageFn> fns;

    // weight buffer: [fp32 matrices][tf32 residuals][vectors][fp16 hi halves][fp16 lo halves][scale16 arena][matrix info]
    static constexpr size_t kScale16Floats = 768 * 1024;
    static constexpr size_t kMaxMatrices = 1024;
    std::vector<std::pair<size_t, size_t>> matrices;   // (offset, floats) of every weight matrix, ascending
    size_t scale16_used = 0;
    float* wmat(size_t off) const { return wbase + off; }
    float* wlo(size_t off) const { return wbase + mat_floats + off; }
    float* wvec(size_t off) const { return wbase + 2 * mat_floats + off; }
    __half* whi16(size_t off) const { return reinterpret_cast<__half*>(wbase + 2 * mat_floats + vec_floats) + off; }
    __half* wlo16(size_t off) const { return whi16(0) + mat_floats + off; }
    float* scale16_arena() const { return wbase + 3 * mat_floats + vec_floats; }
    MatInfo* matinfo() const { return reinterpret_cast<MatInfo*>(scale16_arena() + kScale16Floats); }
    size_t weight_bytes() const { return (3 * mat_floats + vec_floats + kScale16Floats) * sizeof(float) + kMaxMatrices * sizeof(MatInfo); }
    int matrix_of(size_t off) const {
        int m = -1;
        for (size_t i = 0; i < matrices.size(); ++i)
            if (matrices[i].first <= off && off < matrices[i].first + matrices[i].second) m = (int)i;
        return m;
    }
    template <class T = float>
    T* buf(const std::string& n) {
        auto it = bufs.find(n);
        if (it == bufs.end()) { fprintf(stderr, "[detectorch_b200] engine: unknown buffer %s\n", n.c_str()); return nullptr; }
        return reinterpret_cast<T*>(ws + it->second.off);
    }
};

// ---- parameter table ---------------------------------------------------------------------------
size_t add_mat(Engine* e, const std::string& name, ParamKind kind, int rows_total, int K, int d0, int d1, int d2, int d3, int row_off = 0) {
    ParamSlot s;
    s.kind = kind; s.d0 = d0; s.d1 = d1; s.d2 = d2; s.d3 = d3; s.row_off = row_off; s.Kout = K;
    if (row_off == 0) {
        s.off = e->mat_floats;
        e->mat_floats += align_up((size_t)rows_total * K, 64);
        e->matrices.push_back(std::make_pair(s.off, e->mat_floats - s.off));
    }
    e->params[name] = s;
    return s.off;
}
size_t add_vec(Engine* e, const std::string& name, ParamKind kind, int n_total, int n, int elem_off = 0, size_t share_off = (size_t)-1) {
    ParamSlot s;
    s.kind = kind; s.d0 = n; s.d1 = s.d2 = s.d3 = 0; s.row_off = elem_off; s.Kout = 0;
    if (share_off != (size_t)-1) s.off = share_off;
    else { s.off = e->vec_floats; e->vec_floats += align_up((size_t)n_total, 64); }
    e->params[name] = s;
    return s.off;
}

struct ConvW { size_t w, scale, shift; int cout, cin, k; };

void build_param_table(Engine* e, std::map<std::string, ConvW>* cw) {
    const int NC = e->cfg.num_classes;
    // shared "ones" scale vector for bias-only convs (max Cout 2048)
    size_t ones = e->vec_floats; e->vec_floats += 2048;
    (*cw)["__ones"] = ConvW{0, ones, 0, 2048, 0, 0};
    size_t zeros = e->vec_floats; e->vec_floats += 2048;     // zero shift vector for the second half of a K-split convolution
    (*cw)["__zeros"] = ConvW{0, 0, zeros, 2048, 0, 0};
    // stem
    {
        ConvW c; c.cout = 64; c.cin = 160; c.k = 1;
        c.w = add_mat(e, "model.conv1.weight", PK_STEM_W, 64, 160 + 224, 64, 147, 160, 0);   // im2col layout [64][160], then window layout [64][224]
        c.scale = add_vec(e, "model.bn1.weight", PK_BN_SCALE, 64, 64);
        c.shift = add_vec(e, "model.bn1.bias", PK_VEC, 64, 64);
        (*cw)["stem"] = c;
    }
    int inpl = 64;
    for (int li = 1; li <= 4; ++li) {
        const int planes = 64 << (li - 1);
        for (int b = 0; b < e->cfg.arch_blocks[li - 1]; ++b) {
            const std::string p = "model.layer" + std::to_string(li) + "." + std::to_string(b) + ".";
            auto conv = [&](const std::string& cn, const std::string& bn, int cout, int cin, int k) {
                ConvW c; c.cout = cout; c.cin = cin; c.k = k;
                c.w = add_mat(e, p + cn + ".weight", PK_CONV_W, cout, cin * k * k, cout, cin, k, k);
                c.scale = add_vec(e, p + bn + ".weight", PK_BN_SCALE, cout, cout);
                c.shift = add_vec(e, p + bn + ".bias", PK_VEC, cout, cout);
                (*cw)[p + cn] = c;
            };
            conv("conv1", "bn1", planes, inpl, 1);
            conv("conv2", "bn2", planes, planes, 3);
            conv("conv3", "bn3", planes * 4, planes, 1);
            if (b == 0) conv("downsample.0", "downsample.1", planes * 4, inpl, 1);
            inpl = planes * 4;
        }
    }
    auto bias_conv = [&](const std::string& name, int cout, int cin, int k) {
        ConvW c; c.cout = cout; c.cin = cin; c.k = k;
        c.w = add_mat(e, name + ".weight", PK_CONV_W, cout, cin * k * k, cout, cin, k, k);
        c.scale = ones;
        c.shift = add_vec(e, name + ".bias", PK_VEC, cout, cout);
        (*cw)[name] = c;
    };
    const int cins[4] = {256, 512, 1024, 2048};
    for (int i = 0; i < 4; ++i) {
        bias_conv("conv_body.fpn_lateral." + std::to_string(i), 256, cins[i], 1);
        bias_conv("conv_body.fpn_output." + std::to_string(i), 256, 256, 3);
    }
    if (e->cfg.use_rpn) bias_conv("rpn.conv_rpn", 256, 256, 3);
    if (e->cfg.use_rpn) {   // fused RPN 1x1: rows [0,3) objectness, [3,15) deltas, row 15 zero
        ConvW c; c.cout = 16; c.cin = 256; c.k = 1;
        c.w = add_mat(e, "rpn.rpn_cls_prob.weight", PK_ROWS_W, 16, 256, 3, 256, 0, 0);
        e->params["rpn.rpn_cls_prob.weight"].row_off = 0;
        ParamSlot s = e->params["rpn.rpn_cls_prob.weight"];
        s.d0 = 12; s.row_off = 3;
        e->params["rpn.rpn_bbox_pred.weight"] = s;
        c.scale = ones;
        c.shift = add_vec(e, "rpn.rpn_cls_prob.bias", PK_VEC, 16, 3);
        add_vec(e, "rpn.rpn_bbox_pred.bias", PK_VEC, 0, 12, 3, c.shift);
        (*cw)["rpn.head"] = c;
    }
    {   // box head
        ConvW c; c.cout = 1024; c.cin = 256 * 49; c.k = 1;
        c.w = add_mat(e, "conv_head.fc6.weight", PK_FC6_W, 1024, 256 * 49, 1024, 256, 49, 0);
        c.scale = ones; c.shift = add_vec(e, "conv_head.fc6.bias", PK_VEC, 1024, 1024);
        (*cw)["fc6"] = c;
        ConvW d; d.cout = 1024; d.cin = 1024; d.k = 1;
        d.w = add_mat(e, "conv_head.fc7.weight", PK_ROWS_W, 1024, 1024, 1024, 1024, 0, 0);
        d.scale = ones; d.shift = add_vec(e, "conv_head.fc7.bias", PK_VEC, 1024, 1024);
        (*cw)["fc7"] = d;
        const int HN = (int)align_up((size_t)5 * NC, 4);
        ConvW h; h.cout = HN; h.cin = 1024; h.k = 1;
        h.w = add_mat(e, "classif_head.weight", PK_ROWS_W, HN, 1024, NC, 1024, 0, 0);
        ParamSlot s = e->params["classif_head.weight"];
        s.d0 = 4 * NC; s.row_off = NC;
        e->params["bbox_head.weight"] = s;
        h.scale = ones;
        h.shift = add_vec(e, "classif_head.bias", PK_VEC, HN, NC);
        add_vec(e, "bbox_head.bias", PK_VEC, 0, 4 * NC, NC, h.shift);
        (*cw)["head"] = h;
    }
    if (e->cfg.use_mask) {
        for (int i = 1; i <= 4; ++i) bias_conv("mask_head.conv_head.fcn" + std::to_string(i), 256, 256, 3);
        ConvW d; d.cout = 256; d.cin = 256; d.k = 1;
        d.w = add_mat(e, "mask_head.transposed_conv.weight", PK_DECONV_W, 4 * 256, 256, 256, 256, 0, 0);
        d.scale = ones; d.shift = add_vec(e, "mask_head.transposed_conv.bias", PK_VEC, 256, 256);
        (*cw)["deconv"] = d;
        const int MN = (int)align_up((size_t)NC, 4);
        ConvW m; m.cout = MN; m.cin = 256; m.k = 1;
        m.w = add_mat(e, "mask_head.classif_logits.weight", PK_ROWS_W, MN, 256, NC, 256, 0, 0);
        m.scale = ones; m.shift = add_vec(e, "mask_head.classif_logits.bias", PK_VEC, MN, NC);
        (*cw)["mask_logits"] = m;
    }
}

// ---- workspace ---------------------------------------------------------------------------------
void add_buf(Engine* e, const std::string& name, std::initializer_list<long long> dims, int dtype = 0, size_t elem = 4) {
    Buf b;
    size_t n = 1;
    b.nd = 0;
    for (long long d : dims) { b.dims[b.nd++] = (int)d; n *= (size_t)d; }
    b.bytes = n * elem;
    b.off = e->ws_bytes;
    b.dtype = dtype;
    e->ws_bytes += align_up(b.bytes, 1024);
    e->bufs[name] = b;
}

int conv_out(int x, int k, int s, int p) { return (x + 2 * p - k) / s + 1; }

void plan_buffers(Engine* e) {
    const dt_engine_config& c = e->cfg;
    const int B = c.batch;
    e->H1 = conv_out(c.height, 7, 2, 3); e->W1 = conv_out(c.width, 7, 2, 3);
    e->H2 = conv_out(e->H1, 3, 2, 1); e->W2 = conv_out(e->W1, 3, 2, 1);
    e->Hp = std::max(c.height + 6, 2 * e->H1 + 5); e->Wp = std::max(c.width + 6, 2 * e->W1 + 6);
    add_buf(e, "stem_x4", {B, e->Hp, e->Wp, 4});
    add_buf(e, "stem_col", {(long long)B * e->H1 * e->W1, 160});     // fallback path only (see build_program)
    add_buf(e, "c1", {B, e->H1, e->W1, 64});
    add_buf(e, "pool", {B, e->H2, e->W2, 64});
    int h = e->H2, w = e->W2;
    for (int li = 1; li <= 4; ++li) {
        const int planes = 64 << (li - 1);
        if (li > 1) { h = conv_out(h, 1, 2, 0); w = conv_out(w, 1, 2, 0); }
        e->LH[li - 1] = h; e->LW[li - 1] = w;
        for (int b = 0; b < c.arch_blocks[li - 1]; ++b) {
            const std::string p = "l" + std::to_string(li) + "b" + std::to_string(b);
            add_buf(e, p + ".t1", {B, h, w, planes});
            add_buf(e, p + ".t2", {B, h, w, planes});
            if (b == 0) add_buf(e, p + ".ds", {B, h, w, planes * 4});
            add_buf(e, p + ".out", {B, h, w, planes * 4});
        }
    }
    e->LH[4] = (e->LH[3] - 1) / 2 + 1; e->LW[4] = (e->LW[3] - 1) / 2 + 1;    // max_pool2d(k=1,s=2)
    for (int i = 0; i < 4; ++i) {
        add_buf(e, "inner" + std::to_string(i + 2), {B, e->LH[i], e->LW[i], 256});
        add_buf(e, "P" + std::to_string(i + 2), {B, e->LH[i], e->LW[i], 256});
    }
    add_buf(e, "P6", {B, e->LH[4], e->LW[4], 256});
    const int L = 5, pre = c.pre_nms_top_n, post = c.post_nms_top_n;
    if (c.use_rpn) {       // Fast R-CNN with the FPN body (eval_fast_FPN.ipynb) has no RPN: the caller fills `rois` / `roi_levels` / `roi_counts`
        long long anchors_total = 0;
        for (int i = 0; i < 5; ++i) {
            add_buf(e, "rpn_t" + std::to_string(i + 2), {B, e->LH[i], e->LW[i], 256});
            add_buf(e, "rpn_out" + std::to_string(i + 2), {B, e->LH[i], e->LW[i], 16});
            anchors_total += (long long)e->LH[i] * e->LW[i] * 3;
        }
        add_buf(e, "rpn_k0", {B, anchors_total}, 1); add_buf(e, "rpn_k1", {B, anchors_total}, 1);
        add_buf(e, "rpn_v0", {B, anchors_total}, 1); add_buf(e, "rpn_v1", {B, anchors_total}, 1);
        add_buf(e, "rpn_cand", {B, L, pre, 4}); add_buf(e, "rpn_cand_score", {B, L, pre});
        add_buf(e, "rpn_order", {B, L, pre}, 1);
        add_buf(e, "rpn_sel_hist", {B, L, 2, 2048}, 1); add_buf(e, "rpn_sel_cc", {B, L, kRpnMaxChunks}, 1); add_buf(e, "rpn_sel_info", {B, L, 4}, 1);
        add_buf(e, "rpn_cand_counts", {B, L}, 1); add_buf(e, "rpn_nms_mask", {B, L, pre, (pre + 63) / 64, 2}, 1);
        add_buf(e, "props", {B, L, post, 4}); add_buf(e, "prop_scores", {B, L, post}); add_buf(e, "prop_counts", {B, L}, 1);
        add_buf(e, "col_k0", {B, L * post}, 1); add_buf(e, "col_k1", {B, L * post}, 1);
        add_buf(e, "col_v0", {B, L * post}, 1); add_buf(e, "col_v1", {B, L * post}, 1);
    }
    add_buf(e, "rois", {B, post, 5}); add_buf(e, "roi_levels", {B, post}, 1); add_buf(e, "roi_counts", {B}, 1);
    add_buf(e, "roi_feat", {(long long)B * post, 7, 7, 256});
    add_buf(e, "fc6", {(long long)B * post, 1024}); add_buf(e, "fc7", {(long long)B * post, 1024});
    const int NC = c.num_classes, HN = (int)align_up((size_t)5 * NC, 4);
    add_buf(e, "head", {(long long)B * post, HN});
    add_buf(e, "cls_prob", {(long long)B * post, NC}); add_buf(e, "bbox_pred", {(long long)B * post, 4 * NC});
    // detection
    const int cap = c.det_cap;
    add_buf(e, "det_flag", {B, NC, post}, 2, 1);
    add_buf(e, "det_dec", {B, NC, post, 4}); add_buf(e, "det_cls_counts", {B, NC}, 1);
    add_buf(e, "det_k0", {B, (long long)NC * post}, 1); add_buf(e, "det_k1", {B, (long long)NC * post}, 1);
    add_buf(e, "det_v0", {B, (long long)NC * post}, 1); add_buf(e, "det_v1", {B, (long long)NC * post}, 1);
    add_buf(e, "det_boxes", {B, cap, 4}); add_buf(e, "det_scores", {B, cap}); add_buf(e, "det_classes", {B, cap}, 1);
    add_buf(e, "det_roi_idx", {B, cap}, 1); add_buf(e, "det_counts", {B}, 1);
    add_buf(e, "range_flag", {1}, 1);     // raised by a kind::f16 conv when an activation does not fit fp16
    if (c.use_mask) {
        const long long D = (long long)B * cap;
        add_buf(e, "mask_rois", {D, 5}); add_buf(e, "mask_levels", {D}, 1);
        add_buf(e, "mask_feat", {D, 14, 14, 256});
        for (int i = 1; i <= 4; ++i) add_buf(e, "mask_c" + std::to_string(i), {D, 14, 14, 256});
        add_buf(e, "mask_up", {D, 28, 28, 256});
        add_buf(e, "mask_logits", {D, 28, 28, (long long)align_up((size_t)NC, 4)});
        add_buf(e, "masks", {D, 28, 28});
        add_buf(e, "masks_full", {D, NC, 28, 28});
    }
}

// ---- program -----------------------------------------------------------------------------------
enum Stage { ST_TRUNK = 0, ST_FPN = 1, ST_RPN = 2, ST_PROPOSALS = 3, ST_COLLECT = 4, ST_ROI_BOX = 5, ST_BOX_HEAD = 6, ST_DETECT = 7,
             ST_MASK_ROIS = 8, ST_MASK_ROI_FEAT = 9, ST_MASK_HEAD = 10, ST_MASK_OUT = 11, ST_COUNT = 12 };

struct ProgBuilder {
    Engine* e;
    std::map<std::string, ConvW>* cw;
    bool ok = true;

    void conv(int stage, const std::string& wname, const float* x, int N, int H, int W, int xstride, float* y, int ystride, int kpad,
              int stride, bool relu, int res_mode = RES_NONE, const float* res = nullptr, const float* up = nullptr, int up_h = 0,
              int up_w = 0, int sigmoid_ch = 0, size_t w_extra_off = 0, int out_h = 0, int out_w = 0, int out_step = 0, int oy = 0,
              int ox = 0, int force_bn = 0, int tap0 = 0, int ntaps = 0, bool zero_shift = false, int planes_in = 0, int planes_out = 0) {
        const ConvW& c = (*cw)[wname];
        ConvSpec s;
        memset(&s, 0, sizeof(s));
        s.x = x; s.N = N; s.H = H; s.W = W; s.Cin = c.cin; s.x_pix_stride = xstride;
        Op op;
        s.Cout = c.cout; s.kh = c.k; s.kw = c.k; s.pad = kpad; s.stride = stride;
        s.shift = zero_shift ? e->wvec((*cw)["__zeros"].shift) : e->wvec(c.shift);
        s.tap0 = tap0; s.ntaps = ntaps;
        if (e->cfg.conv_kind == 0) {
            // kind::f16 three-term product: fp16 halves of w * multiplier(matrix); the multiplier is undone through a per-op scale vector
            const size_t n16 = align_up((size_t)c.cout, 64);
            op.matrix = e->matrix_of(c.w + w_extra_off);
            if (op.matrix < 0 || e->scale16_used + n16 > Engine::kScale16Floats) {
                ok = false;
                fprintf(stderr, "[detectorch_b200] engine: scale16 arena / matrix lookup failed for %s\n", wname.c_str());
                return;
            }
            op.scale_src = e->wvec(c.scale); op.scale16 = e->scale16_arena() + e->scale16_used; op.scale_n = c.cout;
            e->scale16_used += n16;
            s.kind = KIND_F16X3;
            s.w_hi = e->whi16(c.w + w_extra_off); s.w_lo = e->wlo16(c.w + w_extra_off);
            s.scale = op.scale16;
            s.range_flag = e->buf<int>("range_flag");
        } else {
            s.kind = KIND_TF32X3;
            s.w_hi = e->wmat(c.w + w_extra_off); s.w_lo = e->wlo(c.w + w_extra_off);
            s.scale = e->wvec(c.scale);
        }
        s.y = y; s.y_pix_stride = ystride;
        // fp16 hi/lo plane hand-over (kind::f16 only): the fp32 buffer of N*H*W*C floats holds the two fp16 planes back to back
        if (planes_in && e->cfg.conv_kind == 0) s.x_lo = reinterpret_cast<const __half*>(x) + (size_t)N * H * W * c.cin;
        if (planes_out && e->cfg.conv_kind == 0) {
            const int Ho_ = (H + 2 * kpad - c.k) / stride + 1, Wo_ = (W + 2 * kpad - c.k) / stride + 1;
            s.y_lo = reinterpret_cast<__half*>(y) + (size_t)N * Ho_ * Wo_ * c.cout;
        }
        s.out_h = out_h; s.out_w = out_w; s.out_step = out_step; s.out_y0 = oy; s.out_x0 = ox;
        s.residual = res; s.res_pix_stride = c.cout; s.up_src = up; s.up_h = up_h; s.up_w = up_w;
        s.res_mode = res_mode; s.relu = relu ? 1 : 0; s.sigmoid_ch = sigmoid_ch; s.passes = e->cfg.passes; s.force_block_n = force_bn; s.precise = (force_bn == 128) ? 1 : 0;
        op.stage = stage; op.kind = 0; op.fn = -1;
        {
            const int Ho = (H + 2 * kpad - c.k) / stride + 1, Wo = (W + 2 * kpad - c.k) / stride + 1;
            const double cin_alg = (wname == "stem") ? 147.0 : (double)c.cin;   // the stem K is zero-padded 147 -> 160
            const double cout_alg = (wname == "rpn.head") ? 15.0 : (wname == "head") ? 5.0 * e->cfg.num_classes : (wname == "mask_logits") ? (double)e->cfg.num_classes : (double)c.cout;
            op.flops = 2.0 * (double)N * Ho * Wo * cout_alg * cin_alg * (ntaps > 0 ? ntaps : c.k * c.k);
        }
        if (!conv_build(s, &op.conv)) { ok = false; fprintf(stderr, "[detectorch_b200] engine: conv_build failed for %s\n", wname.c_str()); }
        e->ops.push_back(op);
    }
    void fn(int stage, StageFn f) {
        Op op;
        op.stage = stage; op.kind = 1;
        op.fn = (int)e->fns.size();
        e->fns.push_back(f);
        e->ops.push_back(op);
    }
};

cudaError_t fn_stem_im2col(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->H1 * e->W1 * 40;
    stem_im2col_kernel<<<grid_for(n), 256, 0, s>>>(e->image, e->cfg.batch, e->cfg.height, e->cfg.width, e->H1, e->W1, e->buf("stem_col"));
    return cudaGetLastError();
}
cudaError_t fn_stem_pack(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->Hp * e->Wp;
    stem_pack_nhwc4_kernel<<<grid_for(n), 256, 0, s>>>(e->image, e->cfg.batch, e->cfg.height, e->cfg.width, e->Hp, e->Wp, e->buf("stem_x4"));
    return cudaGetLastError();
}
cudaError_t fn_stem_pack_planes(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->Hp * e->Wp;
    uint2* xh = reinterpret_cast<uint2*>(e->buf("stem_x4"));
    stem_pack_nhwc4_planes_kernel<<<grid_for(n), 256, 0, s>>>(e->image, e->cfg.batch, e->cfg.height, e->cfg.width, e->Hp, e->Wp, xh, xh + n,
                                                             e->buf<int>("range_flag"));
    return cudaGetLastError();
}
cudaError_t fn_maxpool(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->H2 * e->W2 * 16;
    maxpool3x3s2_nhwc_kernel<false><<<grid_for(n), 256, 0, s>>>(e->buf("c1"), e->cfg.batch, e->H1, e->W1, 64, e->H2, e->W2, e->buf("pool"), nullptr);
    return cudaGetLastError();
}
cudaError_t fn_maxpool_planes(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->H2 * e->W2 * 16;
    maxpool3x3s2_nhwc_kernel<true><<<grid_for(n), 256, 0, s>>>(e->buf("c1"), e->cfg.batch, e->H1, e->W1, 64, e->H2, e->W2, e->buf("pool"),
                                                              e->buf<int>("range_flag"));
    return cudaGetLastError();
}

cudaError_t fn_p6(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->LH[4] * e->LW[4] * 64;
    subsample2_nhwc_kernel<<<grid_for(n), 256, 0, s>>>(e->buf("P5"), e->cfg.batch, e->LH[3], e->LW[3], 256, e->LH[4], e->LW[4], e->buf("P6"));
    return cudaGetLastError();
}
// Proposal generation: the keys / two-level radix select / ordered compaction of every (level, image) run at full-GPU width
// (rpn_select_*_kernel, one CTA per 4096 anchors), then one CTA per (level, image) sorts the ~1000 selected candidates, decodes, clips,
// filters and runs the NMS.  DT_RPN_SPLIT=0 keeps the whole level in that one CTA (the round-1 kernel; P2's 182 400 anchors were its long pole).
// which of the two splits a proposal launch uses (also what dt_engine_count_launches reports before the first run)
void rpn_modes(Engine* e, int levels) {
    static int split = -1, nms_split = -1;
    if (split < 0) { const char* v = getenv("DT_RPN_SPLIT"); split = (v && v[0] == '0') ? 0 : 1; }
    if (nms_split < 0) { const char* v = getenv("DT_RPN_NMS_SPLIT"); nms_split = (v && v[0] == '0') ? 0 : 1; }
    RpnParams& P = e->rpn;
    int max_n = 0;
    for (int l = 0; l < levels; ++l) max_n = std::max(max_n, P.lv[l].n);
    P.split = (split && max_n <= kRpnChunk * kRpnMaxChunks) ? 1 : 0;
    P.nms_split = (nms_split && P.pre_nms <= 8192 && P.nms_thresh > 0.f) ? 1 : 0;
}
cudaError_t launch_proposals(Engine* e, cudaStream_t s, int levels) {
    RpnParams& P = e->rpn;
    P.scaling_factor = e->scaling_factor;
    rpn_modes(e, levels);
    int max_n = 0;
    for (int l = 0; l < levels; ++l) max_n = std::max(max_n, P.lv[l].n);
    if (P.split) {
        cudaError_t err = cudaMemsetAsync(P.sel_hist, 0, (size_t)e->cfg.batch * levels * 4096 * sizeof(uint32_t), s);
        if (err != cudaSuccess) return err;
        const dim3 grid((max_n + kRpnChunk - 1) / kRpnChunk, levels, e->cfg.batch);
        rpn_select_keys_kernel<<<grid, 1024, 0, s>>>(P);
        rpn_select_hist2_kernel<<<grid, 1024, 0, s>>>(P);
        rpn_select_count_kernel<<<grid, 1024, 0, s>>>(P);
        rpn_select_scatter_kernel<<<grid, 1024, 0, s>>>(P);
    }
    rpn_proposals_kernel<<<dim3(levels, e->cfg.batch), 1024, 0, s>>>(P);
    if (P.nms_split) {
        // DT_RPN_NMS_SPLIT=0 keeps the NMS inside rpn_proposals_kernel (one CTA per (level, image) sweeping every candidate over the survivors)
        rpn_nms_mask_kernel<<<dim3(P.nms_chunks, P.nms_chunks, levels * e->cfg.batch), 64, 0, s>>>(P);
        rpn_nms_scan_kernel<<<dim3(levels, e->cfg.batch), 1024, 0, s>>>(P);
    }
    return cudaGetLastError();
}
cudaError_t fn_proposals(Engine* e, cudaStream_t s) { return launch_proposals(e, s, 5); }
cudaError_t fn_collect(Engine* e, cudaStream_t s) {
    collect_kernel<<<e->cfg.batch, 1024, 0, s>>>(e->col);
    return cudaGetLastError();
}
cudaError_t fn_roi_box(Engine* e, cudaStream_t s) {
    const int R = e->cfg.batch * e->cfg.post_nms_top_n;
    // per-image counts: padded rows carry zero boxes (collect_kernel) -> harmless, fully defined output
    if (e->cfg.exact_roialign)
        roi_align_nhwc_kernel<<<R < num_sms() * 64 ? R : num_sms() * 64, 256, 0, s>>>(e->roi_lv, e->buf("rois"), e->buf<int>("roi_levels"), nullptr, R, 256, 7, 7,
                                                                          2, e->buf("roi_feat"));
    else
        roi_align_fast_nhwc_kernel<<<R < num_sms() * 64 ? R : num_sms() * 64, 256, 0, s>>>(e->roi_lv, e->buf("rois"), e->buf<int>("roi_levels"), R, 256, 7, 7,
                                                                               e->buf("roi_feat"));
    return cudaGetLastError();
}
cudaError_t fn_softmax(Engine* e, cudaStream_t s) {
    const int M = e->cfg.batch * e->cfg.post_nms_top_n, NC = e->cfg.num_classes;
    softmax_split_kernel<<<(M + 7) / 8, 256, 0, s>>>(e->buf("head"), M, (int)align_up((size_t)5 * NC, 4), NC, e->cfg.output_prob, e->buf("cls_prob"),
                                                     e->buf("bbox_pred"));
    return cudaGetLastError();
}
cudaError_t fn_detect(Engine* e, cudaStream_t s) {
    e->det.scaling_factor = e->scaling_factor;
    e->det.im_h = e->orig_h > 0.f ? e->orig_h : (float)e->cfg.height / e->scaling_factor;
    e->det.im_w = e->orig_w > 0.f ? e->orig_w : (float)e->cfg.width / e->scaling_factor;
    det_class_kernel<<<dim3(e->cfg.num_classes - 1, e->cfg.batch), 256, 0, s>>>(e->det);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    det_limit_kernel<<<e->cfg.batch, 1024, 0, s>>>(e->det);
    return cudaGetLastError();
}
cudaError_t fn_mask_rois(Engine* e, cudaStream_t s) {
    const int n = e->cfg.batch * e->cfg.det_cap;
    mask_rois_kernel<<<(n + 255) / 256, 256, 0, s>>>(e->buf("det_boxes"), e->buf<int>("det_counts"), e->cfg.batch, e->cfg.det_cap, e->scaling_factor, 2, 5,
                                                    e->buf("mask_rois"), e->buf<int>("mask_levels"));
    return cudaGetLastError();
}
cudaError_t fn_mask_roi_feat(Engine* e, cudaStream_t s) {
    const int D = e->cfg.batch * e->cfg.det_cap;
    if (e->cfg.exact_roialign)
        roi_align_nhwc_kernel<<<D < num_sms() * 64 ? D : num_sms() * 64, 256, 0, s>>>(e->roi_lv, e->buf("mask_rois"), e->buf<int>("mask_levels"), nullptr, D, 256, 14,
                                                                          14, 2, e->buf("mask_feat"));
    else
        roi_align_fast_nhwc_kernel<<<D < num_sms() * 64 ? D : num_sms() * 64, 256, 0, s>>>(e->roi_lv, e->buf("mask_rois"), e->buf<int>("mask_levels"), D, 256, 14, 14,
                                                                               e->buf("mask_feat"));
    return cudaGetLastError();
}
cudaError_t fn_mask_out(Engine* e, cudaStream_t s) {
    const int D = e->cfg.batch * e->cfg.det_cap, NC = e->cfg.num_classes;
    const long long n = (long long)D * 28 * 28;
    mask_select_kernel<<<grid_for(n), 256, 0, s>>>(e->buf("mask_logits"), e->buf<int>("det_classes"), D, 28, (int)align_up((size_t)NC, 4), NC,
                                                  e->cfg.output_prob, e->buf("masks"), e->cfg.emit_full_masks ? e->buf("masks_full") : nullptr);
    return cudaGetLastError();
}

// generate_anchors.py:54-122 on the host (float64, np.round == rint half-to-even)
void gen_anchors(double stride, double size, float* out /*3x4*/) {
    const double ratios[3] = {0.5, 1.0, 2.0};
    const double base = stride, cx = 0.5 * (base - 1), area = base * base;
    for (int r = 0; r < 3; ++r) {
        const double wr = nearbyint(sqrt(area / ratios[r]));
        const double hr = nearbyint(wr * ratios[r]);
        const double sc = size / stride;
        const double ws = wr * sc, hs = hr * sc;
        out[r * 4 + 0] = (float)(cx - 0.5 * (ws - 1)); out[r * 4 + 1] = (float)(cx - 0.5 * (hs - 1));
        out[r * 4 + 2] = (float)(cx + 0.5 * (ws - 1)); out[r * 4 + 3] = (float)(cx + 0.5 * (hs - 1));
    }
}

bool build_program(Engine* e, std::map<std::string, ConvW>* cw) {
    const dt_engine_config& c = e->cfg;
    const int B = c.batch;
    ProgBuilder pb{e, cw};
    // ---- trunk (detector.py:170-183)
    {
        // fused-window stem (no im2col buffer); falls back to im2col + GEMM if the driver rejects the overlapping-stride map
        const ConvW& sw = (*cw)["stem"];
        Op op;
        op.stage = ST_TRUNK; op.kind = 0; op.fn = -1;
        op.flops = 2.0 * (double)B * e->H1 * e->W1 * 64.0 * 147.0;
        bool stem_planes = false;
        if (c.stem_im2col) {
            e->stem_fused = false;
        } else if (c.conv_kind == 0) {
            op.matrix = e->matrix_of(sw.w);
            op.scale_src = e->wvec(sw.scale); op.scale16 = e->scale16_arena() + e->scale16_used; op.scale_n = 64;
            e->scale16_used += 64;
            // plane_handover >= 3: the packed image arrives as two fp16 planes (the stem's converter warps -- 7 k-blocks of fp32 -> fp16
            // splits per 64-wide tile -- were what bounded it)
            stem_planes = c.plane_handover >= 3 && (e->Wp % 2) == 0;
            e->stem_fused = conv_build_stem(e->buf("stem_x4"), B, e->Hp, e->Wp, e->H1, e->W1, e->whi16(sw.w + 64 * 160), e->wlo16(sw.w + 64 * 160),
                                            op.scale16, e->wvec(sw.shift), e->buf("c1"), c.passes, &op.conv, KIND_F16X3, e->buf<int>("range_flag"),
                                            stem_planes);
            if (!e->stem_fused) { op.scale16 = nullptr; op.scale_src = nullptr; }
        } else {
            e->stem_fused = conv_build_stem(e->buf("stem_x4"), B, e->Hp, e->Wp, e->H1, e->W1, e->wmat(sw.w + 64 * 160), e->wlo(sw.w + 64 * 160),
                                            e->wvec(sw.scale), e->wvec(sw.shift), e->buf("c1"), c.passes, &op.conv);
        }
        if (e->stem_fused) {
            pb.fn(ST_TRUNK, stem_planes ? fn_stem_pack_planes : fn_stem_pack);
            e->ops.push_back(op);
        } else {
            if (!c.stem_im2col) fprintf(stderr, "[detectorch_b200] engine: fused stem descriptor rejected, using the im2col stem\n");
            pb.fn(ST_TRUNK, fn_stem_im2col);
            pb.conv(ST_TRUNK, "stem", e->buf("stem_col"), 1, 1, B * e->H1 * e->W1, 160, e->buf("c1"), 64, 0, 1, true);
        }
    }
    // plane_handover >= 4 (opt-in): the pooled map leaves as fp16 planes too (its two consumers -- conv1 and the downsample conv of the first
    // bottleneck -- then load their operand tiles directly).  Measured twice, before and after the epilogue rewrite: the consumers gain 7 us
    // each, the pool kernel loses 16 us -- no net gain, so the default hand-over level stays 3.
    const int pool_planes = (c.conv_kind == 0 && c.plane_handover >= 4) ? 1 : 0;
    pb.fn(ST_TRUNK, pool_planes ? fn_maxpool_planes : fn_maxpool);
    const float* x = e->buf("pool");
    int h = e->H2, w = e->W2, cin = 64;
    for (int li = 1; li <= 4; ++li) {
        const int planes = 64 << (li - 1);
        for (int b = 0; b < c.arch_blocks[li - 1]; ++b) {
            const std::string p = "l" + std::to_string(li) + "b" + std::to_string(b);
            const std::string wp = "model.layer" + std::to_string(li) + "." + std::to_string(b) + ".";
            const int stride = (b == 0 && li > 1) ? 2 : 1;
            const int ho = e->LH[li - 1], wo = e->LW[li - 1];
            // conv1 -> conv2 hand-over as fp16 hi/lo planes: the 3x3 conv would otherwise re-convert every input element once per filter tap
            // (the converter warps' fp32->fp16 packs are what bounds the 64/128-wide layers)
            const int pl = c.plane_handover ? 1 : 0;
            const int xin_planes = (li == 1 && b == 0) ? pool_planes : 0;
            pb.conv(ST_TRUNK, wp + "conv1", x, B, h, w, cin, e->buf(p + ".t1"), planes, 0, stride, true, RES_NONE, nullptr, nullptr, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                    0, 0, 0, false, xin_planes, pl);
            // conv2 -> conv3 the same way (plane_handover >= 2): conv3 is a 1x1 conv, so this saves one conversion per element, the converter
            // warps' shared-memory round trip (16 KB read + 16 KB written per k-block) and their issue slots in the epilogue-bound conv3
            const int pl2 = c.plane_handover >= 2 ? 1 : 0;
            pb.conv(ST_TRUNK, wp + "conv2", e->buf(p + ".t1"), B, ho, wo, planes, e->buf(p + ".t2"), planes, 1, 1, true, RES_NONE, nullptr, nullptr, 0, 0, 0,
                    0, 0, 0, 0, 0, 0, 0, 0, 0, false, pl, pl2);
            const float* idt = x;
            if (b == 0) {
                pb.conv(ST_TRUNK, wp + "downsample.0", x, B, h, w, cin, e->buf(p + ".ds"), planes * 4, 0, stride, false, RES_NONE, nullptr, nullptr, 0, 0, 0,
                        0, 0, 0, 0, 0, 0, 0, 0, 0, false, xin_planes, 0);
                idt = e->buf(p + ".ds");
            }
            pb.conv(ST_TRUNK, wp + "conv3", e->buf(p + ".t2"), B, ho, wo, planes, e->buf(p + ".out"), planes * 4, 0, 1, true, RES_TILE, idt, nullptr, 0, 0, 0,
                    0, 0, 0, 0, 0, 0, 0, 0, 0, false, pl2, 0);
            x = e->buf(p + ".out");
            h = ho; w = wo; cin = planes * 4;
        }
        e->bufs["C" + std::to_string(li + 1)] = e->bufs["l" + std::to_string(li) + "b" + std::to_string(c.arch_blocks[li - 1] - 1) + ".out"];
    }
    // ---- FPN (detector.py:35-52)
    const int cins[4] = {256, 512, 1024, 2048};
    for (int i = 3; i >= 0; --i) {
        const std::string ln = "conv_body.fpn_lateral." + std::to_string(i);
        const float* src = e->buf("C" + std::to_string(i + 2));
        if (i == 3)
            pb.conv(ST_FPN, ln, src, B, e->LH[i], e->LW[i], cins[i], e->buf("inner5"), 256, 0, 1, false);
        else
            pb.conv(ST_FPN, ln, src, B, e->LH[i], e->LW[i], cins[i], e->buf("inner" + std::to_string(i + 2)), 256, 0, 1, false, RES_UPSAMPLE2X,
                    nullptr, e->buf("inner" + std::to_string(i + 3)), e->LH[i + 1], e->LW[i + 1]);
    }
    for (int i = 0; i < 4; ++i)
        pb.conv(ST_FPN, "conv_body.fpn_output." + std::to_string(i), e->buf("inner" + std::to_string(i + 2)), B, e->LH[i], e->LW[i], 256,
                e->buf("P" + std::to_string(i + 2)), 256, 1, 1, false);
    pb.fn(ST_FPN, fn_p6);
    // ---- RPN head on P2..P6 (detector.py:251)
    for (int i = 0; i < 5 && c.use_rpn; ++i) {
        const std::string L = std::to_string(i + 2);
        pb.conv(ST_RPN, "rpn.conv_rpn", e->buf("P" + L), B, e->LH[i], e->LW[i], 256, e->buf("rpn_t" + L), 256, 1, 1, true);
        pb.conv(ST_RPN, "rpn.head", e->buf("rpn_t" + L), B, e->LH[i], e->LW[i], 256, e->buf("rpn_out" + L), 16, 0, 1, false, RES_NONE, nullptr,
                nullptr, 0, 0, 3);
    }
    // ---- proposals (generate_proposals.py) + collect (collect_and_distribute...py)
    if (c.use_rpn) {
        RpnParams& P = e->rpn;
        memset(&P, 0, sizeof(P));
        P.num_levels = 5; P.B = B;
        P.pre_nms = c.pre_nms_top_n; P.post_nms = c.post_nms_top_n;
        P.nms_thresh = c.rpn_nms_thresh; P.min_size = c.rpn_min_size; P.scaling_factor = 1.f;
        P.im_h = (float)c.height; P.im_w = (float)c.width;
        long long off = 0;
        for (int i = 0; i < 5; ++i) {
            RpnLevel& lv = P.lv[i];
            lv.rpn_out = e->buf("rpn_out" + std::to_string(i + 2));
            lv.H = e->LH[i]; lv.W = e->LW[i]; lv.A = 3; lv.ch_stride = 16;
            lv.stride = (float)(4 << i);
            gen_anchors((double)(4 << i), (double)(32 << i), lv.anchors);
            lv.n = lv.H * lv.W * 3;
            lv.ws_off = off;
            off += lv.n;
        }
        P.ws_per_image = off;
        P.k0 = e->buf<uint32_t>("rpn_k0"); P.k1 = e->buf<uint32_t>("rpn_k1");
        P.v0 = e->buf<int>("rpn_v0"); P.v1 = e->buf<int>("rpn_v1");
        P.cand = e->buf<float4>("rpn_cand"); P.cand_score = e->buf("rpn_cand_score");
        P.out_props = e->buf("props"); P.out_scores = e->buf("prop_scores"); P.out_counts = e->buf<int>("prop_counts");
        P.dbg_order = e->buf<int>("rpn_order");
        P.sel_hist = e->buf<uint32_t>("rpn_sel_hist"); P.sel_chunk_counts = e->buf<int>("rpn_sel_cc"); P.sel_info = e->buf<int>("rpn_sel_info");
        P.cand_counts = e->buf<int>("rpn_cand_counts"); P.nms_mask = e->buf<unsigned long long>("rpn_nms_mask"); P.nms_chunks = (c.pre_nms_top_n + 63) / 64;
        pb.fn(ST_PROPOSALS, fn_proposals);
        CollectParams& C = e->col;
        memset(&C, 0, sizeof(C));
        C.props = P.out_props; C.scores = P.out_scores; C.counts = P.out_counts;
        C.B = B; C.L = 5; C.post_nms = c.post_nms_top_n; C.top_n = c.post_nms_top_n; C.k_min = 2; C.k_max = 5;
        C.k0 = e->buf<uint32_t>("col_k0"); C.k1 = e->buf<uint32_t>("col_k1"); C.v0 = e->buf<int>("col_v0"); C.v1 = e->buf<int>("col_v1");
        C.rois = e->buf("rois"); C.levels = e->buf<int>("roi_levels"); C.roi_counts = e->buf<int>("roi_counts");
        pb.fn(ST_COLLECT, fn_collect);
    }
    // ---- RoIAlign 7x7 over P2..P5 in collected order (detector.py:259-270)
    e->roi_lv.num_levels = 4;
    for (int i = 0; i < 4; ++i) {
        e->roi_lv.feat[i] = e->buf("P" + std::to_string(i + 2));
        e->roi_lv.H[i] = e->LH[i]; e->roi_lv.W[i] = e->LW[i];
        e->roi_lv.scale[i] = 1.f / (float)(4 << i);
    }
    pb.fn(ST_ROI_BOX, fn_roi_box);
    // ---- box head (detector.py:61-64,277-284)
    const int R = B * c.post_nms_top_n, NC = c.num_classes, HN = (int)align_up((size_t)5 * NC, 4);
    pb.conv(ST_BOX_HEAD, "fc6", e->buf("roi_feat"), 1, 1, R, 49 * 256, e->buf("fc6"), 1024, 0, 1, true);
    pb.conv(ST_BOX_HEAD, "fc7", e->buf("fc6"), 1, 1, R, 1024, e->buf("fc7"), 1024, 0, 1, true);
    pb.conv(ST_BOX_HEAD, "head", e->buf("fc7"), 1, 1, R, 1024, e->buf("head"), HN, 0, 1, false);
    pb.fn(ST_BOX_HEAD, fn_softmax);
    // ---- detection post-processing (result_utils.py:76-168)
    {
        DetParams& D = e->det;
        memset(&D, 0, sizeof(D));
        D.rois = e->buf("rois"); D.roi_counts = e->buf<int>("roi_counts"); D.cls = e->buf("cls_prob"); D.bbox = e->buf("bbox_pred");
        D.B = B; D.R = c.post_nms_top_n; D.NC = NC;
        D.wx = 10.f; D.wy = 10.f; D.ww = 5.f; D.wh = 5.f;
        D.score_thresh = c.score_thresh; D.nms_thresh = c.det_nms_thresh; D.max_dets = c.max_dets; D.out_cap = c.det_cap;
        D.keep_flag = e->buf<unsigned char>("det_flag"); D.dec_box = e->buf<float4>("det_dec"); D.cls_counts = e->buf<int>("det_cls_counts");
        D.k0 = e->buf<uint32_t>("det_k0"); D.k1 = e->buf<uint32_t>("det_k1"); D.v0 = e->buf<int>("det_v0"); D.v1 = e->buf<int>("det_v1");
        D.out_boxes = e->buf("det_boxes"); D.out_scores = e->buf("det_scores"); D.out_classes = e->buf<int>("det_classes");
        D.out_roi_idx = e->buf<int>("det_roi_idx"); D.out_counts = e->buf<int>("det_counts");
        pb.fn(ST_DETECT, fn_detect);
    }
    // ---- mask head (detector.py:99-112)
    if (c.use_mask) {
        const int D = B * c.det_cap, MN = (int)align_up((size_t)NC, 4);
        // The mask logits carry the tightest parity bar (1e-4 absolute) and sit behind four K = 2304 convolutions, where the tensor
        // core's truncating fp32 accumulate is the error floor.  precise_mask shortens the chains by SPLITTING K: each 3x3 convolution
        // runs as two launches over filter taps [0,5) and [5,9); the second adds the first's fp32 result in its epilogue (RES_TILE on the
        // output buffer itself, round-to-nearest) before the ReLU.  precise_mask = 2 instead runs 64-wide tiles with 3 rotating
        // main-term accumulators.
        const int mbn = c.precise_mask == 2 ? 128 : 0;
        pb.fn(ST_MASK_ROIS, fn_mask_rois);
        pb.fn(ST_MASK_ROI_FEAT, fn_mask_roi_feat);
        const float* mx = e->buf("mask_feat");
        for (int i = 1; i <= 4; ++i) {
            const std::string wn = "mask_head.conv_head.fcn" + std::to_string(i);
            float* my = e->buf("mask_c" + std::to_string(i));
            if (c.precise_mask == 1) {
                pb.conv(ST_MASK_HEAD, wn, mx, D, 14, 14, 256, my, 256, 1, 1, false, RES_NONE, nullptr, nullptr, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 5);
                pb.conv(ST_MASK_HEAD, wn, mx, D, 14, 14, 256, my, 256, 1, 1, true, RES_TILE, my, nullptr, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 5, 4, true);
            } else {
                pb.conv(ST_MASK_HEAD, wn, mx, D, 14, 14, 256, my, 256, 1, 1, true, RES_NONE, nullptr, nullptr, 0, 0, 0, 0, 0, 0, 0, 0, 0, mbn);
            }
            mx = my;
        }
        for (int ij = 0; ij < 4; ++ij)     // ConvTranspose2d(2, stride 2) == 4 GEMMs scattered on the 2x grid
            pb.conv(ST_MASK_HEAD, "deconv", mx, D, 14, 14, 256, e->buf("mask_up"), 256, 0, 1, true, RES_NONE, nullptr, nullptr, 0, 0, 0,
                    (size_t)ij * 256 * 256, 28, 28, 2, ij / 2, ij % 2, mbn);
        pb.conv(ST_MASK_HEAD, "mask_logits", e->buf("mask_up"), D, 28, 28, 256, e->buf("mask_logits"), MN, 0, 1, false);
        pb.fn(ST_MASK_OUT, fn_mask_out);
    }
    return pb.ok;
}

#include "engine_c4.inc"

int load_param(Engine* e, const std::string& name, const float* src, long long numel, cudaStream_t st) {
    auto it = e->params.find(name);
    if (it == e->params.end()) return 2;   // not a hot-path parameter (running stats, fc, duplicates): ignored
    ParamSlot& s = it->second;
    if (!e->wbase) { fprintf(stderr, "[detectorch_b200] engine: bind weights before loading parameters\n"); return 0; }
    long long expect = 0;
    switch (s.kind) {
        case PK_CONV_W: expect = (long long)s.d0 * s.d1 * s.d2 * s.d3; break;
        case PK_STEM_W: expect = (long long)s.d0 * s.d1; break;
        case PK_FC6_W: expect = (long long)s.d0 * s.d1 * s.d2; break;
        case PK_ROWS_W: expect = (long long)s.d0 * s.d1; break;
        case PK_DECONV_W: expect = 4ll * s.d0 * s.d1; break;
        default: expect = s.d0;
    }
    if (expect != numel) {
        fprintf(stderr, "[detectorch_b200] engine: parameter %s has %lld elements, expected %lld\n", name.c_str(), numel, expect);
        return 0;
    }
    switch (s.kind) {
        case PK_CONV_W: pack_conv_w_kernel<<<grid_for(numel), 256, 0, st>>>(src, s.d0, s.d1, s.d2, s.d3, e->wmat(s.off)); break;
        case PK_STEM_W:
            pack_rows_kernel<<<grid_for((long long)s.d0 * s.d2), 256, 0, st>>>(src, s.d0, s.d1, s.d2, e->wmat(s.off));
            pack_stem_window_kernel<<<(64 * 224 + 255) / 256, 256, 0, st>>>(src, e->wmat(s.off) + 64 * 160);
            break;
        case PK_FC6_W: pack_fc6_kernel<<<grid_for(numel), 256, 0, st>>>(src, s.d0, s.d1, s.d2, e->wmat(s.off)); break;
        case PK_ROWS_W: pack_rows_kernel<<<grid_for(numel), 256, 0, st>>>(src, s.d0, s.d1, s.d1, e->wmat(s.off) + (size_t)s.row_off * s.Kout); break;
        case PK_DECONV_W: pack_deconv_kernel<<<grid_for(numel), 256, 0, st>>>(src, s.d0, s.d1, e->wmat(s.off)); break;
        case PK_BN_SCALE: bn_scale_kernel<<<(s.d0 + 255) / 256, 256, 0, st>>>(src, s.d0, e->wvec(s.off)); break;
        case PK_VEC: copy_kernel<<<grid_for(numel), 256, 0, st>>>(src, numel, e->wvec(s.off) + s.row_off); break;
    }
    if (cudaGetLastError() != cudaSuccess) return 0;
    s.loaded = true;
    return 1;
}

}  // namespace

// ================================================================================== C ABI
extern "C" {

dt_engine_t dt_engine_create(const dt_engine_config* cfg) {
    if (!cfg || cfg->batch < 1 || cfg->height < 32 || cfg->width < 32 || (cfg->model_type != 1 && ((cfg->height % 32) || (cfg->width % 32)))) {
        fprintf(stderr, "[detectorch_b200] engine: image size must be a multiple of 32 (FPN), batch >= 1\n");
        return nullptr;
    }
    if (cfg->pre_nms_top_n < 1 || cfg->pre_nms_top_n > 8192 || cfg->post_nms_top_n < 1 || cfg->post_nms_top_n > 1024 || cfg->det_cap < cfg->max_dets ||
        cfg->num_classes < 2 || cfg->num_classes > 128) {
        fprintf(stderr, "[detectorch_b200] engine: unsupported proposal/detection limits\n");
        return nullptr;
    }
    Engine* e = new Engine();
    e->cfg = *cfg;
    if (e->cfg.passes != 1) e->cfg.passes = 3;
    std::map<std::string, ConvW> cw;
    if (e->cfg.model_type == 1) { build_param_table_c4(e, &cw); plan_buffers_c4(e); }
    else { build_param_table(e, &cw); plan_buffers(e); }
    return e;
}

void dt_engine_destroy(dt_engine_t h) { delete reinterpret_cast<Engine*>(h); }

int64_t dt_engine_weight_bytes(dt_engine_t h) {
    Engine* e = reinterpret_cast<Engine*>(h);
    return (int64_t)e->weight_bytes();
}
int64_t dt_engine_workspace_bytes(dt_engine_t h) { return (int64_t)reinterpret_cast<Engine*>(h)->ws_bytes; }

static int bind_impl(Engine* e, void* weights, void* workspace, cudaStream_t st, bool fresh) {
    e->wbase = reinterpret_cast<float*>(weights);
    e->ws = reinterpret_cast<uint8_t*>(workspace);
    if (fresh) {
        DT_CHECK_CUDA(cudaMemsetAsync(weights, 0, (2 * e->mat_floats + e->vec_floats) * sizeof(float), st));
        // the shared all-ones scale vector sits at the start of the vector region
        fill_kernel<<<8, 256, 0, st>>>(e->wvec(0), 2048, 1.f);
        if (e->cfg.model_type != 1) fill_kernel<<<8, 256, 0, st>>>(e->wvec(2048), 2048, 0.f);
        DT_CHECK_CUDA(cudaGetLastError());
    }
    e->ops.clear();
    e->scale16_used = 0;
    e->fns.clear();
    std::map<std::string, ConvW> cw;
    {   // rebuild the (deterministic) table to recover the ConvW offsets
        Engine tmp;
        tmp.cfg = e->cfg;
        if (e->cfg.model_type == 1) build_param_table_c4(&tmp, &cw); else build_param_table(&tmp, &cw);
    }
    if (!(e->cfg.model_type == 1 ? build_program_c4(e, &cw) : build_program(e, &cw))) return 0;
    e->bound = true;
    return 1;
}

int dt_engine_bind(dt_engine_t h, void* weights, void* workspace, dt_stream_t stream) {
    return bind_impl(reinterpret_cast<Engine*>(h), weights, workspace, (cudaStream_t)stream, true);
}

// Bind to a weight buffer that ANOTHER engine of the same model configuration (everything in dt_engine_config except batch / height /
// width) has already loaded and finalised: the packed weights, their fp16 halves and the per-launch scale vectors do not depend on the
// input shape, so engines for different image sizes share one copy (the notebook flow meets dozens of padded sizes).  Nothing is
// written to `loaded_weights`; every parameter counts as loaded.
int dt_engine_attach(dt_engine_t h, void* loaded_weights, void* workspace, dt_stream_t stream) {
    Engine* e = reinterpret_cast<Engine*>(h);
    if (!bind_impl(e, loaded_weights, workspace, (cudaStream_t)stream, false)) return 0;
    for (auto& kv : e->params) kv.second.loaded = true;
    return 1;
}

int dt_engine_load_param(dt_engine_t h, const char* name, const float* src_dev, int64_t numel, dt_stream_t stream) {
    return load_param(reinterpret_cast<Engine*>(h), name, src_dev, numel, (cudaStream_t)stream);
}

int dt_engine_finalize_weights(dt_engine_t h, dt_stream_t stream) {
    Engine* e = reinterpret_cast<Engine*>(h);
    int missing = 0;
    for (auto& kv : e->params)
        if (!kv.second.loaded) { fprintf(stderr, "[detectorch_b200] engine: parameter %s was never loaded\n", kv.first.c_str()); ++missing; }
    if (missing) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    tf32_lo_kernel<<<grid_for((long long)e->mat_floats), 256, 0, st>>>(e->wmat(0), e->wlo(0), (long long)e->mat_floats);
    DT_CHECK_CUDA(cudaGetLastError());
    if (e->cfg.conv_kind == 0) {
        // fp16 halves of every matrix, pre-scaled by a per-matrix power of two derived on the device (no host sync)
        const int nm = (int)e->matrices.size();
        if ((size_t)nm > Engine::kMaxMatrices) { fprintf(stderr, "[detectorch_b200] engine: too many weight matrices\n"); return 0; }
        DT_CHECK_CUDA(cudaMemsetAsync(e->matinfo(), 0, nm * sizeof(MatInfo), st));
        for (int m = 0; m < nm; ++m)
            absmax_kernel<<<grid_for((long long)e->matrices[m].second), 256, 0, st>>>(e->wmat(e->matrices[m].first), (long long)e->matrices[m].second,
                                                                                     e->matinfo() + m);
        matmult_kernel<<<(nm + 255) / 256, 256, 0, st>>>(e->matinfo(), nm);
        for (int m = 0; m < nm; ++m)
            fp16_split_dev_kernel<<<grid_for((long long)e->matrices[m].second), 256, 0, st>>>(
                e->wmat(e->matrices[m].first), (long long)e->matrices[m].second, e->matinfo() + m, e->whi16(e->matrices[m].first),
                e->wlo16(e->matrices[m].first));
        for (const Op& op : e->ops)
            if (op.kind == 0 && op.scale16)
                scale16_kernel<<<(op.scale_n + 255) / 256, 256, 0, st>>>(op.scale_src, e->matinfo() + op.matrix, op.scale16, op.scale_n);
        DT_CHECK_CUDA(cudaGetLastError());
    }
    return 1;
}

int dt_engine_buffer(dt_engine_t h, const char* name, int64_t* byte_offset, int* ndim, int* dims5, int* dtype) {
    Engine* e = reinterpret_cast<Engine*>(h);
    auto it = e->bufs.find(name);
    if (it == e->bufs.end()) return 0;
    *byte_offset = (int64_t)it->second.off;
    *ndim = it->second.nd;
    for (int i = 0; i < 5; ++i) dims5[i] = it->second.dims[i];
    *dtype = it->second.dtype;
    return 1;
}

int dt_engine_num_stages(void) { return ST_COUNT; }

int dt_engine_param_count(dt_engine_t h) { return (int)reinterpret_cast<Engine*>(h)->params.size(); }
// i-th parameter name (sorted) and its expected element count; returns 0 when out of range
int dt_engine_param_info(dt_engine_t h, int i, char* name_out, int name_cap, int64_t* numel) {
    Engine* e = reinterpret_cast<Engine*>(h);
    if (i < 0 || i >= (int)e->params.size()) return 0;
    auto it = e->params.begin();
    std::advance(it, i);
    snprintf(name_out, name_cap, "%s", it->first.c_str());
    const ParamSlot& s = it->second;
    long long n = 0;
    switch (s.kind) {
        case PK_CONV_W: n = (long long)s.d0 * s.d1 * s.d2 * s.d3; break;
        case PK_STEM_W: n = (long long)s.d0 * s.d1; break;
        case PK_FC6_W: n = (long long)s.d0 * s.d1 * s.d2; break;
        case PK_ROWS_W: n = (long long)s.d0 * s.d1; break;
        case PK_DECONV_W: n = 4ll * s.d0 * s.d1; break;
        default: n = s.d0;
    }
    *numel = n;
    return 1;
}

int dt_engine_set_original_size(dt_engine_t h, float orig_h, float orig_w) {
    Engine* e = reinterpret_cast<Engine*>(h);
    e->orig_h = orig_h; e->orig_w = orig_w;
    return 1;
}

// Runs stages [first, last] of the program (see enum Stage) on `stream`.  `image` NCHW [B,3,H,W] is read by stage 0 only.
int dt_engine_run(dt_engine_t h, const float* image_nchw, float scaling_factor, int first_stage, int last_stage, dt_stream_t stream) {
    Engine* e = reinterpret_cast<Engine*>(h);
    if (!e->bound) { fprintf(stderr, "[detectorch_b200] engine: not bound\n"); return 0; }
    if (first_stage <= ST_TRUNK && !image_nchw) { fprintf(stderr, "[detectorch_b200] engine: image pointer required\n"); return 0; }
    e->image = image_nchw;
    e->scaling_factor = scaling_factor;
    cudaStream_t st = (cudaStream_t)stream;
    // a run from the first stage reports ITS OWN range flag (it used to stay raised until someone read it through Engine.check_range)
    if (first_stage <= ST_TRUNK && cudaMemsetAsync(e->buf<int>("range_flag"), 0, sizeof(int), st) != cudaSuccess) return 0;
    for (const Op& op : e->ops) {
        if (op.stage < first_stage || op.stage > last_stage) continue;
        cudaError_t err = op.kind == 0 ? conv_launch(op.conv, st) : e->fns[op.fn](e, st);
        if (err != cudaSuccess) {
            fprintf(stderr, "[detectorch_b200] engine: launch failed in stage %d: %s\n", op.stage, cudaGetErrorString(err));
            return 0;
        }
    }
    return 1;
}

// Profiling pass: runs stages [first,last] once with a CUDA-event pair around every op ON `stream`, synchronises, and
// returns per-op milliseconds, algorithmic FLOPs (0 for non-GEMM ops), stage id and BLOCK_N (0 for non-GEMM ops).
// Returns the number of ops written (<= cap).  This is a measurement aid; the production path is dt_engine_run.
int dt_engine_profile(dt_engine_t h, const float* image_nchw, float scaling_factor, int first_stage, int last_stage, dt_stream_t stream,
                      float* ms_out, double* flops_out, int* stage_out, int* block_n_out, int cap) {
    Engine* e = reinterpret_cast<Engine*>(h);
    if (!e->bound) return 0;
    e->image = image_nchw;
    e->scaling_factor = scaling_factor;
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<cudaEvent_t> ev;
    std::vector<const Op*> sel;
    for (const Op& op : e->ops)
        if (op.stage >= first_stage && op.stage <= last_stage && (int)sel.size() < cap) sel.push_back(&op);
    ev.resize(sel.size() + 1);
    for (auto& x : ev) cudaEventCreate(&x);
    cudaEventRecord(ev[0], st);
    for (size_t i = 0; i < sel.size(); ++i) {
        const Op& op = *sel[i];
        cudaError_t err = op.kind == 0 ? conv_launch(op.conv, st) : e->fns[op.fn](e, st);
        if (err != cudaSuccess) { fprintf(stderr, "[detectorch_b200] engine profile: launch failed: %s\n", cudaGetErrorString(err)); return 0; }
        cudaEventRecord(ev[i + 1], st);
    }
    cudaStreamSynchronize(st);
    for (size_t i = 0; i < sel.size(); ++i) {
        cudaEventElapsedTime(&ms_out[i], ev[i], ev[i + 1]);
        flops_out[i] = sel[i]->flops;
        stage_out[i] = sel[i]->stage;
        block_n_out[i] = sel[i]->kind == 0 ? sel[i]->conv.block_n : 0;
    }
    for (auto& x : ev) cudaEventDestroy(x);
    return (int)sel.size();
}

// number of kernel launches stages [first,last] issue (bench.py's gpu_launches)
int dt_engine_count_launches(dt_engine_t h, int first_stage, int last_stage) {
    Engine* e = reinterpret_cast<Engine*>(h);
    int n = 0;
    if (e->cfg.use_rpn) rpn_modes(e, e->rpn.num_levels);
    for (const Op& op : e->ops)
        if (op.stage >= first_stage && op.stage <= last_stage)
            n += (op.kind == 1 && e->fns[op.fn] == fn_detect) ? 2 : ((op.kind == 1 && op.stage == ST_PROPOSALS) ? ((e->rpn.split ? 5 : 1) + (e->rpn.nms_split ? 2 : 0)) : 1);
    return n;
}

}  // extern "C"

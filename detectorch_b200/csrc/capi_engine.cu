// detectorch_b200 -- the fused Mask R-CNN (ResNet-50/101 + FPN) inference engine.
//
// One C++ object owns the whole hot path of reference lib/model/detector.py:233-286 (detector.forward),
// lib/utils/result_utils.py:76-168 (postprocess_output) and lib/model/detector.py:99-112 (mask_head.forward):
// a static program of kernel launches over pre-built TMA descriptors, with zero host synchronisation
// (the reference syncs >= 17 times per image, SURVEY.md 3.1).  Memory is supplied by the caller as two
// flat device buffers (weights, workspace) so that the host language (PyTorch here) stays pure plumbing.
// Both model families of the reference are built by the same code: FPN (R-50/101-FPN) and C4 (Fast / Faster / Mask R-CNN R-50/101-C4:
// trunk to layer3, single-level RPN with 15 anchors, RoIAlign 14x14 with the adaptive sampling grid, the res5 head = layer4 + avgpool
// per RoI, and the 'upshare' mask head that re-runs layer4 on the detections).  What differs between them is data (Family).
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

// element count of the tensor a parameter is loaded from
long long param_numel(const ParamSlot& s) {
    switch (s.kind) {
        case PK_CONV_W: return (long long)s.d0 * s.d1 * s.d2 * s.d3;
        case PK_FC6_W: return (long long)s.d0 * s.d1 * s.d2;
        case PK_STEM_W:
        case PK_ROWS_W: return (long long)s.d0 * s.d1;
        case PK_DECONV_W: return 4ll * s.d0 * s.d1;
        default: return s.d0;
    }
}

// A conv's weight matrix, scale and shift (float offsets into the weight buffer) and its GEMM shape.  flop_cout / flop_cin are the
// layer's own output channels and K per tap before the matrix is padded (what its algorithmic FLOPs count).
struct ConvW { size_t w = 0, scale = 0, shift = 0; int cout = 0, cin = 0, k = 1, flop_cout = 0, flop_cin = 0; };

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
    // kind::f16 convs: scale16 = scale / multiplier(matrix) is (re)derived at finalize time, for each weight matrix the launch reads
    // ([1]: the phase-1 matrix of a RES_STAGED launch)
    const float* scale_src[2] = {nullptr, nullptr};
    float* scale16[2] = {nullptr, nullptr};
    int scale_n[2] = {0, 0};
    int matrix[2] = {-1, -1};
};

// one RoIAlign launch: n RoIs (on the level `levels` gives, or all on level 0 when it is null) -> out [n, res, res, ch]
struct RoiPool { const char* rois; const char* levels; const char* out; int n, ch, res, sampling; bool fast; };

// What the FPN and C4 families build differently.  Level l is the map at stride 2^l (C2..C5, P2..P6); LH / LW[l - 2] is its size.
struct Family {
    bool c4;
    const char* feat;        // the maps the RPN and RoIAlign read: "P" (FPN P2..P6) or "C" (C4)
    int lv_min, lv_max;      // RoI levels (collect, RoIAlign, mask RoIs): FPN 2..5, C4 4
    int rpn_levels;          // RPN levels from lv_min: FPN 5 (P2..P6), C4 1
    int rpn_ch, anchors;     // RPN conv width, anchors per position
    int box_feat;            // input width of the class / box head: FPN fc7, C4 the pooled res5 output
    int mask_in, mask_res;   // mask head: deconv input channels, mask resolution
    RoiPool box_pool, mask_pool;
};

Family family_of(const dt_engine_config& c) {
    Family f;
    f.c4 = c.model_type == 1;
    const int R = c.batch * c.post_nms_top_n, D = c.batch * c.det_cap;
    if (f.c4) {
        // 15 anchors on the one 1024-channel C4 map; RoIAlign always runs the exact kernel with the adaptive sampling grid (ratio 0)
        f.feat = "C"; f.lv_min = f.lv_max = 4; f.rpn_levels = 1; f.rpn_ch = 1024; f.anchors = 15;
        f.box_feat = 2048; f.mask_in = 2048; f.mask_res = 14;
        f.box_pool = RoiPool{"rois", nullptr, "roi_feat", R, 1024, 14, 0, false};
        f.mask_pool = RoiPool{"mask_rois", nullptr, "mask_feat", D, 1024, 14, 0, false};
    } else {
        f.feat = "P"; f.lv_min = 2; f.lv_max = 5; f.rpn_levels = 5; f.rpn_ch = 256; f.anchors = 3;
        f.box_feat = 1024; f.mask_in = 256; f.mask_res = 28;
        f.box_pool = RoiPool{"rois", "roi_levels", "roi_feat", R, 256, 7, 2, !c.exact_roialign};
        f.mask_pool = RoiPool{"mask_rois", "mask_levels", "mask_feat", D, 256, 14, 2, !c.exact_roialign};
    }
    return f;
}

struct Engine;
typedef cudaError_t (*StageFn)(Engine*, cudaStream_t);

struct Engine {
    dt_engine_config cfg;
    Family fam;
    // weights
    std::map<std::string, ParamSlot> params;
    std::map<std::string, ConvW> convs;     // by layer: what the program's conv launches read
    size_t mat_floats = 0;      // hi-region floats (lo region has the same size)
    size_t vec_floats = 0;
    size_t zeros = 0;           // vector-region offset of the zero shift (FPN: the second half of a K-split mask conv)
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
    bool use_image_info = false;        // per-image sizes / scales from the "im_info" buffer (dt_engine_use_image_info)
    // static geometry
    int H1, W1, H2, W2;                 // stem out, pool out
    int Hp, Wp;                         // padded NHWC4 stem input
    int LH[5], LW[5];                   // levels 2..6
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
    // the per-image table the kernels read (image_info), or null when every image fills the canvas
    const float* im_info() { return use_image_info ? buf("im_info") : nullptr; }
};

// ---- parameter table ---------------------------------------------------------------------------
size_t add_mat(Engine* e, const std::string& name, ParamKind kind, int rows_total, int K, int d0, int d1, int d2, int d3) {
    ParamSlot s;
    s.kind = kind; s.d0 = d0; s.d1 = d1; s.d2 = d2; s.d3 = d3; s.row_off = 0; s.Kout = K;
    s.off = e->mat_floats;
    e->mat_floats += align_up((size_t)rows_total * K, 64);
    e->matrices.push_back(std::make_pair(s.off, e->mat_floats - s.off));
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

constexpr size_t kOnes = 0;     // the all-ones scale vector of the bias-only convs (2048 floats) opens the vector region

// conv + frozen BatchNorm (folded into the scale / shift)
void bn_conv(Engine* e, const std::string& name, const std::string& bn, int cout, int cin, int k) {
    ConvW c; c.cout = c.flop_cout = cout; c.cin = c.flop_cin = cin; c.k = k;
    c.w = add_mat(e, name + ".weight", PK_CONV_W, cout, cin * k * k, cout, cin, k, k);
    c.scale = add_vec(e, bn + ".weight", PK_BN_SCALE, cout, cout);
    c.shift = add_vec(e, bn + ".bias", PK_VEC, cout, cout);
    e->convs[name] = c;
}
// conv with a bias
void bias_conv(Engine* e, const std::string& name, int cout, int cin, int k) {
    ConvW c; c.cout = c.flop_cout = cout; c.cin = c.flop_cin = cin; c.k = k;
    c.w = add_mat(e, name + ".weight", PK_CONV_W, cout, cin * k * k, cout, cin, k, k);
    c.scale = kOnes;
    c.shift = add_vec(e, name + ".bias", PK_VEC, cout, cout);
    e->convs[name] = c;
}
// fully connected layer `name` (n outputs) as a 1x1 conv whose matrix has n + n2 rows padded to a multiple of 4 (the padding rows
// stay zero); `name2` fills rows [n, n + n2) (the fused heads: objectness + box deltas, class scores + box deltas)
void fc_rows(Engine* e, const std::string& key, const std::string& name, int n, int cin, const std::string& name2 = "", int n2 = 0) {
    const int rows = (int)align_up((size_t)(n + n2), 4);
    ConvW c; c.cout = rows; c.flop_cout = n + n2; c.cin = c.flop_cin = cin;
    c.w = add_mat(e, name + ".weight", PK_ROWS_W, rows, cin, n, cin, 0, 0);
    c.scale = kOnes;
    c.shift = add_vec(e, name + ".bias", PK_VEC, rows, n);
    if (n2) {
        ParamSlot s = e->params[name + ".weight"];
        s.d0 = n2; s.row_off = n;
        e->params[name2 + ".weight"] = s;
        add_vec(e, name2 + ".bias", PK_VEC, 0, n2, n, c.shift);
    }
    e->convs[key] = c;
}

void build_param_table(Engine* e) {
    const dt_engine_config& c = e->cfg;
    const Family& f = e->fam;
    const int NC = c.num_classes;
    e->vec_floats += 2048;      // kOnes
    if (!f.c4) { e->zeros = e->vec_floats; e->vec_floats += 2048; }
    {   // stem: the window layout [64][224] of conv_build_stem (pack_stem_window_kernel)
        ConvW s; s.cout = s.flop_cout = 64; s.cin = s.flop_cin = 147;
        s.w = add_mat(e, "model.conv1.weight", PK_STEM_W, 64, 224, 64, 147, 0, 0);
        s.scale = add_vec(e, "model.bn1.weight", PK_BN_SCALE, 64, 64);
        s.shift = add_vec(e, "model.bn1.bias", PK_VEC, 64, 64);
        e->convs["stem"] = s;
    }
    int inpl = 64;
    for (int li = 1; li <= 4; ++li) {       // all four layers: the C4 family runs layer4 as its RoI heads
        const int planes = 64 << (li - 1);
        for (int b = 0; b < c.arch_blocks[li - 1]; ++b) {
            const std::string p = "model.layer" + std::to_string(li) + "." + std::to_string(b) + ".";
            bn_conv(e, p + "conv1", p + "bn1", planes, inpl, 1);
            bn_conv(e, p + "conv2", p + "bn2", planes, planes, 3);
            bn_conv(e, p + "conv3", p + "bn3", planes * 4, planes, 1);
            if (b == 0) bn_conv(e, p + "downsample.0", p + "downsample.1", planes * 4, inpl, 1);
            inpl = planes * 4;
        }
    }
    if (!f.c4) {
        const int cins[4] = {256, 512, 1024, 2048};
        for (int i = 0; i < 4; ++i) {
            bias_conv(e, "conv_body.fpn_lateral." + std::to_string(i), 256, cins[i], 1);
            bias_conv(e, "conv_body.fpn_output." + std::to_string(i), 256, 256, 3);
        }
    }
    if (c.use_rpn) {
        bias_conv(e, "rpn.conv_rpn", f.rpn_ch, f.rpn_ch, 3);
        fc_rows(e, "rpn.head", "rpn.rpn_cls_prob", f.anchors, f.rpn_ch, "rpn.rpn_bbox_pred", 4 * f.anchors);
    }
    if (!f.c4) {
        ConvW c6; c6.cout = c6.flop_cout = 1024; c6.cin = c6.flop_cin = 256 * 49;
        c6.w = add_mat(e, "conv_head.fc6.weight", PK_FC6_W, 1024, 256 * 49, 1024, 256, 49, 0);
        c6.scale = kOnes; c6.shift = add_vec(e, "conv_head.fc6.bias", PK_VEC, 1024, 1024);
        e->convs["fc6"] = c6;
        fc_rows(e, "fc7", "conv_head.fc7", 1024, 1024);
    }
    fc_rows(e, "head", "classif_head", NC, f.box_feat, "bbox_head", 4 * NC);
    if (c.use_mask) {
        if (!f.c4)
            for (int i = 1; i <= 4; ++i) bias_conv(e, "mask_head.conv_head.fcn" + std::to_string(i), 256, 256, 3);
        ConvW d; d.cout = d.flop_cout = 256; d.cin = d.flop_cin = f.mask_in;
        d.w = add_mat(e, "mask_head.transposed_conv.weight", PK_DECONV_W, 4 * 256, f.mask_in, f.mask_in, 256, 0, 0);
        d.scale = kOnes; d.shift = add_vec(e, "mask_head.transposed_conv.bias", PK_VEC, 256, 256);
        e->convs["deconv"] = d;
        fc_rows(e, "mask_logits", "mask_head.classif_logits", NC, 256);
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

// the buffers of ResNet layer li (add_layer) over N maps whose output is h x w, named pre + "b<block>.t1" / ".t2" / ".out"
void plan_layer(Engine* e, const std::string& pre, int li, long long N, int h, int w) {
    const int planes = 64 << (li - 1);
    for (int b = 0; b < e->cfg.arch_blocks[li - 1]; ++b) {
        const std::string p = pre + "b" + std::to_string(b);
        add_buf(e, p + ".t1", {N, h, w, planes});
        add_buf(e, p + ".t2", {N, h, w, planes});
        add_buf(e, p + ".out", {N, h, w, planes * 4});
    }
}
std::string layer_out(const Engine* e, const std::string& pre, int li) { return pre + "b" + std::to_string(e->cfg.arch_blocks[li - 1] - 1) + ".out"; }

void plan_buffers(Engine* e) {
    const dt_engine_config& c = e->cfg;
    const Family& f = e->fam;
    const int B = c.batch;
    e->H1 = conv_out(c.height, 7, 2, 3); e->W1 = conv_out(c.width, 7, 2, 3);
    e->H2 = conv_out(e->H1, 3, 2, 1); e->W2 = conv_out(e->W1, 3, 2, 1);
    e->Hp = std::max(c.height + 6, 2 * e->H1 + 5); e->Wp = std::max(c.width + 6, 2 * e->W1 + 6);
    add_buf(e, "stem_x4", {B, e->Hp, e->Wp, 4});
    add_buf(e, "c1", {B, e->H1, e->W1, 64});
    add_buf(e, "pool", {B, e->H2, e->W2, 64});
    int h = e->H2, w = e->W2;
    for (int li = 1; li <= (f.c4 ? 3 : 4); ++li) {
        if (li > 1) { h = conv_out(h, 1, 2, 0); w = conv_out(w, 1, 2, 0); }
        e->LH[li - 1] = h; e->LW[li - 1] = w;
        const std::string pre = "l" + std::to_string(li);
        plan_layer(e, pre, li, B, h, w);
        e->bufs["C" + std::to_string(li + 1)] = e->bufs[layer_out(e, pre, li)];
    }
    if (!f.c4) {
        e->LH[4] = (e->LH[3] - 1) / 2 + 1; e->LW[4] = (e->LW[3] - 1) / 2 + 1;    // max_pool2d(k=1,s=2)
        for (int i = 0; i < 4; ++i) {
            add_buf(e, "inner" + std::to_string(i + 2), {B, e->LH[i], e->LW[i], 256});
            add_buf(e, "P" + std::to_string(i + 2), {B, e->LH[i], e->LW[i], 256});
        }
        add_buf(e, "P6", {B, e->LH[4], e->LW[4], 256});
    }
    const int L = f.rpn_levels, pre = c.pre_nms_top_n, post = c.post_nms_top_n;
    if (c.use_rpn) {       // Fast R-CNN (eval_fast*.ipynb) has no RPN: the caller fills `rois` / `roi_levels` / `roi_counts`
        long long anchors_total = 0, anchors_max = 0;
        for (int l = f.lv_min; l < f.lv_min + L; ++l) {
            add_buf(e, "rpn_t" + std::to_string(l), {B, e->LH[l - 2], e->LW[l - 2], f.rpn_ch});
            add_buf(e, "rpn_out" + std::to_string(l), {B, e->LH[l - 2], e->LW[l - 2], e->convs["rpn.head"].cout});
            anchors_total += (long long)e->LH[l - 2] * e->LW[l - 2] * f.anchors;
            anchors_max = std::max(anchors_max, (long long)e->LH[l - 2] * e->LW[l - 2] * f.anchors);
        }
        add_buf(e, "rpn_k0", {B, anchors_total}, 1); add_buf(e, "rpn_k1", {B, anchors_total}, 1);
        add_buf(e, "rpn_v0", {B, anchors_total}, 1); add_buf(e, "rpn_v1", {B, anchors_total}, 1);
        add_buf(e, "rpn_cand", {B, L, pre, 4}); add_buf(e, "rpn_cand_score", {B, L, pre});
        add_buf(e, "rpn_order", {B, L, pre}, 1);
        add_buf(e, "rpn_sel_hist", {B, L, 2, 2048}, 1); add_buf(e, "rpn_sel_cc", {B, L, (anchors_max + kRpnChunk - 1) / kRpnChunk}, 1); add_buf(e, "rpn_sel_info", {B, L, 4}, 1);
        add_buf(e, "rpn_cand_counts", {B, L}, 1); add_buf(e, "rpn_nms_mask", {B, L, pre, (pre + 63) / 64, 2}, 1);
        add_buf(e, "props", {B, L, post, 4}); add_buf(e, "prop_scores", {B, L, post}); add_buf(e, "prop_counts", {B, L}, 1);
        add_buf(e, "col_k0", {B, L * post}, 1); add_buf(e, "col_k1", {B, L * post}, 1);
        add_buf(e, "col_v0", {B, L * post}, 1); add_buf(e, "col_v1", {B, L * post}, 1);
    }
    add_buf(e, "rois", {B, post, 5}); add_buf(e, "roi_levels", {B, post}, 1); add_buf(e, "roi_counts", {B}, 1);
    const long long R = (long long)B * post;
    add_buf(e, "roi_feat", {R, f.box_pool.res, f.box_pool.res, f.box_pool.ch});
    if (f.c4) {
        plan_layer(e, "r5", 4, R, 7, 7);
        add_buf(e, "pooled", {R, 2048});
    } else {
        add_buf(e, "fc6", {R, 1024}); add_buf(e, "fc7", {R, 1024});
    }
    const int NC = c.num_classes;
    add_buf(e, "head", {R, e->convs["head"].cout});
    add_buf(e, "cls_prob", {R, NC}); add_buf(e, "bbox_pred", {R, 4 * NC});
    // detection
    const int cap = c.det_cap;
    add_buf(e, "det_flag", {B, NC, post}, 2, 1);
    add_buf(e, "det_dec", {B, NC, post, 4}); add_buf(e, "det_cls_counts", {B, NC}, 1);
    add_buf(e, "det_k0", {B, (long long)NC * post}, 1); add_buf(e, "det_k1", {B, (long long)NC * post}, 1);
    add_buf(e, "det_v0", {B, (long long)NC * post}, 1); add_buf(e, "det_v1", {B, (long long)NC * post}, 1);
    add_buf(e, "det_boxes", {B, cap, 4}); add_buf(e, "det_scores", {B, cap}); add_buf(e, "det_classes", {B, cap}, 1);
    add_buf(e, "det_roi_idx", {B, cap}, 1); add_buf(e, "det_counts", {B}, 1);
    add_buf(e, "range_flag", {1}, 1);     // raised by a kind::f16 conv when an activation does not fit fp16
    // per-image (net_h, net_w, scaling_factor, orig_h, orig_w), read when dt_engine_use_image_info is on (FPN only)
    if (!f.c4) add_buf(e, "im_info", {B, 5});
    if (c.use_mask) {
        const long long D = (long long)B * cap;
        const int M = f.mask_res;
        add_buf(e, "mask_rois", {D, 5}); add_buf(e, "mask_levels", {D}, 1);
        add_buf(e, "mask_feat", {D, 14, 14, f.mask_pool.ch});
        if (f.c4) plan_layer(e, "m5", 4, D, 7, 7);
        else
            for (int i = 1; i <= 4; ++i) add_buf(e, "mask_c" + std::to_string(i), {D, 14, 14, 256});
        add_buf(e, "mask_up", {D, M, M, 256});
        add_buf(e, "mask_logits", {D, M, M, e->convs["mask_logits"].cout});
        add_buf(e, "masks", {D, M, M});
        add_buf(e, "masks_full", {D, NC, M, M});
    }
    // Fast R-CNN on the FPN body: each image's pre-computed proposals in original-image coordinates, which the ST_COLLECT op scales,
    // deduplicates and maps to levels into rois / roi_levels / roi_counts (Engine.set_proposals).  Last, so no other offset moves.
    if (!f.c4 && !c.use_rpn) { add_buf(e, "fast_props", {B, post, 4}); add_buf(e, "fast_prop_counts", {B}, 1); }
    // the reference's detection count per image, which exceeds det_counts when ties at the top-max_dets threshold overflow det_cap
    add_buf(e, "det_total", {B}, 1);
}

// ---- program -----------------------------------------------------------------------------------
enum Stage { ST_TRUNK = 0, ST_FPN = 1, ST_RPN = 2, ST_PROPOSALS = 3, ST_COLLECT = 4, ST_ROI_BOX = 5, ST_BOX_HEAD = 6, ST_DETECT = 7,
             ST_MASK_ROIS = 8, ST_MASK_ROI_FEAT = 9, ST_MASK_HEAD = 10, ST_MASK_OUT = 11, ST_COUNT = 12 };

// the optional parts of a conv launch (ProgBuilder::conv); a call site sets the fields it uses
struct ConvOpt {
    int res_mode = RES_NONE;
    const float* res = nullptr;                             // RES_TILE: added before the ReLU (the output's geometry)
    const float* up = nullptr; int up_h = 0, up_w = 0;      // RES_UPSAMPLE2X: the coarser map, upsampled 2x and added
    int sigmoid_ch = 0;                                     // output channels [0, sigmoid_ch) get a sigmoid (RPN objectness)
    size_t w_off = 0;                                       // float offset of the weight sub-matrix (a deconv quadrant)
    int out_h = 0, out_w = 0, out_step = 0, out_y0 = 0, out_x0 = 0;   // output remap (transposed conv, see ConvSpec)
    int tap0 = 0, ntaps = 0;                                // K-split: only filter taps [tap0, tap0 + ntaps)
    bool zero_shift = false;                                // add no shift (the other half of the K-split adds it)
    bool planes_in = false, planes_out = false;             // fp16 hi/lo plane hand-over (kind::f16 only, see add_layer)
};

// one convolution of the program: the weights of layer `w` over x [N, H, W] (xstride floats per pixel) into y (ystride floats per pixel)
struct ConvCall {
    std::string w;
    const float* x; int N, H, W, xstride;
    float* y; int ystride, pad, stride;
    bool relu;
    ConvOpt o;
};

struct ProgBuilder {
    Engine* e;
    bool ok = true;
    int img_stride = 0;     // > 0: the following convs write image-shaped maps at this stride (masked per image when the table is on)

    // the ConvSpec of c; its weight matrix / scale vector go to slot `slot` of op, its FLOPs are added to op's
    bool spec(const ConvCall& k, Op& op, int slot, ConvSpec& s) {
        const ConvW& c = e->convs[k.w];
        const ConvOpt& o = k.o;
        memset(&s, 0, sizeof(s));
        s.x = k.x; s.N = k.N; s.H = k.H; s.W = k.W; s.Cin = c.cin; s.x_pix_stride = k.xstride;
        s.Cout = c.cout; s.kh = c.k; s.kw = c.k; s.pad = k.pad; s.stride = k.stride;
        s.shift = e->wvec(o.zero_shift ? e->zeros : c.shift);
        s.tap0 = o.tap0; s.ntaps = o.ntaps;
        if (e->cfg.conv_kind == 0) {
            // kind::f16 three-term product: fp16 halves of w * multiplier(matrix); the multiplier is undone through a per-op scale vector
            const size_t n16 = align_up((size_t)c.cout, 64);
            op.matrix[slot] = e->matrix_of(c.w + o.w_off);
            if (op.matrix[slot] < 0 || e->scale16_used + n16 > Engine::kScale16Floats) {
                fprintf(stderr, "[detectorch_b200] engine: scale16 arena / matrix lookup failed for %s\n", k.w.c_str());
                return false;
            }
            op.scale_src[slot] = e->wvec(c.scale); op.scale16[slot] = e->scale16_arena() + e->scale16_used; op.scale_n[slot] = c.cout;
            e->scale16_used += n16;
            s.kind = KIND_F16X3;
            s.w_hi = e->whi16(c.w + o.w_off); s.w_lo = e->wlo16(c.w + o.w_off);
            s.scale = op.scale16[slot];
            s.range_flag = e->buf<int>("range_flag");
        } else {
            s.kind = KIND_TF32X3;
            s.w_hi = e->wmat(c.w + o.w_off); s.w_lo = e->wlo(c.w + o.w_off);
            s.scale = e->wvec(c.scale);
        }
        s.y = k.y; s.y_pix_stride = k.ystride;
        const int Ho = conv_out(k.H, c.k, k.stride, k.pad), Wo = conv_out(k.W, c.k, k.stride, k.pad);
        // fp16 hi/lo plane hand-over (kind::f16 only): the fp32 buffer of N*H*W*C floats holds the two fp16 planes back to back
        if (o.planes_in) s.x_lo = reinterpret_cast<const __half*>(k.x) + (size_t)k.N * k.H * k.W * c.cin;
        if (o.planes_out) s.y_lo = reinterpret_cast<__half*>(k.y) + (size_t)k.N * Ho * Wo * c.cout;
        s.out_h = o.out_h; s.out_w = o.out_w; s.out_step = o.out_step; s.out_y0 = o.out_y0; s.out_x0 = o.out_x0;
        s.residual = o.res; s.res_pix_stride = c.cout; s.up_src = o.up; s.up_h = o.up_h; s.up_w = o.up_w;
        s.res_mode = o.res_mode; s.relu = k.relu ? 1 : 0; s.sigmoid_ch = o.sigmoid_ch; s.passes = e->cfg.passes;
        s.im_stride = img_stride;
        op.flops += 2.0 * (double)k.N * Ho * Wo * c.flop_cout * c.flop_cin * (o.ntaps > 0 ? o.ntaps : c.k * c.k);
        return true;
    }
    // one launch of c, or with phase1: one launch of c whose residual is phase1's result (RES_STAGED; c's own residual options are not
    // used).  When the two need different tile shapes, phase 1 runs as a launch of its own into c's output, which c then adds in place
    // (RES_TILE on its own output, tile by tile).
    void conv(int stage, const ConvCall& c, const ConvCall* phase1 = nullptr) {
        Op op;
        op.stage = stage; op.kind = 0; op.fn = -1;
        ConvSpec s, s1;
        if (!spec(c, op, 0, s) || (phase1 && !spec(*phase1, op, 1, s1))) { ok = false; return; }
        if (phase1) {
            s.res_mode = RES_STAGED; s.phase1 = &s1;
            if (!conv_staged_ok(s)) {
                ConvCall p1 = *phase1;
                p1.y = c.y; p1.ystride = c.ystride;
                conv(stage, p1);
                ConvCall p2 = c;
                p2.o.res_mode = RES_TILE; p2.o.res = c.y;
                conv(stage, p2);
                return;
            }
        }
        if (!conv_build(s, &op.conv)) { ok = false; fprintf(stderr, "[detectorch_b200] engine: conv_build failed for %s\n", c.w.c_str()); }
        e->ops.push_back(op);
    }
    void conv(int stage, const std::string& wname, const float* x, int N, int H, int W, int xstride, float* y, int ystride, int kpad,
              int stride, bool relu, const ConvOpt& o = ConvOpt()) {
        conv(stage, ConvCall{wname, x, N, H, W, xstride, y, ystride, kpad, stride, relu, o});
    }
    void fn(int stage, StageFn f) {
        Op op;
        op.stage = stage; op.kind = 1;
        op.fn = (int)e->fns.size();
        e->fns.push_back(f);
        e->ops.push_back(op);
    }
};

cudaError_t fn_stem_pack(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->Hp * e->Wp;
    stem_pack_nhwc4_kernel<<<grid_for(n), 256, 0, s>>>(e->image, e->cfg.batch, e->cfg.height, e->cfg.width, e->Hp, e->Wp, e->buf("stem_x4"), e->im_info());
    return cudaGetLastError();
}
cudaError_t fn_stem_pack_planes(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->Hp * e->Wp;
    uint2* xh = reinterpret_cast<uint2*>(e->buf("stem_x4"));
    stem_pack_nhwc4_planes_kernel<<<grid_for(n), 256, 0, s>>>(e->image, e->cfg.batch, e->cfg.height, e->cfg.width, e->Hp, e->Wp, xh, xh + n,
                                                             e->buf<int>("range_flag"), e->im_info());
    return cudaGetLastError();
}
cudaError_t fn_maxpool(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->H2 * e->W2 * 16;
    maxpool3x3s2_nhwc_kernel<<<grid_for(n), 256, 0, s>>>(e->buf("c1"), e->cfg.batch, e->H1, e->W1, 64, e->H2, e->W2, e->buf("pool"), e->im_info());
    return cudaGetLastError();
}

cudaError_t fn_p6(Engine* e, cudaStream_t s) {
    const long long n = (long long)e->cfg.batch * e->LH[4] * e->LW[4] * 64;
    subsample2_nhwc_kernel<<<grid_for(n), 256, 0, s>>>(e->buf("P5"), e->cfg.batch, e->LH[3], e->LW[3], 256, e->LH[4], e->LW[4], e->buf("P6"));
    return cudaGetLastError();
}
// Proposal generation: the keys / two-level radix select / ordered compaction of every (level, image) run at full-GPU width
// (rpn_select_*_kernel, one CTA per 4096 anchors), then one CTA per (level, image) sorts the ~1000 selected candidates, decodes, clips
// and filters them; the NMS runs as the suppression bit-matrix on every SM (nms_mask_kernel) and a survivor walk per (level, image).
cudaError_t fn_proposals(Engine* e, cudaStream_t s) {
    RpnParams& P = e->rpn;
    const int levels = P.num_levels;
    P.scaling_factor = e->scaling_factor;
    P.im_info = e->im_info();
    cudaError_t err = cudaMemsetAsync(P.sel_hist, 0, (size_t)e->cfg.batch * levels * 4096 * sizeof(uint32_t), s);
    if (err != cudaSuccess) return err;
    const dim3 grid(P.sel_chunks, levels, e->cfg.batch);
    rpn_select_keys_kernel<<<grid, 1024, 0, s>>>(P);
    rpn_select_hist2_kernel<<<grid, 1024, 0, s>>>(P);
    rpn_select_count_kernel<<<grid, 1024, 0, s>>>(P);
    rpn_select_scatter_kernel<<<grid, 1024, 0, s>>>(P);
    rpn_proposals_kernel<<<dim3(levels, e->cfg.batch), 1024, 0, s>>>(P);
    if (P.nms_thresh > 0.f) {
        nms_mask_kernel<<<dim3(P.nms_chunks, P.nms_chunks, levels * e->cfg.batch), 64, 0, s>>>(P.cand, P.cand_counts, P.pre_nms, P.nms_chunks,
                                                                                            P.nms_thresh, P.nms_mask);
        rpn_nms_scan_kernel<<<dim3(levels, e->cfg.batch), 1024, 0, s>>>(P);
    }
    return cudaGetLastError();
}
cudaError_t fn_collect(Engine* e, cudaStream_t s) {
    collect_kernel<<<e->cfg.batch, 1024, 0, s>>>(e->col);
    return cudaGetLastError();
}
cudaError_t fn_fast_props(Engine* e, cudaStream_t s) {
    FastPropsParams P;
    P.boxes = e->buf("fast_props"); P.counts = e->buf<int>("fast_prop_counts");
    P.im_info = e->im_info(); P.scaling_factor = e->scaling_factor;
    P.top_n = e->cfg.post_nms_top_n; P.k_min = e->fam.lv_min; P.k_max = e->fam.lv_max;
    P.rois = e->buf("rois"); P.levels = e->buf<int>("roi_levels"); P.roi_counts = e->buf<int>("roi_counts");
    fast_props_kernel<<<e->cfg.batch, 1024, (size_t)P.top_n * 9, s>>>(P);
    return cudaGetLastError();
}
// per-image counts: padded rows carry zero boxes (collect_kernel) -> harmless, fully defined output
cudaError_t roi_align(Engine* e, const RoiPool& a, cudaStream_t s) {
    e->roi_lv.im_info = e->im_info();
    const int* levels = a.levels ? e->buf<int>(a.levels) : nullptr;
    const int grid = std::min(a.n, num_sms() * 64);
    if (a.fast)
        roi_align_fast_nhwc_kernel<<<grid, 256, 0, s>>>(e->roi_lv, e->buf(a.rois), levels, a.n, a.ch, a.res, a.res, e->buf(a.out));
    else
        roi_align_nhwc_kernel<<<grid, 256, 0, s>>>(e->roi_lv, e->buf(a.rois), levels, nullptr, a.n, a.ch, a.res, a.res, a.sampling, e->buf(a.out));
    return cudaGetLastError();
}
cudaError_t fn_roi_box(Engine* e, cudaStream_t s) { return roi_align(e, e->fam.box_pool, s); }
cudaError_t fn_mask_roi_feat(Engine* e, cudaStream_t s) { return roi_align(e, e->fam.mask_pool, s); }
cudaError_t fn_avgpool(Engine* e, cudaStream_t s) {
    const int R = e->cfg.batch * e->cfg.post_nms_top_n;
    avgpool_nhwc_kernel<<<grid_for((long long)R * 512), 256, 0, s>>>(e->buf(layer_out(e, "r5", 4)), R, 49, 2048, e->buf("pooled"));
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
    e->det.im_info = e->im_info();
    det_class_kernel<<<dim3(e->cfg.num_classes - 1, e->cfg.batch), 256, 0, s>>>(e->det);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    det_limit_kernel<<<e->cfg.batch, 1024, 0, s>>>(e->det);
    return cudaGetLastError();
}
cudaError_t fn_mask_rois(Engine* e, cudaStream_t s) {
    const int n = e->cfg.batch * e->cfg.det_cap;
    mask_rois_kernel<<<(n + 255) / 256, 256, 0, s>>>(e->buf("det_boxes"), e->buf<int>("det_counts"), e->cfg.batch, e->cfg.det_cap, e->scaling_factor,
                                                    e->fam.lv_min, e->fam.lv_max, e->buf("mask_rois"), e->buf<int>("mask_levels"), e->im_info());
    return cudaGetLastError();
}
cudaError_t fn_mask_out(Engine* e, cudaStream_t s) {
    const int D = e->cfg.batch * e->cfg.det_cap, NC = e->cfg.num_classes, M = e->fam.mask_res;
    mask_select_kernel<<<grid_for((long long)D * M * M), 256, 0, s>>>(e->buf("mask_logits"), e->buf<int>("det_classes"), D, M, (int)align_up((size_t)NC, 4), NC,
                                                                    e->cfg.output_prob, e->buf("masks"), e->cfg.emit_full_masks ? e->buf("masks_full") : nullptr);
    return cudaGetLastError();
}

// generate_anchors.py:54-122 on the host (float64, np.round == rint half-to-even): ratio-major, size-minor rows
void gen_anchors(double stride, const double* sizes, int nsizes, float* out) {
    const double ratios[3] = {0.5, 1.0, 2.0};
    const double cx = 0.5 * (stride - 1), area = stride * stride;
    int row = 0;
    for (int r = 0; r < 3; ++r) {
        const double wr = nearbyint(sqrt(area / ratios[r]));
        const double hr = nearbyint(wr * ratios[r]);
        for (int s = 0; s < nsizes; ++s, ++row) {
            const double sc = sizes[s] / stride, ws = wr * sc, hs = hr * sc;
            out[row * 4 + 0] = (float)(cx - 0.5 * (ws - 1)); out[row * 4 + 1] = (float)(cx - 0.5 * (hs - 1));
            out[row * 4 + 2] = (float)(cx + 0.5 * (ws - 1)); out[row * 4 + 3] = (float)(cx + 0.5 * (hs - 1));
        }
    }
}

// the stem (detector.py:170-172): the fused-window conv over the packed image.  f16: the packed image arrives as two fp16 planes and
// the stem runs the kind::f16 product (the stem's converter warps -- 7 k-blocks of fp32 -> fp16 splits per 64-wide tile -- were what
// bounded it); else 3xTF32 from the fp32 image and weights.
void add_stem(ProgBuilder& pb, bool f16) {
    Engine* e = pb.e;
    const dt_engine_config& c = e->cfg;
    const int B = c.batch;
    const ConvW& sw = e->convs["stem"];
    Op op;
    op.stage = ST_TRUNK; op.kind = 0; op.fn = -1;
    op.flops = 2.0 * (double)B * e->H1 * e->W1 * sw.flop_cout * sw.flop_cin;
    bool ok;
    if (f16) {
        op.matrix[0] = e->matrix_of(sw.w);
        op.scale_src[0] = e->wvec(sw.scale); op.scale16[0] = e->scale16_arena() + e->scale16_used; op.scale_n[0] = 64;
        e->scale16_used += 64;
        ok = conv_build_stem(e->buf("stem_x4"), B, e->Hp, e->Wp, e->H1, e->W1, e->whi16(sw.w), e->wlo16(sw.w), op.scale16[0], e->wvec(sw.shift),
                             e->buf("c1"), c.passes, &op.conv, KIND_F16X3, e->buf<int>("range_flag"));
    } else {
        ok = conv_build_stem(e->buf("stem_x4"), B, e->Hp, e->Wp, e->H1, e->W1, e->wmat(sw.w), e->wlo(sw.w), e->wvec(sw.scale), e->wvec(sw.shift),
                             e->buf("c1"), c.passes, &op.conv);
    }
    if (!ok) { pb.ok = false; fprintf(stderr, "[detectorch_b200] engine: conv_build_stem failed\n"); return; }
    pb.fn(ST_TRUNK, f16 ? fn_stem_pack_planes : fn_stem_pack);
    op.conv.p.im_stride = 2;        // c1 is an image-shaped map at stride 2 (masked per image when the table is on)
    e->ops.push_back(op);
}

// ResNet layer li (detector.py:183; the C4 res5 head: detector.py:136,191,217) over N maps of h x w, into the buffers
// plan_layer(pre) made: bottlenecks 1x1 -> 3x3 -> 1x1 + identity (downsample in the first block, which has stride 2 unless li == 1).
// handover: conv1 -> conv2 -> conv3 inside each block hand fp16 planes over (kind::f16 only).  Returns the output map and leaves its
// size in h, w.
const float* add_layer(ProgBuilder& pb, int stage, const std::string& pre, int li, const float* x, int N, int& h, int& w, bool handover) {
    Engine* e = pb.e;
    const int planes = 64 << (li - 1);
    for (int b = 0; b < e->cfg.arch_blocks[li - 1]; ++b) {
        const std::string p = pre + "b" + std::to_string(b);
        const std::string wp = "model.layer" + std::to_string(li) + "." + std::to_string(b) + ".";
        const int stride = (b == 0 && li > 1) ? 2 : 1, cin = e->convs[wp + "conv1"].cin;
        const int ho = conv_out(h, 1, stride, 0), wo = conv_out(w, 1, stride, 0);
        // conv1 -> conv2 hand-over as fp16 hi/lo planes: the 3x3 conv would otherwise re-convert every input element once per filter tap
        // (the converter warps' fp32->fp16 packs are what bounds the 64/128-wide layers)
        ConvOpt o1; o1.planes_out = handover;
        pb.conv(stage, wp + "conv1", x, N, h, w, cin, e->buf(p + ".t1"), planes, 0, stride, true, o1);
        // conv2 -> conv3 the same way: conv3 is a 1x1 conv, so this saves one conversion per element, the converter warps' shared-memory
        // round trip (16 KB read + 16 KB written per k-block) and their issue slots in the epilogue-bound conv3
        ConvOpt o2; o2.planes_in = handover; o2.planes_out = handover;
        pb.conv(stage, wp + "conv2", e->buf(p + ".t1"), N, ho, wo, planes, e->buf(p + ".t2"), planes, 1, 1, true, o2);
        ConvOpt o3; o3.planes_in = handover;
        const ConvCall c3{wp + "conv3", e->buf(p + ".t2"), N, ho, wo, planes, e->buf(p + ".out"), planes * 4, 0, 1, true, o3};
        if (b == 0) {
            // the downsample is conv3's phase 1: its result stays on chip as conv3's residual
            const ConvCall ds{wp + "downsample.0", x, N, h, w, cin, e->buf(p + ".out"), planes * 4, 0, stride, false, ConvOpt()};
            pb.conv(stage, c3, &ds);
        } else {
            ConvCall c3r = c3;
            c3r.o.res_mode = RES_TILE; c3r.o.res = x;
            pb.conv(stage, c3r);
        }
        x = e->buf(p + ".out");
        h = ho; w = wo;
    }
    return x;
}

// FPN (detector.py:35-52): 1x1 laterals top-down, each adding the coarser one upsampled 2x, then the 3x3 outputs and P6
void add_fpn(ProgBuilder& pb) {
    Engine* e = pb.e;
    const int B = e->cfg.batch;
    const int cins[4] = {256, 512, 1024, 2048};
    for (int i = 3; i >= 0; --i) {
        pb.img_stride = 4 << i;
        ConvOpt o;
        if (i < 3) { o.res_mode = RES_UPSAMPLE2X; o.up = e->buf("inner" + std::to_string(i + 3)); o.up_h = e->LH[i + 1]; o.up_w = e->LW[i + 1]; }
        pb.conv(ST_FPN, "conv_body.fpn_lateral." + std::to_string(i), e->buf("C" + std::to_string(i + 2)), B, e->LH[i], e->LW[i], cins[i],
                e->buf("inner" + std::to_string(i + 2)), 256, 0, 1, false, o);
    }
    for (int i = 0; i < 4; ++i) {
        pb.img_stride = 4 << i;
        pb.conv(ST_FPN, "conv_body.fpn_output." + std::to_string(i), e->buf("inner" + std::to_string(i + 2)), B, e->LH[i], e->LW[i], 256,
                e->buf("P" + std::to_string(i + 2)), 256, 1, 1, false);
    }
    pb.fn(ST_FPN, fn_p6);
}

// RPN head on every RPN level (detector.py:251), the proposals (generate_proposals.py) and collect (collect_and_distribute...py;
// for one level it only formats the RoIs as [batch,x1,y1,x2,y2] rows, the scores being already descending)
void add_rpn(ProgBuilder& pb) {
    Engine* e = pb.e;
    const dt_engine_config& c = e->cfg;
    const Family& f = e->fam;
    const int B = c.batch, A = f.anchors, rows = e->convs["rpn.head"].cout;
    for (int l = f.lv_min; l < f.lv_min + f.rpn_levels; ++l) {
        const std::string L = std::to_string(l);
        pb.img_stride = 1 << l;
        pb.conv(ST_RPN, "rpn.conv_rpn", e->buf(f.feat + L), B, e->LH[l - 2], e->LW[l - 2], f.rpn_ch, e->buf("rpn_t" + L), f.rpn_ch, 1, 1, true);
        ConvOpt o; o.sigmoid_ch = A;
        pb.conv(ST_RPN, "rpn.head", e->buf("rpn_t" + L), B, e->LH[l - 2], e->LW[l - 2], f.rpn_ch, e->buf("rpn_out" + L), rows, 0, 1, false, o);
    }
    RpnParams& P = e->rpn;
    memset(&P, 0, sizeof(P));
    P.num_levels = f.rpn_levels; P.B = B;
    P.pre_nms = c.pre_nms_top_n; P.post_nms = c.post_nms_top_n;
    P.nms_thresh = c.rpn_nms_thresh; P.min_size = c.rpn_min_size; P.scaling_factor = 1.f;
    P.im_h = (float)c.height; P.im_w = (float)c.width;
    long long off = 0;
    for (int i = 0; i < f.rpn_levels; ++i) {
        const int l = f.lv_min + i;
        RpnLevel& lv = P.lv[i];
        lv.rpn_out = e->buf("rpn_out" + std::to_string(l));
        lv.H = e->LH[l - 2]; lv.W = e->LW[l - 2]; lv.A = A; lv.ch_stride = rows;
        lv.stride = (float)(1 << l);
        double sizes[5];        // A / 3 anchor sizes, doubling from 32 << i
        for (int s = 0; s < A / 3; ++s) sizes[s] = (double)(32 << (i + s));
        gen_anchors((double)(1 << l), sizes, A / 3, lv.anchors);
        lv.n = lv.H * lv.W * A;
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
    P.sel_chunks = e->bufs["rpn_sel_cc"].dims[2];
    P.cand_counts = e->buf<int>("rpn_cand_counts"); P.nms_mask = e->buf<unsigned long long>("rpn_nms_mask"); P.nms_chunks = (c.pre_nms_top_n + 63) / 64;
    pb.fn(ST_PROPOSALS, fn_proposals);
    CollectParams& C = e->col;
    memset(&C, 0, sizeof(C));
    C.props = P.out_props; C.scores = P.out_scores; C.counts = P.out_counts;
    C.B = B; C.L = f.rpn_levels; C.post_nms = c.post_nms_top_n; C.top_n = c.post_nms_top_n; C.k_min = f.lv_min; C.k_max = f.lv_max;
    C.k0 = e->buf<uint32_t>("col_k0"); C.k1 = e->buf<uint32_t>("col_k1"); C.v0 = e->buf<int>("col_v0"); C.v1 = e->buf<int>("col_v1");
    C.rois = e->buf("rois"); C.levels = e->buf<int>("roi_levels"); C.roi_counts = e->buf<int>("roi_counts");
    pb.fn(ST_COLLECT, fn_collect);
}

// detection post-processing (result_utils.py:76-168)
void setup_detect(Engine* e) {
    const dt_engine_config& c = e->cfg;
    DetParams& D = e->det;
    memset(&D, 0, sizeof(D));
    D.rois = e->buf("rois"); D.roi_counts = e->buf<int>("roi_counts"); D.cls = e->buf("cls_prob"); D.bbox = e->buf("bbox_pred");
    D.B = c.batch; D.R = c.post_nms_top_n; D.NC = c.num_classes;
    D.wx = 10.f; D.wy = 10.f; D.ww = 5.f; D.wh = 5.f;
    D.score_thresh = c.score_thresh; D.nms_thresh = c.det_nms_thresh; D.max_dets = c.max_dets; D.out_cap = c.det_cap;
    D.keep_flag = e->buf<unsigned char>("det_flag"); D.dec_box = e->buf<float4>("det_dec"); D.cls_counts = e->buf<int>("det_cls_counts");
    D.k0 = e->buf<uint32_t>("det_k0"); D.k1 = e->buf<uint32_t>("det_k1"); D.v0 = e->buf<int>("det_v0"); D.v1 = e->buf<int>("det_v1");
    D.out_boxes = e->buf("det_boxes"); D.out_scores = e->buf("det_scores"); D.out_classes = e->buf<int>("det_classes");
    D.out_roi_idx = e->buf<int>("det_roi_idx"); D.out_counts = e->buf<int>("det_counts"); D.out_total = e->buf<int>("det_total");
}

// mask head (detector.py:99-112): RoIs from the detections, their 14x14 features, the FPN 4-conv tower or the C4 'upshare' head
// (layer4 again, on the detections: detector.py:217-218), then the 2x deconv and the per-class logits
void add_mask_head(ProgBuilder& pb) {
    Engine* e = pb.e;
    const dt_engine_config& c = e->cfg;
    const Family& f = e->fam;
    const int D = c.batch * c.det_cap, M = f.mask_res;
    pb.fn(ST_MASK_ROIS, fn_mask_rois);
    pb.fn(ST_MASK_ROI_FEAT, fn_mask_roi_feat);
    const float* mx = e->buf("mask_feat");
    if (f.c4) {
        int h = 14, w = 14;
        mx = add_layer(pb, ST_MASK_HEAD, "m5", 4, mx, D, h, w, false);
    } else {
        // The mask logits carry the tightest parity bar (1e-4 absolute) and sit behind four K = 2304 convolutions, where the tensor
        // core's truncating fp32 accumulate is the error floor.  The chains are shortened by SPLITTING K: each 3x3 convolution runs
        // filter taps [0,5) as phase 1 and [5,9) as phase 2 of one launch; phase 2's epilogue adds phase 1's fp32 result
        // (round-to-nearest) before the ReLU.
        for (int i = 1; i <= 4; ++i) {
            const std::string wn = "mask_head.conv_head.fcn" + std::to_string(i);
            float* my = e->buf("mask_c" + std::to_string(i));
            ConvOpt lo; lo.ntaps = 5;
            ConvOpt hi; hi.tap0 = 5; hi.ntaps = 4; hi.zero_shift = true;
            const ConvCall first{wn, mx, D, 14, 14, 256, my, 256, 1, 1, false, lo};
            pb.conv(ST_MASK_HEAD, ConvCall{wn, mx, D, 14, 14, 256, my, 256, 1, 1, true, hi}, &first);
            mx = my;
        }
    }
    for (int ij = 0; ij < 4; ++ij) {     // ConvTranspose2d(2, stride 2) == 4 GEMMs scattered on the 2x grid
        ConvOpt o;
        o.w_off = (size_t)ij * 256 * f.mask_in;
        o.out_h = o.out_w = M; o.out_step = 2; o.out_y0 = ij / 2; o.out_x0 = ij % 2;
        pb.conv(ST_MASK_HEAD, "deconv", mx, D, M / 2, M / 2, f.mask_in, e->buf("mask_up"), 256, 0, 1, true, o);
    }
    pb.conv(ST_MASK_HEAD, "mask_logits", e->buf("mask_up"), D, M, M, 256, e->buf("mask_logits"), e->convs["mask_logits"].cout, 0, 1, false);
    pb.fn(ST_MASK_OUT, fn_mask_out);
}

bool build_program(Engine* e) {
    const dt_engine_config& c = e->cfg;
    const Family& f = e->fam;
    const int B = c.batch;
    ProgBuilder pb{e};
    // ---- trunk (detector.py:170-183): to layer4 for FPN, to layer3 for C4 (which runs layer4 per RoI).  The C4 family always builds
    // the fused stem from the fp32 weights and hands no fp16 planes over.
    const bool f16_planes = !f.c4 && c.conv_kind == 0;
    add_stem(pb, f16_planes);
    pb.fn(ST_TRUNK, fn_maxpool);
    const float* x = e->buf("pool");
    int h = e->H2, w = e->W2;
    for (int li = 1; li <= (f.c4 ? 3 : 4); ++li) {
        pb.img_stride = 4 << (li - 1);
        x = add_layer(pb, ST_TRUNK, "l" + std::to_string(li), li, x, B, h, w, f16_planes);
    }
    if (!f.c4) add_fpn(pb);
    if (c.use_rpn) add_rpn(pb);
    else if (!f.c4) pb.fn(ST_COLLECT, fn_fast_props);      // forward() fills the RoIs itself and skips this stage
    pb.img_stride = 0;      // everything below is RoI-shaped
    // ---- RoIAlign in collected order (detector.py:259-270)
    e->roi_lv.num_levels = f.lv_max - f.lv_min + 1;
    for (int l = f.lv_min; l <= f.lv_max; ++l) {
        const int i = l - f.lv_min;
        e->roi_lv.feat[i] = e->buf(f.feat + std::to_string(l));
        e->roi_lv.H[i] = e->LH[l - 2]; e->roi_lv.W[i] = e->LW[l - 2];
        e->roi_lv.scale[i] = 1.f / (float)(1 << l);
        e->roi_lv.stride[i] = 1 << l;
    }
    pb.fn(ST_ROI_BOX, fn_roi_box);
    // ---- box head (detector.py:61-64,277-284; C4: the res5 head, detector.py:136,191,273)
    const int R = B * c.post_nms_top_n;
    if (f.c4) {
        int rh = 14, rw = 14;
        add_layer(pb, ST_BOX_HEAD, "r5", 4, e->buf("roi_feat"), R, rh, rw, false);
        pb.fn(ST_BOX_HEAD, fn_avgpool);
    } else {
        pb.conv(ST_BOX_HEAD, "fc6", e->buf("roi_feat"), 1, 1, R, 49 * 256, e->buf("fc6"), 1024, 0, 1, true);
        pb.conv(ST_BOX_HEAD, "fc7", e->buf("fc6"), 1, 1, R, 1024, e->buf("fc7"), 1024, 0, 1, true);
    }
    pb.conv(ST_BOX_HEAD, "head", e->buf(f.c4 ? "pooled" : "fc7"), 1, 1, R, f.box_feat, e->buf("head"), e->convs["head"].cout, 0, 1, false);
    pb.fn(ST_BOX_HEAD, fn_softmax);
    setup_detect(e);
    pb.fn(ST_DETECT, fn_detect);
    if (c.use_mask) add_mask_head(pb);
    return pb.ok;
}

int load_param(Engine* e, const std::string& name, const float* src, long long numel, cudaStream_t st) {
    auto it = e->params.find(name);
    if (it == e->params.end()) return 2;   // not a hot-path parameter (running stats, fc, duplicates): ignored
    ParamSlot& s = it->second;
    if (!e->wbase) { fprintf(stderr, "[detectorch_b200] engine: bind weights before loading parameters\n"); return 0; }
    const long long expect = param_numel(s);
    if (expect != numel) {
        fprintf(stderr, "[detectorch_b200] engine: parameter %s has %lld elements, expected %lld\n", name.c_str(), numel, expect);
        return 0;
    }
    switch (s.kind) {
        case PK_CONV_W: pack_conv_w_kernel<<<grid_for(numel), 256, 0, st>>>(src, s.d0, s.d1, s.d2, s.d3, e->wmat(s.off)); break;
        case PK_STEM_W: pack_stem_window_kernel<<<(64 * 224 + 255) / 256, 256, 0, st>>>(src, e->wmat(s.off)); break;
        case PK_FC6_W: pack_fc6_kernel<<<grid_for(numel), 256, 0, st>>>(src, s.d0, s.d1, s.d2, e->wmat(s.off)); break;
        case PK_ROWS_W: copy_kernel<<<grid_for(numel), 256, 0, st>>>(src, numel, e->wmat(s.off) + (size_t)s.row_off * s.Kout); break;
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
    e->fam = family_of(e->cfg);
    build_param_table(e);
    plan_buffers(e);
    return e;
}

void dt_engine_destroy(dt_engine_t h) { delete reinterpret_cast<Engine*>(h); }

int64_t dt_engine_weight_bytes(dt_engine_t h) {
    Engine* e = reinterpret_cast<Engine*>(h);
    return (int64_t)e->weight_bytes();
}
int64_t dt_engine_workspace_bytes(dt_engine_t h) { return (int64_t)reinterpret_cast<Engine*>(h)->ws_bytes; }

// the image-shaped conv launches read the table (or not) -- the other kernels take e->im_info() when they are launched
static void apply_image_info(Engine* e) {
    for (Op& op : e->ops)
        if (op.kind == 0 && op.conv.p.im_stride > 0) op.conv.p.im_info = e->im_info();
}

static int bind_impl(Engine* e, void* weights, void* workspace, cudaStream_t st, bool fresh) {
    e->wbase = reinterpret_cast<float*>(weights);
    e->ws = reinterpret_cast<uint8_t*>(workspace);
    if (fresh) {
        DT_CHECK_CUDA(cudaMemsetAsync(weights, 0, (2 * e->mat_floats + e->vec_floats) * sizeof(float), st));
        // the shared all-ones scale vector sits at the start of the vector region
        fill_kernel<<<8, 256, 0, st>>>(e->wvec(kOnes), 2048, 1.f);
        DT_CHECK_CUDA(cudaGetLastError());
    }
    e->ops.clear();
    e->scale16_used = 0;
    e->fns.clear();
    if (!build_program(e)) return 0;
    apply_image_info(e);
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
            for (int m = 0; m < 2; ++m)
                if (op.kind == 0 && op.scale16[m])
                    scale16_kernel<<<(op.scale_n[m] + 255) / 256, 256, 0, st>>>(op.scale_src[m], e->matinfo() + op.matrix[m], op.scale16[m], op.scale_n[m]);
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
    *numel = param_numel(it->second);
    return 1;
}

int dt_engine_set_original_size(dt_engine_t h, float orig_h, float orig_w) {
    Engine* e = reinterpret_cast<Engine*>(h);
    e->orig_h = orig_h; e->orig_w = orig_w;
    return 1;
}

int dt_engine_use_image_info(dt_engine_t h, int enabled) {
    Engine* e = reinterpret_cast<Engine*>(h);
    if (enabled && (e->cfg.model_type != 0 || e->bufs.find("im_info") == e->bufs.end())) {
        fprintf(stderr, "[detectorch_b200] engine: per-image sizes are built for the FPN engine only\n");
        return 0;
    }
    e->use_image_info = enabled != 0;
    apply_image_info(e);
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

// The proposals of the last run (FPN engine with the RPN, run through ST_COLLECT): boxes [batch, post_nms_top_n, 4] in original-image
// coordinates and scores [batch, post_nms_top_n], zero past each image's roi_counts.  One launch on `stream`; graph-capturable.
int dt_engine_proposals(dt_engine_t h, float* boxes, float* scores, dt_stream_t stream) {
    Engine* e = reinterpret_cast<Engine*>(h);
    if (!e->bound || e->cfg.model_type != 0 || !e->cfg.use_rpn) {
        fprintf(stderr, "[detectorch_b200] engine: proposals are built for the FPN engine with the RPN\n");
        return 0;
    }
    if (!boxes || !scores || ((uintptr_t)boxes & 15)) { fprintf(stderr, "[detectorch_b200] engine: proposals: bad output pointer\n"); return 0; }
    collect_outputs_kernel<<<e->cfg.batch, 256, 0, (cudaStream_t)stream>>>(e->col, e->im_info(), e->scaling_factor, boxes, scores);
    DT_CHECK_CUDA(cudaGetLastError());
    return 1;
}

// number of kernel launches stages [first,last] issue (bench.py's gpu_launches)
int dt_engine_count_launches(dt_engine_t h, int first_stage, int last_stage) {
    Engine* e = reinterpret_cast<Engine*>(h);
    int n = 0;
    for (const Op& op : e->ops)
        if (op.stage >= first_stage && op.stage <= last_stage)
            n += (op.kind == 1 && e->fns[op.fn] == fn_detect) ? 2 : ((op.kind == 1 && op.stage == ST_PROPOSALS) ? (e->rpn.nms_thresh > 0.f ? 7 : 5) : 1);
    return n;
}

}  // extern "C"

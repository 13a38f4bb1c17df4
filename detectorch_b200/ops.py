"""Torch-tensor front-ends of the C-ABI operators.  Torch is only plumbing here (device memory,
current stream); all compute happens in detectorch_b200/csrc.  Every function requires CUDA
tensors -- there is no CPU path."""
import ctypes

import numpy as np
import torch

from . import _lib


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise TypeError("detectorch_b200 operators run on CUDA tensors only (no CPU fallback)")


def roi_align_forward_nchw(features, rois, pooled_height, pooled_width, spatial_scale, sampling_ratio, out=None):
    """features [B,C,H,W] fp32 contiguous, rois [R,4|5] -> [R,C,ph,pw].  Mirrors
    roialign.roi_align_forward_cuda of the reference (lib/model/roi_align.py:46-63)."""
    _need_cuda(features, rois)
    if features.dim() != 4 or rois.dim() != 2 or rois.size(1) not in (4, 5):
        raise RuntimeError("roi_align: features must be [B,C,H,W] and rois [R,4|5]")
    if not (features.is_contiguous() and rois.is_contiguous()):
        raise RuntimeError("roi_align: features and rois must be contiguous")   # reference AT_CHECK, roi_align_forward_cuda.cu:189
    if features.dtype != torch.float32 or rois.dtype != torch.float32:
        raise RuntimeError("roi_align: fp32 only")
    R, C = rois.size(0), features.size(1)
    if out is None:
        out = torch.empty((R, C, pooled_height, pooled_width), device=features.device, dtype=torch.float32)
    ok = _lib.lib().dt_roi_align_forward_nchw(_p(features), _p(rois), R, rois.size(1), C, features.size(2), features.size(3),
                                              int(pooled_height), int(pooled_width), float(spatial_scale), int(sampling_ratio),
                                              _p(out), _stream())
    _lib.check(ok, "dt_roi_align_forward_nchw")
    return out


def roi_align_backward_nchw(rois, grad_output, features_size, pooled_height, pooled_width, spatial_scale, sampling_ratio):
    """grad_output [R,C,ph,pw], rois [R,4|5] -> gradient w.r.t. the NCHW features [B,C,H,W] (lib/model/roi_align.py:91-147)."""
    _need_cuda(rois, grad_output)
    B, C, H, W = [int(v) for v in features_size]
    R = rois.size(0)
    if grad_output.dim() != 4 or grad_output.size(0) != R or grad_output.size(1) != C:
        raise RuntimeError("roi_align backward: grad_output must be [R,C,ph,pw]")
    grad_input = torch.zeros((B, C, H, W), device=grad_output.device, dtype=torch.float32)
    ok = _lib.lib().launch_roi_align_backward_cuda(int(grad_output.numel() & 0x7fffffff), _p(grad_output), R, float(spatial_scale), C, H, W,
                                                   int(pooled_height), int(pooled_width), int(sampling_ratio), _p(grad_input), _p(rois),
                                                   rois.size(1), _stream())
    _lib.check(ok, "launch_roi_align_backward_cuda")
    return grad_input


def roi_align_backward_nchw_deterministic(rois, grad_output, features_size, pooled_height, pooled_width, spatial_scale, sampling_ratio, grad_input=None):
    """Same contract as roi_align_backward_nchw, without atomics: every feature-map cell sums its contributions in the order of the
    reference's single-threaded CPU backward (lib/cppcuda/roi_align_backward_cpu.cpp:79-186), so the result is bit-identical to that loop
    and bit-reproducible run to run.  One host read (the contribution count: the sampling grid is adaptive when sampling_ratio == 0)."""
    _need_cuda(rois, grad_output)
    B, C, H, W = [int(v) for v in features_size]
    R = rois.size(0)
    if grad_output.dim() != 4 or grad_output.size(0) != R or grad_output.size(1) != C:
        raise RuntimeError("roi_align backward: grad_output must be [R,C,ph,pw]")
    rois, grad_output = rois.contiguous().float(), grad_output.contiguous().float()
    if grad_input is None:
        grad_input = torch.zeros((B, C, H, W), device=grad_output.device, dtype=torch.float32)
    if R == 0:
        return grad_input
    L = _lib.lib()
    dev = grad_output.device
    with torch.cuda.device(dev):
        scratch = torch.empty((L.dt_roi_align_backward_det_workspace_bytes(R, 0),), dtype=torch.uint8, device=dev)
        total = torch.zeros((1,), dtype=torch.int64, device=dev)
        _lib.check(L.dt_roi_align_backward_plan(_p(rois), R, rois.size(1), float(spatial_scale), int(pooled_height), int(pooled_width),
                                                int(sampling_ratio), _p(scratch), _p(total), _stream()), "dt_roi_align_backward_plan")
        m = int(total.item())
        ws = torch.empty((L.dt_roi_align_backward_det_workspace_bytes(R, m),), dtype=torch.uint8, device=dev)
        _lib.check(L.dt_roi_align_backward_deterministic(_p(grad_output), _p(rois), R, rois.size(1), B, C, H, W, int(pooled_height), int(pooled_width),
                                                         float(spatial_scale), int(sampling_ratio), m, _p(grad_input), _p(ws), _stream()),
                   "dt_roi_align_backward_deterministic")
    return grad_input


def roi_align_forward_nchw_fast(features, rois, pooled_height, pooled_width, spatial_scale, sampling_ratio, out=None):
    """Same contract as roi_align_forward_nchw; sampling_ratio == 2 takes the separable / FMA fast path (fp32 re-association
    differences only), anything else is forwarded to the exact kernel."""
    _need_cuda(features, rois)
    if not (features.is_contiguous() and rois.is_contiguous()):
        raise RuntimeError("roi_align: features and rois must be contiguous")
    B, C, H, W = features.shape
    R = rois.size(0)
    if out is None:
        out = torch.empty((R, C, pooled_height, pooled_width), device=features.device, dtype=torch.float32)
    L = _lib.lib()
    ws = torch.empty((L.dt_roi_align_fast_workspace_bytes(B, C, H, W, R, int(pooled_height), int(pooled_width)),), dtype=torch.uint8, device=features.device)
    ok = L.dt_roi_align_forward_nchw_fast(_p(features), B, _p(rois), R, rois.size(1), C, H, W, int(pooled_height), int(pooled_width),
                                          float(spatial_scale), int(sampling_ratio), _p(out), _p(ws), _stream())
    _lib.check(ok, "dt_roi_align_forward_nchw_fast")
    return out


def roi_align_forward_nhwc(feats, scales, rois, level, pooled_height, pooled_width, sampling_ratio, num_rois=None):
    """feats: list of NHWC maps [B,H,W,C]; rois [R,5]; level int32 [R] or None -> out [R,ph,pw,C]."""
    _need_cuda(rois, *feats)
    n = len(feats)
    ptrs = (ctypes.c_void_p * n)(*[f.data_ptr() for f in feats])
    hs = (ctypes.c_int * n)(*[f.size(1) for f in feats])
    ws = (ctypes.c_int * n)(*[f.size(2) for f in feats])
    sc = (ctypes.c_float * n)(*[float(s) for s in scales])
    C = feats[0].size(3)
    R = rois.size(0)
    out = torch.empty((R, pooled_height, pooled_width, C), device=rois.device, dtype=torch.float32)
    ok = _lib.lib().dt_roi_align_forward_nhwc(ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(hs, ctypes.c_void_p),
                                              ctypes.cast(ws, ctypes.c_void_p), ctypes.cast(sc, ctypes.c_void_p), n, _p(rois),
                                              _p(level), _p(num_rois), R, C, pooled_height, pooled_width, sampling_ratio, _p(out),
                                              _stream())
    _lib.check(ok, "dt_roi_align_forward_nhwc")
    return out


def nms(dets, thresh):
    """dets [N,5] fp32 CUDA (x1,y1,x2,y2,score) -> int64 CUDA tensor of ascending kept indices
    (the contract of lib/utils/boxes.py:332-336)."""
    _need_cuda(dets)
    n = dets.size(0)
    if n == 0:
        return torch.zeros((0,), dtype=torch.int64, device=dets.device)
    dets = dets.contiguous().float()
    L = _lib.lib()
    ws = torch.empty((L.dt_nms_workspace_bytes(n),), dtype=torch.uint8, device=dets.device)
    keep = torch.empty((n,), dtype=torch.int64, device=dets.device)
    cnt = torch.zeros((1,), dtype=torch.int32, device=dets.device)
    _lib.check(L.dt_nms(_p(dets), n, float(thresh), _p(keep), _p(cnt), _p(ws), _stream()), "dt_nms")
    return keep[:int(cnt.item())]


def _segm_grow_and_redo(run, runs_cap):
    """run(runs_cap) -> (the most runs a detection needed beyond runs_cap, or 0; result), redone with a larger runs_cap until it is 0."""
    while True:
        need, out = run(runs_cap)
        if need == 0:
            return out
        runs_cap = max(2 * runs_cap, need + 1)     # a detection needed more runs than provisioned: grow and redo


def _segm_batch_args(who, masks, classes, boxes, num_dets):
    """Checks a batch's masks [B,cap,M,M] or [B,cap,K,M,M] (with classes [B,cap]) and boxes [B,cap,4], and converts them and num_dets
    ([B], None = all cap slots) for the device: -> (B, cap, K, M, masks, classes, boxes, num_dets)."""
    if masks.dim() not in (4, 5) or boxes.dim() != 3 or boxes.size(2) != 4:
        raise ValueError("%s: masks must be [B,cap,M,M] or [B,cap,K,M,M] and boxes [B,cap,4]" % who)
    B, cap, M = masks.size(0), masks.size(1), masks.size(-1)
    if tuple(boxes.shape[:2]) != (B, cap) or masks.size(-2) != M:
        raise ValueError("%s: masks %s and boxes %s disagree" % (who, tuple(masks.shape), tuple(boxes.shape)))
    if (masks.dim() == 5) != (classes is not None) or (classes is not None and tuple(classes.shape) != (B, cap)):
        raise ValueError("%s: [B,cap,K,M,M] masks need classes [B,cap]; [B,cap,M,M] masks take none" % who)
    K = masks.size(2) if masks.dim() == 5 else 1
    masks, boxes = masks.contiguous().float(), boxes.contiguous().float()
    if classes is not None:
        classes = classes.contiguous().to(torch.int32)
    nd = torch.full((B,), cap, dtype=torch.int32, device=masks.device) if num_dets is None else num_dets.contiguous().to(torch.int32)
    return B, cap, K, M, masks, classes, boxes, nd


def segm_rle(masks, classes, boxes, im_h, im_w, thresh=0.5, expanded=False, num_dets=None, runs_cap=4096):
    """Mask paste + COCO RLE on the device (lib/utils/result_utils.py:170-228).
    masks [D,K,M,M] (classes int32 [D] selects the plane) or [D,M,M]; boxes [D,4] fp32 reference boxes, or int32 already
    expanded boxes when expanded=True.  Returns (counts list of uint32 arrays, strings list of bytes)."""
    _need_cuda(masks, boxes, classes)
    D = masks.size(0)
    if D == 0:
        return [], []
    masks = masks.contiguous().float()
    M = masks.size(-1)
    K = masks.size(1) if masks.dim() == 4 else 1
    boxes = boxes.contiguous()
    if expanded and boxes.dtype != torch.int32:
        raise TypeError("segm_rle: expanded boxes must be int32")
    if not expanded:
        boxes = boxes.float()
    if classes is not None:
        classes = classes.contiguous().to(torch.int32)
    L = _lib.lib()
    dev = masks.device

    def run(runs_cap):
        ws = torch.empty((L.dt_segm_workspace_bytes(D, runs_cap),), dtype=torch.uint8, device=dev)
        counts = torch.empty((D, runs_cap), dtype=torch.int32, device=dev)
        ncount = torch.empty((D,), dtype=torch.int32, device=dev)
        strings = torch.empty((L.dt_segm_strings_bytes(D, runs_cap),), dtype=torch.uint8, device=dev)
        offs = torch.empty((D + 1,), dtype=torch.int64, device=dev)
        over = torch.zeros((1,), dtype=torch.int32, device=dev)
        ok = L.dt_segm_rle(_p(masks), _p(classes), K, M, _p(None if expanded else boxes), _p(boxes if expanded else None), _p(num_dets), D,
                           int(im_h), int(im_w), float(thresh), _p(counts), _p(ncount), runs_cap, _p(strings), _p(offs), _p(over), _p(ws),
                           _stream())
        _lib.check(ok, "dt_segm_rle")
        return int(over.item()), (counts, ncount, strings, offs)

    counts, ncount, strings, offs = _segm_grow_and_redo(run, runs_cap)
    offs_h = offs.cpu().numpy()
    str_h = strings[:int(offs_h[-1])].cpu().numpy().tobytes()
    n_h = ncount.cpu().numpy()
    nmax = int(n_h.max()) if D else 0
    cnt_h = counts[:, :max(nmax, 1)].cpu().numpy().view("uint32")
    return [cnt_h[d, :n_h[d]].copy() for d in range(D)], [str_h[offs_h[d]:offs_h[d + 1]] for d in range(D)]


def to_host(*ts):
    """Device tensors -> numpy arrays of the same dtypes and shapes, through ONE device-to-host copy (and so one synchronisation)."""
    ts = [t.contiguous() for t in ts]
    flat = torch.cat([t.reshape(-1).view(torch.uint8) for t in ts]).cpu().numpy()
    out, o = [], 0
    for t in ts:
        n = t.numel() * t.element_size()
        out.append(flat[o:o + n].view(str(t.dtype).replace("torch.", "")).reshape(tuple(t.shape)))
        o += n
    return out


def segm_image_sizes(im_sizes, B):
    """Host (height, width) RLE canvas per image -> int64 numpy [B, 2]: int() of each value, as the notebooks pass int(h), int(w)."""
    v = im_sizes.detach().cpu().numpy() if torch.is_tensor(im_sizes) else np.asarray(im_sizes)
    if v.ndim != 2 or v.shape != (B, 2):
        raise ValueError("expected one (height, width) per image: shape [%d, 2], got %s" % (B, tuple(v.shape)))
    v = v.astype(np.float64)
    if not np.all(np.isfinite(v)):
        raise ValueError("image sizes must be finite")
    sz = np.array([[int(h), int(w)] for h, w in v], dtype=np.int64).reshape(B, 2)
    if np.any(sz < 1) or np.any(sz[:, 0] * sz[:, 1] >= 2 ** 32):
        raise ValueError("image sizes must be at least 1 x 1 and below 2^32 pixels")
    return sz


def segm_rle_batch_device(masks, classes, boxes, num_dets, im_sizes, thresh=0.5, runs_cap=4096, extra=()):
    """The launch half of segm_rle_batch: -> (packed strings on the device, host copies of [offsets int64 [B*cap+1], num_dets [B]] + the
    `extra` device tensors), all read in one synchronisation (after a grow-and-redo, one more per redo)."""
    _need_cuda(masks, classes, boxes, num_dets)
    B, cap, K, M, masks, classes, boxes, nd = _segm_batch_args("segm_rle_batch", masks, classes, boxes, num_dets)
    sz = segm_image_sizes(im_sizes, B)
    dev = masks.device
    if B * cap == 0:
        host = to_host(nd, *extra)
        return torch.empty((0,), dtype=torch.uint8, device=dev), [np.zeros((B * cap + 1,), np.int64)] + host
    sizes = torch.from_numpy(sz.astype(np.int32)).to(dev)
    L = _lib.lib()

    def run(runs_cap):
        ws = torch.empty((L.dt_segm_batch_workspace_bytes(B, cap, runs_cap),), dtype=torch.uint8, device=dev)
        strings = torch.empty((L.dt_segm_batch_strings_bytes(B, cap, runs_cap),), dtype=torch.uint8, device=dev)
        offs = torch.empty((B * cap + 1,), dtype=torch.int64, device=dev)
        over = torch.zeros((1,), dtype=torch.int32, device=dev)
        ok = L.dt_segm_rle_batch(_p(masks), _p(classes), K, M, _p(boxes), _p(nd), _p(sizes), B, cap, int(sz[:, 0].max()), int(sz[:, 1].max()),
                                 float(thresh), runs_cap, _p(strings), _p(offs), _p(over), _p(ws), _stream())
        _lib.check(ok, "dt_segm_rle_batch")
        host = to_host(offs, over, nd, *extra)
        return int(host[1][0]), (strings, [host[0], host[2]] + host[3:])

    return _segm_grow_and_redo(run, runs_cap)


SEGM_APPEND_MAX_SIDE = 8192     # DT_SEGM_APPEND_MAX_SIDE: the largest image side segm_rle_batch_append encodes


def segm_rle_batch_append(masks, classes, boxes, num_dets, im_sizes, arena, cursor, thresh=0.5, runs_cap=4096):
    """segm_rle_batch's strings appended to a device char arena, without reading anything back (capturable in a CUDA graph).
    masks, classes, boxes, num_dets: as for segm_rle_batch; im_sizes int32 [B,2] on the device; arena uint8 [capacity] (or None for
    capacity 0); cursor int64 [1] on the device, the arena's used length.  -> (offsets int64 [B*cap+1] into the arena, flags int32 [3]),
    both on the device: flags [0] the runs a slot needed beyond runs_cap, [1] an image size outside [1, SEGM_APPEND_MAX_SIDE], [2] the
    strings did not fit (cursor + offsets[-1] - offsets[0] > capacity).  With a flag raised, the arena and the cursor are untouched."""
    _need_cuda(masks, classes, boxes, num_dets, im_sizes, arena, cursor)
    B, cap, K, M, masks, classes, boxes, nd = _segm_batch_args("segm_rle_batch_append", masks, classes, boxes, num_dets)
    if tuple(im_sizes.shape) != (B, 2) or im_sizes.dtype != torch.int32 or cursor.dtype != torch.int64 or cursor.numel() != 1:
        raise ValueError("segm_rle_batch_append: im_sizes must be int32 [%d, 2] and cursor int64 [1]" % B)
    if arena is not None and (arena.dtype != torch.uint8 or arena.dim() != 1 or not arena.is_contiguous()):
        raise ValueError("segm_rle_batch_append: the arena must be a contiguous uint8 vector")
    dev = masks.device
    im_sizes = im_sizes.contiguous()
    offs = torch.empty((B * cap + 1,), dtype=torch.int64, device=dev)
    flags = torch.zeros((3,), dtype=torch.int32, device=dev)
    if B * cap == 0:
        offs.copy_(cursor.reshape(1))
        return offs, flags
    L = _lib.lib()
    ws = torch.empty((L.dt_segm_batch_workspace_bytes(B, cap, runs_cap),), dtype=torch.uint8, device=dev)
    _lib.check(L.dt_segm_rle_batch_append(_p(masks), _p(classes), K, M, _p(boxes), _p(nd), _p(im_sizes), B, cap, float(thresh), int(runs_cap),
                                          _p(arena), 0 if arena is None else arena.numel(), _p(cursor), _p(offs), _p(flags), _p(ws), _stream()),
               "dt_segm_rle_batch_append")
    return offs, flags


def segm_rle_batch(masks, classes, boxes, num_dets, im_sizes, thresh=0.5, runs_cap=4096):
    """Mask paste + COCO RLE of a batch of images on the device (lib/utils/result_utils.py:170-228 for every image at once).
    masks [B,cap,M,M] (the selected class, detect()'s 'masks') or [B,cap,K,M,M] with classes int32 [B,cap] selecting the plane;
    boxes [B,cap,4] fp32 image-space boxes; num_dets int32 [B] live slots per image (detect()'s 'counts'; None = all);
    im_sizes host [B,2] (height, width) of each image's RLE canvas.  -> per image, a list of RLE strings (bytes), one per live slot."""
    strings, (offs, nd) = segm_rle_batch_device(masks, classes, boxes, num_dets, im_sizes, thresh, runs_cap)
    cap = masks.size(1)
    str_h = strings[:int(offs[-1])].cpu().numpy().tobytes() if offs[-1] > 0 else b""
    return [[str_h[offs[b * cap + d]:offs[b * cap + d + 1]] for d in range(min(max(int(nd[b]), 0), cap))] for b in range(masks.size(0))]


def segm_paste(masks, classes, boxes, im_h, im_w, thresh=0.5, expanded=False, num_dets=None):
    """Pasted binary masks uint8 [D, im_h, im_w] (the im_mask of result_utils.py:203-217 for every detection)."""
    _need_cuda(masks, boxes, classes)
    D = masks.size(0)
    masks = masks.contiguous().float()
    M = masks.size(-1)
    K = masks.size(1) if masks.dim() == 4 else 1
    boxes = boxes.contiguous() if expanded else boxes.contiguous().float()
    if classes is not None:
        classes = classes.contiguous().to(torch.int32)
    out = torch.empty((D, int(im_h), int(im_w)), dtype=torch.uint8, device=masks.device)
    ok = _lib.lib().dt_segm_paste(_p(masks), _p(classes), K, M, _p(None if expanded else boxes), _p(boxes if expanded else None),
                                  _p(num_dets), D, int(im_h), int(im_w), float(thresh), _p(out), _stream())
    _lib.check(ok, "dt_segm_paste")
    return out


def tf32_residual(w):
    lo = torch.empty_like(w)
    _lib.check(_lib.lib().dt_tf32_residual(_p(w), _p(lo), w.numel(), _stream()), "dt_tf32_residual")
    return lo


def fp16_split(w, multiplier=1.0):
    """w fp32 -> (hi, lo) fp16 tensors of w * multiplier (multiplier must be a power of two)."""
    _need_cuda(w)
    hi = torch.empty(w.shape, dtype=torch.float16, device=w.device)
    lo = torch.empty_like(hi)
    _lib.check(_lib.lib().dt_fp16_split(_p(w.contiguous()), w.numel(), float(multiplier), _p(hi), _p(lo), _stream()), "dt_fp16_split")
    return hi, lo


def weight_multiplier(w):
    """Power of two that brings max|w| into [2^13, 2^14): the fp16 low half then stays a normal number for every weight
    within 2^-9 of the largest one."""
    m = float(w.abs().max())
    if not (m > 0.0):
        return 1.0
    import math
    return 2.0 ** (13 - math.floor(math.log2(m)))


def conv2d_nhwc(x, w_kmajor, scale, shift, kh, kw, pad, stride, w_lo=None, residual=None, up_src=None, relu=False, sigmoid_ch=0,
                passes=3, force_block_n=0, out=None, kind="tf32", range_flag=None):
    """x [N,H,W,Cin] fp32 (channels-last memory), w_kmajor [Cout, kh*kw*Cin] -> y [N,Ho,Wo,Cout].
    kind "tf32": 3xTF32 (w_lo = tf32 residual); kind "f16": 3xFP16 on the kind::f16 pipe (weights split here)."""
    _need_cuda(x, w_kmajor)
    N, H, W, Cin = x.shape
    Cout = w_kmajor.size(0)
    Ho = (H + 2 * pad - kh) // stride + 1
    Wo = (W + 2 * pad - kw) // stride + 1
    if out is None:
        out = torch.empty((N, Ho, Wo, Cout), device=x.device, dtype=torch.float32)
    res_mode = 1 if residual is not None else (2 if up_src is not None else 0)
    up_h = up_src.size(1) if up_src is not None else 0
    up_w = up_src.size(2) if up_src is not None else 0
    if kind == "f16":
        mult = weight_multiplier(w_kmajor)
        hi, lo = fp16_split(w_kmajor, mult)
        sc = (scale / mult).contiguous()
        ok = _lib.lib().dt_conv2d_nhwc_f16x3(_p(x), N, H, W, Cin, Cin, _p(hi), _p(lo), Cout, kh, kw, pad, stride, _p(sc), _p(shift), _p(residual),
                                             res_mode, _p(up_src), up_h, up_w, int(relu), int(sigmoid_ch), int(passes), int(force_block_n),
                                             _p(range_flag), _p(out), Cout, _stream())
        _lib.check(ok, "dt_conv2d_nhwc_f16x3")
        return out
    if w_lo is None:
        w_lo = tf32_residual(w_kmajor)
    ok = _lib.lib().dt_conv2d_nhwc(_p(x), N, H, W, Cin, Cin, _p(w_kmajor), _p(w_lo), Cout, kh, kw, pad, stride, _p(scale), _p(shift),
                                   _p(residual), res_mode, _p(up_src), up_h, up_w, int(relu), int(sigmoid_ch), int(passes),
                                   int(force_block_n), _p(out), Cout, _stream())
    _lib.check(ok, "dt_conv2d_nhwc")
    return out


class ConvOperand(ctypes.Structure):
    """dt_conv_operand of include/detectorch_b200.h"""
    _fields_ = [("x", ctypes.c_void_p), ("H", ctypes.c_int), ("W", ctypes.c_int), ("Cin", ctypes.c_int), ("w_hi", ctypes.c_void_p),
                ("w_lo", ctypes.c_void_p), ("kh", ctypes.c_int), ("kw", ctypes.c_int), ("pad", ctypes.c_int), ("stride", ctypes.c_int),
                ("tap0", ctypes.c_int), ("ntaps", ctypes.c_int), ("scale", ctypes.c_void_p), ("shift", ctypes.c_void_p)]


def conv2d_nhwc_two_phase(phase2, phase1=None, residual=None, relu=False, passes=3, force_block_n=0, out=None, kind="tf32", range_flag=None,
                          im_info=None, im_stride=0):
    """One launch of y = act(conv(phase2) + conv(phase1)), phase 1's fp32 result staying on chip as phase 2's residual: rounded exactly as
    phase 1 into a buffer, then phase 2 with residual=that buffer.  A phase is a dict: x [N,H,W,Cin] fp32, w [Cout, kh*kw*Cin],
    scale, shift [Cout], k (or kh, kw), pad, stride, and optionally the filter taps tap0, ntaps (0 = all).  phase1=None runs phase 2
    alone (+ residual).  im_info [N,5] with im_stride > 0 zeroes output pixels outside each image."""
    keep = []

    def operand(ph):
        x, w = ph["x"], ph["w"]
        _need_cuda(x, w)
        kh, kw = ph.get("kh", ph.get("k")), ph.get("kw", ph.get("k"))
        if kind == "f16":
            mult = weight_multiplier(w)
            hi, lo = fp16_split(w, mult)
            sc = (ph["scale"] / mult).contiguous()
        else:
            hi, lo, sc = w.contiguous(), tf32_residual(w.contiguous()), ph["scale"].contiguous()
        sh = ph["shift"].contiguous()
        x = x.contiguous()
        keep.extend([x, hi, lo, sc, sh])
        return ConvOperand(x.data_ptr(), x.size(1), x.size(2), x.size(3), hi.data_ptr(), lo.data_ptr(), kh, kw, ph["pad"], ph["stride"],
                           ph.get("tap0", 0), ph.get("ntaps", 0), sc.data_ptr(), sh.data_ptr())

    o2 = operand(phase2)
    o1 = operand(phase1) if phase1 is not None else None
    N, H, W, _ = phase2["x"].shape
    Cout = phase2["w"].size(0)
    Ho = (H + 2 * o2.pad - o2.kh) // o2.stride + 1
    Wo = (W + 2 * o2.pad - o2.kw) // o2.stride + 1
    if out is None:
        out = torch.empty((N, Ho, Wo, Cout), device=phase2["x"].device, dtype=torch.float32)
    ok = _lib.lib().dt_conv2d_nhwc_two_phase(1 if kind == "f16" else 0, ctypes.byref(o1) if o1 is not None else None, ctypes.byref(o2),
                                             _p(residual), N, Cout, int(relu), int(passes), int(force_block_n), _p(range_flag), _p(im_info),
                                             int(im_stride), _p(out), _stream())
    _lib.check(ok, "dt_conv2d_nhwc_two_phase")
    return out

"""
ORACLE -- test infrastructure only.  Never imported by the product path
(detectorch_b200/).  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this module.

CPU restatement of the reference's host-side hot-path logic (numpy where the
reference uses numpy, torch-CPU where the reference uses torch, so the fp32
results are bit-identical to the reference run on CPU):

  generate_anchors            lib/utils/generate_anchors.py:54-122
  generate_proposals_level    lib/model/generate_proposals.py:31-238
  nms                         lib/utils/boxes.py:332-336 -> lib/utils_cython/cython_nms.pyx:37-87
  map_rois_to_fpn_levels      lib/utils/multilevel_rois.py:41-53
  collect_and_distribute      lib/model/collect_and_distribute_fpn_rpn_proposals.py:84-128
  multilevel_rois_for_test    lib/utils/multilevel_rois.py:19-82
  bbox_transform / clip       lib/utils/boxes.py:150-208
  box_results_with_nms_and_limit / postprocess_output   lib/utils/result_utils.py:76-168
  roi_align_forward           lib/cppcuda_cffi/src/cpp/roi_align_cpu_loop.cpp:118-224 (oracle/roi_align_ref.c)
  expand_boxes / segm_results lib/utils/boxes.py:245-261, lib/utils/result_utils.py:170-228  (SURVEY 8f rank 1)
  resize_linear_f32           cv2.resize(float32, INTER_LINEAR) -- OpenCV's own (non-IPP) algorithm, modules/imgproc/src/resize.cpp
  rle_encode / rle_to_string  pycocotools maskApi.c rleEncode / rleToString (third-party, not installed here)
  prep_im_for_blob / im_list_to_blob   lib/utils/blob.py:27-87  (SURVEY 8f rank 3)

Parity pinned: tests/test_oracle.py checks every function here against (a) the
reference's own modules imported from /root/reference when that tree is
present (this container) and (b) the committed vectors in tests/golden/
generated from the reference by tests/golden/make_golden.py.
"""
import ctypes
import os
import subprocess

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None

BBOX_XFORM_CLIP = 4.135166556742356  # boxes.py:73 / generate_proposals.py:165


def build():
    """Compile the C restatement (oracle/liboracle.so) and, when /root/reference is
    present, the reference's own sources into oracle/_ref/ (build_ref.sh)."""
    subprocess.check_call(["make", "-s", "-C", _HERE])
    subprocess.check_call(["bash", os.path.join(_HERE, "build_ref.sh")], stdout=subprocess.DEVNULL)


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", _HERE])
        _lib = ctypes.CDLL(path)
        _lib.oracle_nms.restype = ctypes.c_int64
    return _lib


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ----------------------------------------------------------------------------- RoIAlign
def roi_align_forward(features, rois, pooled_h, pooled_w, spatial_scale, sampling_ratio):
    """features [B,C,H,W] fp32, rois [R,4|5] fp32 -> [R,C,ph,pw] fp32 (numpy)."""
    f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
    r = np.ascontiguousarray(np.asarray(rois, dtype=np.float32))
    B, C, H, W = f.shape
    R, cols = r.shape
    out = np.zeros((R, C, pooled_h, pooled_w), np.float32)
    lib().oracle_roi_align_forward(_fp(f), _fp(r), ctypes.c_int64(R), ctypes.c_int(cols),
                                   ctypes.c_int(C), ctypes.c_int(H), ctypes.c_int(W),
                                   ctypes.c_int(pooled_h), ctypes.c_int(pooled_w),
                                   ctypes.c_float(spatial_scale), ctypes.c_int(sampling_ratio), _fp(out))
    return out


def roi_align_forward_ref(features, rois, pooled_h, pooled_w, spatial_scale, sampling_ratio):
    """Same through the reference's own compiled loop (oracle/_ref/libroialign_ref.so)."""
    so = ctypes.CDLL(os.path.join(_HERE, "_ref", "libroialign_ref.so"))
    f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
    r = np.ascontiguousarray(np.asarray(rois, dtype=np.float32))
    B, C, H, W = f.shape
    R, cols = r.shape
    out = np.zeros((R, C, pooled_h, pooled_w), np.float32)
    so.roi_align_forward_loop(ctypes.c_int(out.size), _fp(f), _fp(r), ctypes.c_float(spatial_scale),
                              ctypes.c_int(C), ctypes.c_int(H), ctypes.c_int(W), ctypes.c_int(pooled_h),
                              ctypes.c_int(pooled_w), ctypes.c_int(sampling_ratio), ctypes.c_int(cols), _fp(out))
    return out


def roi_align_backward(top_diff, rois, features_shape, pooled_h, pooled_w, spatial_scale, sampling_ratio):
    """top_diff [R,C,ph,pw] fp32, rois [R,4|5] -> gradient w.r.t. the features [B,C,H,W] (numpy), the order of additions into every
    cell being that of the reference's single-threaded CPU loop (lib/cppcuda/roi_align_backward_cpu.cpp:79-186)."""
    t = np.ascontiguousarray(np.asarray(top_diff, dtype=np.float32))
    r = np.ascontiguousarray(np.asarray(rois, dtype=np.float32))
    B, C, H, W = [int(v) for v in features_shape]
    out = np.zeros((B, C, H, W), np.float32)
    lib().oracle_roi_align_backward(_fp(t), _fp(r), ctypes.c_int64(r.shape[0]), ctypes.c_int(r.shape[1]), ctypes.c_int(C), ctypes.c_int(H),
                                    ctypes.c_int(W), ctypes.c_int(pooled_h), ctypes.c_int(pooled_w), ctypes.c_float(spatial_scale),
                                    ctypes.c_int(sampling_ratio), _fp(out))
    return out


def roi_align_backward_ref(top_diff, rois, features_shape, pooled_h, pooled_w, spatial_scale, sampling_ratio):
    """Same through the reference's own loop template (oracle/_ref/libroialign_bwd_ref.so, cut out of roi_align_backward_cpu.cpp by build_ref.sh)."""
    so = ctypes.CDLL(os.path.join(_HERE, "_ref", "libroialign_bwd_ref.so"))
    t = np.ascontiguousarray(np.asarray(top_diff, dtype=np.float32))
    r = np.ascontiguousarray(np.asarray(rois, dtype=np.float32))
    B, C, H, W = [int(v) for v in features_shape]
    out = np.zeros((B, C, H, W), np.float32)
    so.roi_align_backward_loop_f32(ctypes.c_int(t.size), _fp(t), ctypes.c_int(r.shape[0]), ctypes.c_float(spatial_scale), ctypes.c_int(C), ctypes.c_int(H),
                                   ctypes.c_int(W), ctypes.c_int(pooled_h), ctypes.c_int(pooled_w), ctypes.c_int(sampling_ratio), _fp(out), _fp(r),
                                   ctypes.c_int(r.shape[1]))
    return out


# ----------------------------------------------------------------------------- NMS
def nms(dets, thresh, order="numpy"):
    """dets [N,5] fp32 (x1,y1,x2,y2,score) -> ascending original indices kept (int64).
    boxes.py:332-336: empty input returns [].
    order: the visiting order of tied scores.  "numpy" is the reference's own (pyx:45, numpy's unstable argsort reversed, which
    may differ between hosts and numpy builds); "stable" is (score desc, index asc), the order the device kernels document."""
    dets = np.ascontiguousarray(np.asarray(dets, dtype=np.float32))
    n = dets.shape[0]
    if n == 0:
        return np.zeros((0,), np.int64)
    if order == "numpy":
        order = dets[:, 4].argsort()[::-1]                                       # pyx:45
    elif order == "stable":
        order = np.argsort(-dets[:, 4], kind="stable")
    else:
        raise ValueError("nms: order must be 'numpy' or 'stable'")
    order = np.ascontiguousarray(order.astype(np.int64))
    keep = np.empty((n,), np.int64)
    k = lib().oracle_nms(_fp(dets), _fp(order), ctypes.c_int64(n), ctypes.c_float(thresh), _fp(keep))
    return keep[:k].copy()


# ----------------------------------------------------------------------------- anchors
def generate_anchors(stride=16, sizes=(32, 64, 128, 256, 512), aspect_ratios=(0.5, 1, 2)):
    """(A,4) float64 anchor table; rows ordered ratio-major, size-minor.
    generate_anchors.py:54-122 (ratio enumeration with np.round, then scales)."""
    base = float(stride)
    scales = np.asarray(sizes, dtype=np.float64) / stride
    ratios = np.asarray(aspect_ratios, dtype=np.float64)
    # reference window (0,0,base-1,base-1): w=h=base, centre (base-1)/2
    w0 = h0 = base
    cx = cy = 0.5 * (base - 1)
    rows = []
    area = w0 * h0
    for r in ratios:
        wr = np.round(np.sqrt(area / r))
        hr = np.round(wr * r)
        for s in scales:
            ws, hs = wr * s, hr * s
            rows.append([cx - 0.5 * (ws - 1), cy - 0.5 * (hs - 1), cx + 0.5 * (ws - 1), cy + 0.5 * (hs - 1)])
    return np.asarray(rows, dtype=np.float64)


def all_anchors(anchors, feat_h, feat_w, spatial_scale):
    """generate_proposals.py:124-149: shifted anchors in (H,W,A) order, float64."""
    stride = 1. / spatial_scale
    sx = np.arange(0, feat_w) * stride
    sy = np.arange(0, feat_h) * stride
    sx, sy = np.meshgrid(sx, sy)
    shifts = np.stack([sx.ravel(), sy.ravel(), sx.ravel(), sy.ravel()], axis=1)
    return (anchors[None, :, :] + shifts[:, None, :]).reshape(-1, 4)


# ----------------------------------------------------------------------------- proposals
def _decode_torch(boxes, deltas, weights=(1.0, 1.0, 1.0, 1.0)):
    """generate_proposals.py:165-214 (torch fp32 arithmetic, columns x1,y1,x2,y2)."""
    widths = boxes[:, 2] - boxes[:, 0] + 1.0
    heights = boxes[:, 3] - boxes[:, 1] + 1.0
    ctr_x = boxes[:, 0] + 0.5 * widths
    ctr_y = boxes[:, 1] + 0.5 * heights
    wx, wy, ww, wh = weights
    dx, dy = deltas[:, 0::4] / wx, deltas[:, 1::4] / wy
    dw, dh = deltas[:, 2::4] / ww, deltas[:, 3::4] / wh
    clip = torch.tensor([BBOX_XFORM_CLIP], dtype=torch.float32)
    dw, dh = torch.min(dw, clip), torch.min(dh, clip)
    pcx = dx * widths.unsqueeze(1) + ctr_x.unsqueeze(1)
    pcy = dy * heights.unsqueeze(1) + ctr_y.unsqueeze(1)
    pw = torch.exp(dw) * widths.unsqueeze(1)
    ph = torch.exp(dh) * heights.unsqueeze(1)
    return torch.cat((pcx - 0.5 * pw, pcy - 0.5 * ph, pcx + 0.5 * pw - 1, pcy + 0.5 * ph - 1), 1)


def generate_proposals_level(rpn_cls_prob, rpn_bbox_pred, im_h, im_w, scaling_factor, spatial_scale,
                             anchor_sizes, aspect_ratios=(0.5, 1, 2), pre_nms_top_n=6000, post_nms_top_n=1000,
                             nms_thresh=0.7, min_size=0, return_stages=False, tie_order="numpy"):
    """One image, one level.  rpn_cls_prob [1,A,H,W], rpn_bbox_pred [1,4A,H,W] (torch CPU fp32).
    generate_proposals.py:31-122.  Returns (proposals [n,4], scores [n,1]) torch fp32;
    with return_stages also a dict of the integer stages (order, filter keep, nms keep).
    tie_order: the order of equal scores in the top-k and in the NMS.  "numpy" is the reference's own (argpartition / argsort,
    unspecified among ties); "stable" is (score desc, anchor index asc), the order the device documents."""
    anchors = generate_anchors(stride=1. / spatial_scale, sizes=anchor_sizes, aspect_ratios=aspect_ratios)
    A = anchors.shape[0]
    H, W = rpn_cls_prob.shape[2], rpn_cls_prob.shape[3]
    anc_np = all_anchors(anchors, H, W, spatial_scale)
    anc = torch.FloatTensor(anc_np)                                               # :55 float64 -> fp32
    deltas = rpn_bbox_pred.squeeze(0).permute(1, 2, 0).contiguous().view(-1, 4)    # :64
    scores = rpn_cls_prob.squeeze(0).permute(1, 2, 0).contiguous().view(-1, 1)     # :72
    s_np = scores.numpy()
    if tie_order == "stable":
        order = np.argsort(-s_np.squeeze(1), kind="stable")
        if 0 < pre_nms_top_n < len(s_np):
            order = order[:pre_nms_top_n]
    elif tie_order != "numpy":
        raise ValueError("generate_proposals_level: tie_order must be 'numpy' or 'stable'")
    elif pre_nms_top_n <= 0 or pre_nms_top_n >= len(s_np):
        order = np.argsort(-s_np.squeeze())                                        # :78
    else:
        inds = np.argpartition(-s_np.squeeze(), pre_nms_top_n)[:pre_nms_top_n]      # :82-84
        order = inds[np.argsort(-s_np[inds].squeeze())]
    deltas, scores, anc = deltas[order, :], scores[order, :], anc[order, :]
    s_np = s_np[order, :]
    props = _decode_torch(anc, deltas)                                             # :96
    lim_w = torch.tensor([float(im_w)]) - 1
    lim_h = torch.tensor([float(im_h)]) - 1
    z = torch.tensor([0.0])
    props[:, 0::4] = torch.max(torch.min(props[:, 0::4], lim_w), z)                # :231-237
    props[:, 1::4] = torch.max(torch.min(props[:, 1::4], lim_h), z)
    props[:, 2::4] = torch.max(torch.min(props[:, 2::4], lim_w), z)
    props[:, 3::4] = torch.max(torch.min(props[:, 3::4], lim_h), z)
    p_np = props.numpy()
    ms = min_size * scaling_factor                                                 # :155
    ws = p_np[:, 2] - p_np[:, 0] + 1
    hs = p_np[:, 3] - p_np[:, 1] + 1
    xc = p_np[:, 0] + ws / 2.
    yc = p_np[:, 1] + hs / 2.
    fkeep = np.where((ws >= ms) & (hs >= ms) & (xc < im_w) & (yc < im_h))[0]        # :160-162
    props, scores = props[fkeep, :], scores[fkeep, :]
    p_np, s_np = p_np[fkeep, :], s_np[fkeep]
    nkeep = None
    if nms_thresh > 0:
        nkeep = nms(np.hstack((p_np, s_np)), nms_thresh, order=tie_order)          # :115
        if post_nms_top_n > 0:
            nkeep = nkeep[:post_nms_top_n]
        props, scores = props[nkeep, :], scores[nkeep, :]
    if return_stages:
        return props, scores, {"order": order, "filter_keep": fkeep, "nms_keep": nkeep}
    return props, scores


# ----------------------------------------------------------------------------- FPN level mapping
def boxes_area(boxes):
    return (boxes[:, 2] - boxes[:, 0] + 1) * (boxes[:, 3] - boxes[:, 1] + 1)        # boxes.py:75-81


def map_rois_to_fpn_levels(rois, k_min, k_max, s0=224, lvl0=4):
    """multilevel_rois.py:41-53 (numpy, dtype of `rois` preserved: fp32 in the detector)."""
    s = np.sqrt(boxes_area(rois))
    lv = np.floor(lvl0 + np.log2(s / s0 + 1e-6))
    return np.clip(lv, k_min, k_max)


def collect_and_distribute(roi_list, score_list, lvl_min=2, lvl_max=5, post_nms_top_n=1000, stable=False):
    """collect...py:84-128.  roi_list: per-level torch [n_l,4]; score_list: [n_l,1].
    Returns (per-level roi tensors, idx_restore int64 numpy, collected rois [n,4], lvls).
    stable: equal scores keep their concatenated (level, rank) order, as the device sorts them; the reference's torch.sort leaves
    that order unspecified."""
    rois = torch.cat(tuple(roi_list), 0)
    scores = torch.cat(tuple(score_list), 0).reshape(-1)
    _, inds = torch.sort(-scores, stable=stable)                                   # :102
    rois = rois[inds[:post_nms_top_n], :]
    lvls = map_rois_to_fpn_levels(rois.numpy(), lvl_min, lvl_max)
    order = np.empty((0,))
    per_level = []
    for lvl in range(lvl_min, lvl_max + 1):
        idx = np.where(lvls == lvl)[0]
        per_level.append(rois[idx, :])
        order = np.concatenate((order, idx))
    return per_level, np.argsort(order), rois, lvls


def multilevel_rois_for_test(rois, lvl_min=2, lvl_max=5):
    """multilevel_rois.py:19-82: numpy rois [n,4] -> (per-level arrays, idx_restore int32)."""
    lvls = map_rois_to_fpn_levels(rois, lvl_min, lvl_max)
    order = np.empty((0,))
    per_level = []
    for lvl in range(lvl_min, lvl_max + 1):
        idx = np.where(lvls == lvl)[0]
        per_level.append(rois[idx, :])
        order = np.concatenate((order, idx))
    return per_level, np.argsort(order).astype(np.int32)


# ----------------------------------------------------------------------------- detection post-processing
def bbox_transform(boxes, deltas, weights=(1.0, 1.0, 1.0, 1.0)):
    """boxes.py:168-208 (numpy)."""
    if boxes.shape[0] == 0:
        return np.zeros((0, deltas.shape[1]), dtype=deltas.dtype)
    boxes = boxes.astype(deltas.dtype, copy=False)
    w = boxes[:, 2] - boxes[:, 0] + 1.0
    h = boxes[:, 3] - boxes[:, 1] + 1.0
    cx = boxes[:, 0] + 0.5 * w
    cy = boxes[:, 1] + 0.5 * h
    wx, wy, ww, wh = weights
    dx, dy = deltas[:, 0::4] / wx, deltas[:, 1::4] / wy
    dw = np.minimum(deltas[:, 2::4] / ww, BBOX_XFORM_CLIP)
    dh = np.minimum(deltas[:, 3::4] / wh, BBOX_XFORM_CLIP)
    pcx = dx * w[:, None] + cx[:, None]
    pcy = dy * h[:, None] + cy[:, None]
    pw = np.exp(dw) * w[:, None]
    ph = np.exp(dh) * h[:, None]
    out = np.zeros(deltas.shape, dtype=deltas.dtype)
    out[:, 0::4] = pcx - 0.5 * pw
    out[:, 1::4] = pcy - 0.5 * ph
    out[:, 2::4] = pcx + 0.5 * pw - 1
    out[:, 3::4] = pcy + 0.5 * ph - 1
    return out


def clip_tiled_boxes(boxes, im_shape):
    """boxes.py:150-165."""
    boxes[:, 0::4] = np.maximum(np.minimum(boxes[:, 0::4], im_shape[1] - 1), 0)
    boxes[:, 1::4] = np.maximum(np.minimum(boxes[:, 1::4], im_shape[0] - 1), 0)
    boxes[:, 2::4] = np.maximum(np.minimum(boxes[:, 2::4], im_shape[1] - 1), 0)
    boxes[:, 3::4] = np.maximum(np.minimum(boxes[:, 3::4], im_shape[0] - 1), 0)
    return boxes


def _nms_and_limit(scores, boxes, num_classes, score_thresh, overlap_thresh, max_detections_per_img, tie_order):
    """result_utils.py:96-168 keeping track of the rows: (cls_boxes, cls_inds) with cls_inds[j] the RoI index of each row of
    cls_boxes[j], and the image threshold of the limit (None when it did not cut)."""
    cls_boxes = [[] for _ in range(num_classes)]
    cls_inds = [np.zeros((0,), np.int64) for _ in range(num_classes)]
    for j in range(1, num_classes):
        inds = np.where(scores[:, j] > score_thresh)[0]
        dets_j = np.hstack((boxes[inds, j * 4:(j + 1) * 4], scores[inds, j][:, None])).astype(np.float32, copy=False)
        keep = nms(dets_j, overlap_thresh, order=tie_order)
        cls_boxes[j] = dets_j[keep, :]
        cls_inds[j] = inds[keep]
    image_thresh = None
    if max_detections_per_img > 0:
        image_scores = np.hstack([cls_boxes[j][:, -1] for j in range(1, num_classes)])
        if len(image_scores) > max_detections_per_img:
            image_thresh = np.sort(image_scores)[-max_detections_per_img]
            for j in range(1, num_classes):
                k = np.where(cls_boxes[j][:, -1] >= image_thresh)[0]
                cls_boxes[j] = cls_boxes[j][k, :]
                cls_inds[j] = cls_inds[j][k]
    return cls_boxes, cls_inds, image_thresh


def box_results_with_nms_and_limit(scores, boxes, num_classes=81, score_thresh=0.05, overlap_thresh=0.5,
                                   max_detections_per_img=100, tie_order="numpy"):
    """result_utils.py:96-168 (hard-NMS branch; soft-NMS / voting are off by default).  tie_order: the NMS visiting order of tied
    scores (nms's `order`); the limit itself does not depend on it."""
    cls_boxes = _nms_and_limit(scores, boxes, num_classes, score_thresh, overlap_thresh, max_detections_per_img, tie_order)[0]
    im_results = np.vstack([cls_boxes[j] for j in range(1, num_classes)])
    return im_results[:, -1], im_results[:, :-1], cls_boxes


def detection_tail(case, b, tie_order="numpy", max_dets=100):
    """postprocess_output + box_results_with_nms_and_limit on image b of a teacher-forced detection case (the fields of
    tests/detect_tail_cases.Case: rois [B,R,5] at network scale, roi_counts [B], cls_prob [B*R,NC], bbox_pred [B*R,4NC], scale [B],
    orig_hw [B,2]).  Returns (classes, roi_idx, scores, boxes, image_thresh) in the reference's class-major, RoI-ascending order."""
    R, NC = case.rois.shape[1], case.cls_prob.shape[1]
    n = int(case.roi_counts[b])
    rois = case.rois[b, :n, 1:5].astype(np.float32)
    boxes = (rois / np.float32(case.scale[b])).astype(np.float32)                 # rois.div(scaling_factor) in fp32
    deltas = case.bbox_pred[b * R:b * R + n].astype(np.float32)
    im = np.asarray(case.orig_hw[b], np.float32)
    pred = clip_tiled_boxes(bbox_transform(boxes, deltas, (10.0, 10.0, 5.0, 5.0)), im)
    sc = case.cls_prob[b * R:b * R + n].astype(np.float32)
    cls_boxes, cls_inds, thresh = _nms_and_limit(sc, pred, NC, 0.05, 0.5, max_dets, tie_order)
    cls = np.concatenate([np.full(len(cls_inds[j]), j, np.int64) for j in range(1, NC)])
    dets = np.vstack([np.asarray(cls_boxes[j], np.float32).reshape(-1, 5) for j in range(1, NC)])
    return cls, np.concatenate(cls_inds[1:]), dets[:, 4], dets[:, :4], thresh


def expected_device(case, det_cap, max_dets=100, tie_order="stable"):
    """What the device detection tail writes for each image of `case` with det_cap output rows: the reference's detections with
    stable tie order (detection_tail(..., "stable")) and, when more than det_cap of them tie through the limit, the surplus
    removed from the end of those tied at the image threshold (class-major, RoI-ascending order).  Every detection scoring above
    the threshold is kept: there are fewer than max_dets <= det_cap of them.  Per image (classes, roi_idx, scores, boxes, total)
    with total the reference's own count."""
    out = []
    for b in range(case.rois.shape[0]):
        cls, idx, sc, bx, thresh = detection_tail(case, b, tie_order, max_dets)
        total = len(sc)
        if total > det_cap:
            assert thresh is not None, "more detections than det_cap without the limit"
            tied = np.flatnonzero(sc == thresh)
            drop = tied[len(tied) - (total - det_cap):]
            assert len(drop) == total - det_cap, "the surplus is not all tied at the image threshold"
            keep = np.setdiff1d(np.arange(total), drop)
            cls, idx, sc, bx = cls[keep], idx[keep], sc[keep], bx[keep]
        out.append((cls, idx, sc, bx, total))
    return out


def postprocess_output(rois, scaling_factor, im_size, class_scores, bbox_deltas, bbox_reg_weights=(10.0, 10.0, 5.0, 5.0)):
    """result_utils.py:76-94.  rois torch [R,4]; scaling_factor torch/float; im_size (h,w)."""
    sf = scaling_factor if torch.is_tensor(scaling_factor) else torch.tensor(float(scaling_factor))
    boxes = rois.div(sf).squeeze(0).numpy()
    deltas = bbox_deltas.numpy() if torch.is_tensor(bbox_deltas) else bbox_deltas
    im = np.asarray(im_size.numpy() if torch.is_tensor(im_size) else im_size).squeeze()
    pred = clip_tiled_boxes(bbox_transform(boxes, deltas, bbox_reg_weights), im)
    sc = class_scores.numpy() if torch.is_tensor(class_scores) else class_scores
    return box_results_with_nms_and_limit(sc, pred)


# ------------------------------------------------------------------------------------------------ mask paste + COCO RLE
# The step right after the hot path (SURVEY.md 8f rank 1): lib/utils/result_utils.py:170-228.  Two third-party pieces:
#  * cv2.resize(float32 30x30 -> (w, h), INTER_LINEAR).  OpenCV 4.13 is importable in the build container; with IPP switched
#    off (cv2.ipp.setUseIPP(False)) resize_linear_f32 below is BIT-IDENTICAL to it (tests/test_oracle.py, and the committed
#    golden vectors were produced by cv2 itself).  IPP-enabled builds use Intel's kernel, which differs by <= 1.6e-6 in value
#    and flips ~2e-7 of the thresholded pixels; OpenCV's own algorithm is the one restated.
#  * pycocotools.mask.encode (maskApi.c rleEncode + rleToString): NOT installed here and not vendored by the reference, so
#    the RLE string is "parity unpinned" against pycocotools; it is restated from the published algorithm and checked by a
#    decode round trip and hand-computed strings.
def resize_linear_f32(src, w, h):
    """OpenCV resize, CV_32F, INTER_LINEAR, 1 channel: horizontal pass then vertical pass, float coefficients
    (resize.cpp: resizeGeneric_ / HResizeLinear / VResizeLinear; coefficient set-up in cv::resize)."""
    f32 = np.float32
    src = np.ascontiguousarray(src, dtype=f32)
    sh, sw = src.shape
    if 2 * w == sw and 2 * h == sh:
        # cv::resize turns INTER_LINEAR into the "area fast" kernel when both scale factors are exactly 2: 2x2 box average,
        # 4-wide SIMD body (a+b)+(c+d), scalar tail ((a+b)+c)+d, times 0.25f (ResizeAreaFast_ / ResizeAreaFastVec_SIMD_32f)
        a, b, c, d = src[0::2, 0::2], src[0::2, 1::2], src[1::2, 0::2], src[1::2, 1::2]
        simd = (((a + b).astype(f32) + (c + d).astype(f32)).astype(f32) * f32(.25)).astype(f32)
        tail = ((((a + b).astype(f32) + c).astype(f32) + d).astype(f32) * f32(.25)).astype(f32)
        return np.where(np.arange(w)[None, :] < (w & ~3), simd, tail).astype(f32)

    def axis(dst, n):
        scale = 1.0 / (float(dst) / n)                                   # double, as in cv::resize
        f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(f32)
        s = np.floor(f).astype(np.int64)
        return s, (f - s.astype(f32)).astype(f32)

    sx, fx = axis(w, sw)
    sy, fy = axis(h, sh)
    lo = sx < 0                                                          # x: clamped cells get weight (1, 0)
    fx = np.where(lo, f32(0), fx); sx = np.where(lo, 0, sx)
    hi = sx >= sw - 1
    fx = np.where(hi, f32(0), fx); sx = np.where(hi, sw - 1, sx)
    a0, a1 = (f32(1) - fx).astype(f32), fx
    sx1 = np.minimum(sx + 1, sw - 1)
    hbuf = ((src[:, sx] * a0[None, :]).astype(f32) + (src[:, sx1] * a1[None, :]).astype(f32)).astype(f32)
    r0, r1 = np.clip(sy, 0, sh - 1), np.clip(sy + 1, 0, sh - 1)          # y: row indices are clipped, weights kept
    b0, b1 = (f32(1) - fy).astype(f32), fy
    return ((hbuf[r0, :] * b0[:, None]).astype(f32) + (hbuf[r1, :] * b1[:, None]).astype(f32)).astype(f32)


def expand_boxes(boxes, scale):
    """lib/utils/boxes.py:245-261 (fp32 arithmetic on fp32 boxes, result widened to float64)."""
    w_half = (boxes[:, 2] - boxes[:, 0]) * .5
    h_half = (boxes[:, 3] - boxes[:, 1]) * .5
    x_c = (boxes[:, 2] + boxes[:, 0]) * .5
    y_c = (boxes[:, 3] + boxes[:, 1]) * .5
    w_half *= scale
    h_half *= scale
    out = np.zeros(boxes.shape)
    out[:, 0] = x_c - w_half
    out[:, 2] = x_c + w_half
    out[:, 1] = y_c - h_half
    out[:, 3] = y_c + h_half
    return out


def rle_encode(mask):
    """maskApi.c rleEncode: run lengths of the column-major flattening, starting with the zeros run."""
    flat = np.asarray(mask, dtype=np.uint8).flatten(order='F')
    if flat.size == 0:
        return np.zeros((1,), np.uint32)
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    pos = np.concatenate([[0], change, [flat.size]])
    counts = np.diff(pos)
    if flat[0] != 0:
        counts = np.concatenate([[0], counts])
    return counts.astype(np.uint32)


def rle_to_string(counts):
    """maskApi.c rleToString: LEB128-like, 5 data bits + continuation bit per char, offset 48; counts[i>2] are
    delta-coded against counts[i-2]."""
    out = bytearray()
    cn = [int(c) for c in counts]
    for i, x in enumerate(cn):
        if i > 2:
            x -= cn[i - 2]
        more = True
        while more:
            c = x & 0x1f
            x >>= 5
            more = (x != -1) if (c & 0x10) else (x != 0)
            if more:
                c |= 0x20
            out.append(c + 48)
    return bytes(out)


def rle_from_string(s):
    """maskApi.c rleFrString (inverse of rle_to_string), used for the round-trip check."""
    s = s if isinstance(s, (bytes, bytearray)) else s.encode()
    counts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    return np.asarray(counts, dtype=np.uint32)


def rle_decode(counts, h, w):
    flat = np.zeros((h * w,), np.uint8)
    pos, v = 0, 0
    for c in counts:
        flat[pos:pos + int(c)] = v
        pos += int(c)
        v ^= 1
    return flat.reshape((w, h)).T


def paste_mask(mask_mm, ref_box_i32, im_h, im_w, thresh_binarize=0.5):
    """One detection of result_utils.py:195-217: zero-pad by one cell, resize to the (expanded, int32) box, threshold,
    paste into an im_h x im_w uint8 image."""
    M = mask_mm.shape[0]
    padded = np.zeros((M + 2, M + 2), np.float32)
    padded[1:-1, 1:-1] = mask_mm
    w = max(int(ref_box_i32[2]) - int(ref_box_i32[0]) + 1, 1)
    h = max(int(ref_box_i32[3]) - int(ref_box_i32[1]) + 1, 1)
    m = (resize_linear_f32(padded, w, h) > thresh_binarize).astype(np.uint8)
    im = np.zeros((im_h, im_w), np.uint8)
    x0, x1 = max(int(ref_box_i32[0]), 0), min(int(ref_box_i32[2]) + 1, im_w)
    y0, y1 = max(int(ref_box_i32[1]), 0), min(int(ref_box_i32[3]) + 1, im_h)
    if x1 > x0 and y1 > y0:
        im[y0:y1, x0:x1] = m[y0 - int(ref_box_i32[1]):y1 - int(ref_box_i32[1]), x0 - int(ref_box_i32[0]):x1 - int(ref_box_i32[0])]
    return im


def segm_results(cls_boxes, masks, ref_boxes, im_h, im_w, num_classes=81, M=14, cls_specific_mask=True, thresh_binarize=0.5):
    """lib/utils/result_utils.py:170-228 with cv2.resize -> resize_linear_f32 and mask_util.encode -> rle_encode/rle_to_string."""
    cls_segms = [[] for _ in range(num_classes)]
    mask_ind = 0
    scale = (M + 2.0) / M
    ref_boxes = expand_boxes(ref_boxes, scale).astype(np.int32)
    for j in range(1, num_classes):
        segms = []
        for _ in range(cls_boxes[j].shape[0]):
            m = masks[mask_ind, j if cls_specific_mask else 0, :, :]
            im_mask = paste_mask(m, ref_boxes[mask_ind], im_h, im_w, thresh_binarize)
            segms.append({'size': [im_h, im_w], 'counts': rle_to_string(rle_encode(im_mask)).decode()})
            mask_ind += 1
        cls_segms[j] = segms
    assert mask_ind == masks.shape[0]
    return cls_segms


# ------------------------------------------------------------------------------------------------ image pre-processing (8f rank 3)
def resize_linear_f32_scale(src, fx):
    """cv2.resize(src float32 HxWxC, None, None, fx=fx, fy=fx, INTER_LINEAR): dsize = cvRound(size * fx), coefficients from
    scale = 1/fx (not src/dst); fx == 0.5 is routed by OpenCV to its area-fast kernel whatever the size: a full 2x2 cell is
    ((a+b)+c)+d times 0.25f (for C == 3), and the partial cells of an odd side whose half rounds up (the last column, row or
    corner) are the sum of their in-range pixels, row-major from 0, divided by their count."""
    f32 = np.float32
    src = np.ascontiguousarray(src, dtype=f32)
    sh, sw = src.shape[:2]
    w, h = int(np.rint(sw * fx)), int(np.rint(sh * fx))
    scale = 1.0 / fx
    if (h, w) == (sh, sw):
        return src.copy()                                                # cv::resize copies when dsize == ssize, whatever fx
    if abs(scale - 2.0) < np.finfo(np.float64).eps:
        hf, wf = min(h, sh // 2), min(w, sw // 2)                        # full cells
        out = np.empty((h, w) + src.shape[2:], f32)
        a, b, c, d = src[0:2 * hf:2, 0:2 * wf:2], src[0:2 * hf:2, 1:2 * wf:2], src[1:2 * hf:2, 0:2 * wf:2], src[1:2 * hf:2, 1:2 * wf:2]
        out[:hf, :wf] = ((((a + b).astype(f32) + c).astype(f32) + d).astype(f32) * f32(.25)).astype(f32)
        for y in range(h):
            for x in range(wf if y < hf else 0, w):
                s = np.zeros(src.shape[2:], f32)
                rows, cols = range(2 * y, min(2 * y + 2, sh)), range(2 * x, min(2 * x + 2, sw))
                for r in rows:
                    for q in cols:
                        s = (s + src[r, q]).astype(f32)
                out[y, x] = (s / f32(len(rows) * len(cols))).astype(f32)
        return out

    def axis(dst):
        f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(f32)
        s = np.floor(f).astype(np.int64)
        return s, (f - s.astype(f32)).astype(f32)

    sx, fxw = axis(w)
    sy, fyw = axis(h)
    lo = sx < 0
    fxw = np.where(lo, f32(0), fxw); sx = np.where(lo, 0, sx)
    hi = sx >= sw - 1
    fxw = np.where(hi, f32(0), fxw); sx = np.where(hi, sw - 1, sx)
    a0, a1 = (f32(1) - fxw).astype(f32), fxw
    sx1 = np.minimum(sx + 1, sw - 1)
    hb = ((src[:, sx] * a0[None, :, None]).astype(f32) + (src[:, sx1] * a1[None, :, None]).astype(f32)).astype(f32)
    r0, r1 = np.clip(sy, 0, sh - 1), np.clip(sy + 1, 0, sh - 1)
    b0, b1 = (f32(1) - fyw).astype(f32), fyw
    return ((hb[r0] * b0[:, None, None]).astype(f32) + (hb[r1] * b1[:, None, None]).astype(f32)).astype(f32)


def prep_im_for_blob(im, pixel_means=(122.7717, 115.9465, 102.9801), target_sizes=(800,), max_size=1333):
    """lib/utils/blob.py:57-87 with cv2.resize -> resize_linear_f32_scale."""
    im = im.astype(np.float32, copy=True)
    im -= list(pixel_means)
    im_size_min, im_size_max = np.min(im.shape[0:2]), np.max(im.shape[0:2])
    ims, im_scales = [], []
    for target_size in target_sizes:
        im_scale = float(target_size) / float(im_size_min)
        if np.round(im_scale * im_size_max) > max_size:
            im_scale = float(max_size) / float(im_size_max)
        ims.append(resize_linear_f32_scale(im, im_scale))
        im_scales.append(im_scale)
    return ims, im_scales


def im_list_to_blob(ims, fpn_on=False, fpn_coarsest_stride=32):
    """lib/utils/blob.py:27-55."""
    max_shape = np.array([im.shape for im in ims]).max(axis=0)
    if fpn_on:
        stride = float(fpn_coarsest_stride)
        max_shape[0] = int(np.ceil(max_shape[0] / stride) * stride)
        max_shape[1] = int(np.ceil(max_shape[1] / stride) * stride)
    blob = np.zeros((len(ims), max_shape[0], max_shape[1], 3), dtype=np.float32)
    for i, im in enumerate(ims):
        blob[i, 0:im.shape[0], 0:im.shape[1], :] = im
    return blob.transpose((0, 3, 1, 2))

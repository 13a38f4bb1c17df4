"""Mirror of the hot-path part of the reference lib/utils/result_utils.py: postprocess_output (:76-94)
and box_results_with_nms_and_limit (:96-168), computed by the engine's on-device detection stage
(decode with weights (10,10,5,5), clip, score > 0.05, per-class NMS 0.5, top-100) and returned in the
reference's numpy structures; and of segm_results (:170-228): mask paste + COCO RLE on the device.  batch_results gives both, per
image, for a whole detector.detect() batch."""
import numpy as np
import torch

from ..engine import ST_DETECT, engine_owning


def to_np(x):
    """result_utils.py:25-30."""
    if isinstance(x, np.ndarray):
        return x
    return x.detach().cpu().numpy()


def empty_results(num_classes, num_images):
    """result_utils.py:32-52: all_boxes[cls][image] = N x 5 array (x1, y1, x2, y2, score); all_segms[cls][image] = list of COCO RLE dicts in
    1:1 correspondence; all_keyps likewise (unused by the detectors here).  Three independent nested lists (no shared inner lists)."""
    def nest():
        return [[[] for _ in range(num_images)] for _ in range(num_classes)]
    return nest(), nest(), nest()


def extend_results(index, all_res, im_res):
    """result_utils.py:54-60: file one image's per-class results at `index`; class 0 (background) is skipped."""
    for cls_idx in range(1, len(im_res)):
        all_res[cls_idx][index] = im_res[cls_idx]


def _as_float(x):
    if torch.is_tensor(x):
        return float(x.reshape(-1)[0])
    return float(np.asarray(x).reshape(-1)[0])


def postprocess_output(rois, scaling_factor, im_size, class_scores, bbox_deltas, bbox_reg_weights=(10.0, 10.0, 5.0, 5.0)):
    """-> (scores_final [D], boxes_final [D,4], boxes_per_class list[81] of [n_j,5]) numpy, like result_utils.py:76-94.
    The engine that runs the detection stage is the one whose buffers `class_scores` / `bbox_deltas` / `rois` are views of (what
    detector.forward returned) -- there is no global "current engine", so several models / image sizes can be in flight."""
    eng = engine_owning(class_scores, bbox_deltas, rois)
    if eng is None:
        raise RuntimeError("postprocess_output: class_scores / bbox_deltas must be the tensors returned by detector.forward "
                           "(views of the engine's device buffers; clones or CPU copies carry no engine)")
    if tuple(bbox_reg_weights) != (10.0, 10.0, 5.0, 5.0):
        raise NotImplementedError("only the reference's default bbox_reg_weights are built")
    R = eng.cfg.post_nms_top_n
    n = int(class_scores.shape[0])
    nr = rois.shape[-2] if len(rois.shape) == 3 else rois.shape[0]
    if nr != n:
        raise RuntimeError("postprocess_output: %d rois for %d score rows" % (nr, n))
    if n > R:
        raise RuntimeError("postprocess_output: %d RoIs exceed the engine capacity %d" % (n, R))
    rois = rois if torch.is_tensor(rois) else torch.as_tensor(np.asarray(rois))
    r = rois.reshape(-1, rois.shape[-1]).to(eng.device).float()
    er, ec, eb, en = eng.buffer("rois"), eng.buffer("cls_prob"), eng.buffer("bbox_pred"), eng.buffer("roi_counts")
    # inputs that already are the engine's own views are left in place; anything else is copied in
    if r.data_ptr() != er[0, :, 1:5].data_ptr():
        er[0].zero_(); er[0, :n, 1:5] = r[:, -4:]
    if class_scores.data_ptr() != ec.data_ptr():
        ec[:n] = class_scores.to(eng.device).float()
    if bbox_deltas.data_ptr() != eb.data_ptr():
        eb[:n] = bbox_deltas.to(eng.device).float()
    en[0] = n
    sf = _as_float(scaling_factor)
    im = (im_size.detach().cpu().numpy() if torch.is_tensor(im_size) else np.asarray(im_size)).squeeze()
    eng.set_original_size(float(im[0]), float(im[1]))
    eng.run(None, sf, ST_DETECT, ST_DETECT)
    cnt = int(eng.buffer("det_counts")[0].item())
    boxes = eng.buffer("det_boxes")[0, :cnt].cpu().numpy()
    scores = eng.buffer("det_scores")[0, :cnt].cpu().numpy()
    classes = eng.buffer("det_classes")[0, :cnt].cpu().numpy()
    NC = eng.cfg.num_classes
    cls_boxes = [[] for _ in range(NC)]
    for j in range(1, NC):
        m = classes == j
        cls_boxes[j] = np.hstack((boxes[m], scores[m][:, None])).astype(np.float32, copy=False)
    return scores, boxes, cls_boxes


def segm_results(cls_boxes, masks, ref_boxes, im_h, im_w, num_classes=81, M=14, cls_specific_mask=True, thresh_binarize=0.5):
    """Mirror of result_utils.segm_results (:170-228).  `masks` may be the CUDA tensor returned by model.mask_head
    (no 25 MB device->host copy) or a numpy array [D, K, M, M]; returns cls_segms: per class a list of
    {'size': [im_h, im_w], 'counts': str} exactly like pycocotools' encode() + .decode()."""
    from .. import ops
    n_per_class = [0] + [int(np.asarray(cls_boxes[j]).reshape(-1, 5).shape[0]) if len(cls_boxes[j]) else 0 for j in range(1, num_classes)]
    D = int(sum(n_per_class))
    dev = torch.device("cuda", torch.cuda.current_device())
    m = masks if torch.is_tensor(masks) else torch.from_numpy(np.ascontiguousarray(masks))
    if m.shape[0] != D:
        raise AssertionError("segm_results: %d masks for %d detections" % (m.shape[0], D))    # reference: assert mask_ind == masks.shape[0]
    if m.shape[-1] != M:
        raise ValueError("segm_results: masks are %dx%d but M=%d" % (m.shape[-1], m.shape[-1], M))
    cls_segms = [[] for _ in range(num_classes)]
    if D == 0:
        return cls_segms
    m = m.to(dev)
    classes = np.repeat(np.arange(num_classes), n_per_class).astype(np.int32)
    if not cls_specific_mask:
        classes[:] = 0
    # the reference expands the boxes on the host in the dtype it is given (boxes.py:245-261) and truncates to int32
    rb = np.asarray(ref_boxes)
    scale = (M + 2.0) / M
    w_half = (rb[:, 2] - rb[:, 0]) * .5
    h_half = (rb[:, 3] - rb[:, 1]) * .5
    x_c = (rb[:, 2] + rb[:, 0]) * .5
    y_c = (rb[:, 3] + rb[:, 1]) * .5
    w_half *= scale
    h_half *= scale
    exp = np.zeros(rb.shape)
    exp[:, 0] = x_c - w_half
    exp[:, 2] = x_c + w_half
    exp[:, 1] = y_c - h_half
    exp[:, 3] = y_c + h_half
    exp = torch.from_numpy(exp.astype(np.int32)).to(dev)
    _, strings = ops.segm_rle(m, torch.from_numpy(classes).to(dev), exp, im_h, im_w, thresh_binarize, expanded=True)
    k = 0
    for j in range(1, num_classes):
        cls_segms[j] = [{'size': [int(im_h), int(im_w)], 'counts': strings[k + i].decode()} for i in range(n_per_class[j])]
        k += n_per_class[j]
    return cls_segms


def batch_results(out, original_sizes, num_classes=81, thresh_binarize=0.5):
    """detector.detect()'s padded output dict -> per image (scores_final, boxes_final, boxes_per_class, cls_segms): exactly what
    postprocess_output and then segm_results(cls_boxes, masks, boxes_final, int(h_orig), int(w_orig), M) return for that image alone.
    original_sizes [B,2]: each image's un-scaled (height, width); int() of each value is the RLE canvas, as in the notebooks.
    cls_segms is None when `out` has no masks (Faster R-CNN).  The masks are pasted and encoded on the device for the whole batch in
    one launch; boxes, scores, classes, counts and the offsets of the strings come back in one copy, the strings in one more."""
    from .. import ops
    B, cap = int(out["boxes"].shape[0]), int(out["boxes"].shape[1])
    sizes = ops.segm_image_sizes(original_sizes, B)           # validated before anything is launched
    fields = (out["boxes"], out["scores"], out["classes"], out["counts"])
    masks = out.get("masks")
    if masks is None:
        boxes, scores, classes, counts = ops.to_host(*fields)
        offs = str_h = None
    else:
        strings, host = ops.segm_rle_batch_device(masks, None, out["boxes"], out["counts"], sizes, thresh_binarize, extra=fields)
        offs, (boxes, scores, classes, counts) = host[0], host[2:]
        str_h = strings[:int(offs[-1])].cpu().numpy().tobytes() if offs[-1] > 0 else b""
    results = []
    for b in range(B):
        n = min(max(int(counts[b]), 0), cap)
        bx, sc, cl = boxes[b, :n].copy(), scores[b, :n].copy(), classes[b, :n]
        # the slots of an image are class-major (the engine's detection stage emits them class by class), which segm_results assumes;
        # class j's rows are then one slice [bounds[j-1], bounds[j]) of the image's detections
        if np.any(np.diff(cl) < 0) or np.any((cl < 1) | (cl >= num_classes)):
            raise RuntimeError("batch_results: the detections of image %d are not grouped by class in 1..%d" % (b, num_classes - 1))
        bounds = np.searchsorted(cl, np.arange(1, num_classes + 1))
        dets = np.hstack((bx, sc[:, None])).astype(np.float32, copy=False)
        cls_boxes = [[]] + [dets[bounds[j - 1]:bounds[j]] for j in range(1, num_classes)]
        cls_segms = None
        if str_h is not None:
            size = [int(sizes[b, 0]), int(sizes[b, 1])]
            segs = [{'size': list(size), 'counts': str_h[offs[b * cap + d]:offs[b * cap + d + 1]].decode()} for d in range(n)]
            cls_segms = [[]] + [segs[bounds[j - 1]:bounds[j]] for j in range(1, num_classes)]
        results.append((sc, bx, cls_boxes, cls_segms))
    return results

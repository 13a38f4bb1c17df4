"""Regenerates tests/golden/ref_golden.npz by running the REFERENCE's own code (needs the reference tree and oracle/_ref, see
oracle/build_ref.sh; run from the repository root: python tests/golden/make_ref_golden.py).  What it stores:

  * name_*    utils/utils.py parse_th_to_caffe2 over every torchvision trunk key of resnet50 / resnet101
  * pkl_*     per eval_*.ipynb configuration: the trunk keys of the reference detector (the blobs a Detectron pickle must hold), the FPN
              blob stems, and -- after the reference loader read a synthetic pickle of oracle.network.synthetic_params -- the name, shape,
              bit-pattern sum and first 8 values of every loaded parameter
  * nms_* / roi_*   the reference's Cython NMS keep lists and its RoIAlign CPU loop on seeded random inputs
  * prep_* / segm_* the reference's blob.prep_im_for_blob + im_list_to_blob (cv2 with IPP off) and segm_results (the pasted masks it
              hands to mask_util.encode, and the returned structure) on seeded random inputs
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import network as net  # noqa: E402
from oracle import ref  # noqa: E402
from oracle import reference_shim as rs  # noqa: E402
import ref_cases as rc  # noqa: E402


def main():
    rs.install()
    import cv2
    import torchvision.models as models
    import utils.blob as rb
    import utils.boxes as box_utils
    import utils.result_utils as ru
    from model.detector import detector as ref_detector
    from utils.utils import parse_th_to_caffe2
    out = {}
    # ---- caffe2 blob names
    for arch in ("resnet50", "resnet101"):
        keys = [k for k in getattr(models, arch)().state_dict().keys() if not ('running' in k or 'fc' in k or 'num_batches' in k)]
        out["name_%s_th" % arch] = np.array(keys)
        out["name_%s_c2" % arch] = np.array([parse_th_to_caffe2(k.split('.')) for k in keys])
    # ---- Detectron pickle import, per notebook configuration
    import tempfile
    for name in sorted(rc.CONFIGS):
        kw, flags = rc.CONFIGS[name]
        P = net.synthetic_params("resnet50", **flags)
        ref_kw = dict(kw, roi_feature_channels=1024) if flags["fpn"] else kw
        proto = ref_detector(**ref_kw)
        trunk = list(proto.model.state_dict().keys())
        fpn_stems = [(l + '.' + list(getattr(proto.model, l).state_dict().keys())[-1]) for l in rc.FPN['fpn_layers']] if flags["fpn"] else []
        layout = {"trunk": trunk, "c2": {k: parse_th_to_caffe2(k.split('.')) for k in trunk}, "fpn": [parse_th_to_caffe2(s.split('.')) for s in fpn_stems]}
        with tempfile.TemporaryDirectory() as d:
            pkl = os.path.join(d, "model_final.pkl")
            rc.write_detectron_pickle(pkl, layout, P, flags)
            sd = ref_detector(detector_pkl_file=pkl, **kw).state_dict()
        keys = sorted(P)
        out["pkl_%s_trunk" % name] = np.array(trunk)
        out["pkl_%s_trunk_c2" % name] = np.array([layout["c2"][k] for k in trunk])
        out["pkl_%s_fpn" % name] = np.array(layout["fpn"], dtype=str)
        out["pkl_%s_keys" % name] = np.array(keys)
        out["pkl_%s_shapes" % name] = np.array([list(sd[k].shape) + [0] * (4 - sd[k].dim()) for k in keys], np.int64)
        out["pkl_%s_bitsums" % name] = np.array([rc.bitsum(sd[k]) for k in keys], np.int64)
        out["pkl_%s_head" % name] = np.array([rc.head8(sd[k]) for k in keys], np.float32)
    # ---- NMS and RoIAlign
    for i, (d, t) in enumerate(rc.nms_cases()):
        out["nms%d_keep" % i] = np.asarray(box_utils.nms(d, t), dtype=np.int64)
    f, r = rc.roi_case()
    for (p, sr) in rc.ROI_CFGS:
        out["roi_p%d_sr%d" % (p, sr)] = ref.roi_align_forward_ref(f, r, p, p, 1 / 32., sr)[:rc.ROI_KEEP[p]]
    # ---- image prep and mask paste + RLE
    cv2.ipp.setUseIPP(False)
    for i, (im, ts, ms) in enumerate(rc.prep_cases()):
        ims, scales = rb.prep_im_for_blob(im.copy(), target_sizes=[ts], max_size=ms)
        out["prep%d_scale" % i] = np.float64(scales[0])
        out["prep%d_blob" % i] = rb.im_list_to_blob(ims, fpn_on=True)
    captured = []
    ru.mask_util.encode = lambda arr: (captured.append(np.ascontiguousarray(arr[:, :, 0])) or
                                       [{'size': list(arr.shape[:2]), 'counts': ref.rle_to_string(ref.rle_encode(arr[:, :, 0]))}])
    M, K, im_h, im_w, boxes, cls, masks, cls_boxes = rc.segm_case()
    want = ru.segm_results(cls_boxes, masks, boxes, im_h, im_w, num_classes=K, M=M)
    out["segm_counts"] = np.array([s['counts'] for j in range(1, K) for s in want[j]])
    out["segm_sizes"] = np.array([s['size'] for j in range(1, K) for s in want[j]], np.int64)
    out["segm_per_class"] = np.array([len(want[j]) for j in range(K)], np.int64)
    out["segm_pasted_bits"] = np.packbits(np.stack(captured).reshape(len(captured), -1), axis=1)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_golden.npz"), **out)


if __name__ == "__main__":
    main()

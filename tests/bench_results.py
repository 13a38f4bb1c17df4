"""Throughput from uint8 photos to per-image COCO results (scores_final, boxes_final, boxes_per_class, cls_segms with the RLE strings),
Mask R-CNN R-50-FPN with synthetic weights, three ways:
  detect_images   detector.detect_images: one detect() per canvas of `--batch` images, one batched paste + RLE, one copy of the results
  detect_segm     utils.blob.images_to_batch + detect() + one segm_results call per image (the batched option without batch_results)
  notebook        the batch-1 notebook flow per image: image_to_blob(fpn_on=True), forward, postprocess_output, add_multilevel_rois_for_test,
                  mask_head, segm_results(M=28)
Inputs: seeded uint8 images of sizes typical of photo datasets, grouped by orientation into 800x1344 (landscape, square) and 1344x800
(portrait) canvases, full batches only.  The first two arms run with engine_defaults emit_full_masks=False, det_cap=100 (they only read
the detected class's mask); the notebook flow needs the full [D,81,28,28] masks of mask_head.  Every arm runs once over all images first
(engines built, kernels warmed up, results of the three arms compared), then `--passes` rounds in which each arm times one pass over all
images in turn; each timed window ends in a device synchronise.  Prints one JSON line: the median img/s of each arm and every pass.

    python tests/bench_results.py [--images 48] [--batch 8] [--passes 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

PHOTO_SIZES = [(480, 640), (640, 480), (427, 640), (640, 427), (640, 640), (375, 500), (500, 375), (512, 640), (612, 612), (360, 640),
               (424, 640), (640, 512)]          # (height, width) of the original images
CANVAS = {"landscape": (800, 1344), "portrait": (1344, 800)}


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


def make_model(params, **engine_defaults):
    from detectorch_b200.model.detector import detector
    model = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                     conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                     roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                     use_rpn_head=True, use_mask_head=True, mask_head_type='1up4convs')
    sd = model.state_dict()
    for k, v in params.items():
        sd[k].copy_(v)
    model = model.cuda()
    model.engine_defaults.update(engine_defaults)
    model.max_cached_engines = 32                    # one batch-1 engine per distinct blob size stays alive while timing
    return model


def per_class(boxes, scores, classes, num_classes=81):
    cls_boxes = [[] for _ in range(num_classes)]
    for j in range(1, num_classes):
        m = classes == j
        cls_boxes[j] = np.hstack((boxes[m], scores[m][:, None])).astype(np.float32, copy=False)
    return cls_boxes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=48)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--passes", type=int, default=5, help="timed passes over all images, per arm")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    from detectorch_b200.utils import blob, result_utils
    from detectorch_b200.utils.multilevel_rois import add_multilevel_rois_for_test
    from oracle import network as net

    dev = torch.device("cuda:0")
    params = net.synthetic_params("resnet50")
    batched = make_model(params, emit_full_masks=False, det_cap=100)
    single = make_model(params)

    rng = np.random.RandomState(a.seed)
    shapes = [PHOTO_SIZES[i] for i in rng.randint(0, len(PHOTO_SIZES), a.images)]
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    groups = {"landscape": [i for i, (h, w) in enumerate(shapes) if h <= w], "portrait": [i for i, (h, w) in enumerate(shapes) if h > w]}
    batches = []
    for g, idx in groups.items():
        for s in range(0, len(idx) - a.batch + 1, a.batch):           # full batches only
            batches.append(([ims[i] for i in idx[s:s + a.batch]], CANVAS[g]))
    n = sum(len(b) for b, _ in batches)

    def arm_detect_images():
        res = []
        for part, canvas in batches:
            res += batched.detect_images(part, canvas=canvas)
        return res

    def arm_detect_segm():
        res = []
        for part, canvas in batches:
            data, sizes, scales, orig = blob.images_to_batch(part, canvas=canvas)
            out = batched.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
            counts, boxes = out["counts"].cpu().numpy(), out["boxes"].cpu().numpy()
            scores, classes = out["scores"].cpu().numpy(), out["classes"].cpu().numpy()
            for b in range(len(part)):
                k = int(counts[b])
                bx, sc = boxes[b, :k], scores[b, :k]
                cb = per_class(bx, sc, classes[b, :k])
                segms = result_utils.segm_results(cb, out["masks"][b, :k], bx, int(orig[b, 0]), int(orig[b, 1]), M=28, cls_specific_mask=False)
                res.append((sc, bx, cb, segms))
        return res

    def arm_notebook():
        res = []
        for part, _ in batches:
            for im in part:
                data, s = blob.image_to_blob(im, fpn_on=True)
                sf = torch.tensor([s])
                with torch.no_grad():
                    cls, box, rois, feats = single(data, scaling_factor=sf)
                sc, bx, cb = result_utils.postprocess_output(rois, sf, torch.tensor([im.shape[:2]]), cls, box)
                masks = torch.zeros((0, 81, 28, 28), device=dev)
                if len(bx):
                    blobs = add_multilevel_rois_for_test({"mask_rois": bx * np.float32(s)}, "mask_rois")
                    lst = [torch.from_numpy(blobs["mask_rois_fpn%d" % l]).to(dev) if len(blobs["mask_rois_fpn%d" % l]) else None for l in range(2, 6)]
                    masks = single.mask_head(feats, lst, torch.from_numpy(blobs["mask_rois_idx_restore_int32"].astype(np.int64)).to(dev))
                segms = result_utils.segm_results(cb, masks, bx, im.shape[0], im.shape[1], M=28)
                res.append((sc, bx, cb, segms))
        return res

    def same(x, y):
        return all(np.array_equal(p[0], q[0]) and np.array_equal(p[1], q[1]) and p[3] == q[3] and
                   all(np.array_equal(u, v) for u, v in zip(p[2][1:], q[2][1:])) for p, q in zip(x, y)) and len(x) == len(y)

    arms = (("detect_images", arm_detect_images), ("detect_segm", arm_detect_segm), ("notebook", arm_notebook))
    first = {name: fn() for name, fn in arms}          # builds the engines, warms every kernel and shape up
    torch.cuda.synchronize()
    agree = same(first["detect_images"], first["detect_segm"]) and same(first["detect_images"], first["notebook"])
    rates = {name: [] for name, _ in arms}
    for _ in range(a.passes):                          # the arms alternate, so a drift of the clocks or of the host load hits all three
        for name, fn in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            rates[name].append(n / (time.perf_counter() - t0))
    res = {name: float(np.median(r)) for name, r in rates.items()}
    print(json.dumps({"metric": "coco_results_img_per_s", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "images": n, "batch": a.batch, "passes": a.passes, "results_agree": bool(agree),
                      "detections": int(sum(len(r[0]) for r in first["detect_images"])),
                      **{name + "_img_per_s": round(v, 2) for name, v in res.items()},
                      **{name + "_img_per_s_each_pass": [round(v, 1) for v in r] for name, r in rates.items()},
                      "detect_images_vs_detect_segm": round(res["detect_images"] / res["detect_segm"], 3),
                      "detect_images_vs_notebook": round(res["detect_images"] / res["notebook"], 3)}))


if __name__ == "__main__":
    main()

"""Throughput of Fast R-CNN R-50-FPN (eval_fast_FPN.ipynb's model, synthetic weights) from uint8 photos and roidb proposals to per-image
results (scores_final, boxes_final, boxes_per_class), two ways:
  detect_images   detector.detect_images(ims, proposals=): one detect() per canvas of `--batch` images; the proposals are scaled,
                  deduplicated and mapped to the FPN levels on the device
  notebook        the batch-1 notebook flow per image: preprocess_sample(fpn_on=True) (image_to_blob, numpy deduplication and level map),
                  forward(image, [rois_fpn2..5], roi_original_idx), postprocess_output
Inputs: seeded uint8 images of sizes typical of photo datasets, grouped by orientation into 800x1344 (landscape, square) and 1344x800
(portrait) canvases, full batches only; each image has `--proposals` seeded boxes in a Detectron-like size and aspect distribution
(sides log-uniform in 16..0.8*max side, aspect 1/3..3), of which ~4 % repeat or nearly repeat another box after scaling.  Both arms run
once over all images first (engines built, kernels warmed up, results compared), then `--passes` rounds in which each arm times one pass
over all images in turn; each timed window ends in a device synchronise.  Prints one JSON line: the median img/s of each arm and every pass.

    python tests/bench_fast.py [--images 48] [--batch 8] [--passes 5] [--proposals 1000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_results import CANVAS, PHOTO_SIZES, power_limit  # noqa: E402

FAST_FPN = dict(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], roi_height=7, roi_width=7,
                roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2)


def make_model(params):
    from detectorch_b200.model.detector import detector
    model = detector(**FAST_FPN)
    sd = model.state_dict()
    for k, v in params.items():
        sd[k].copy_(v)
    model = model.cuda()
    model.max_cached_engines = 64                    # the batch-1 flow meets one engine per (blob size, rounded proposal count)
    return model


def roidb_boxes(rng, n, h, w):
    """n float32 boxes inside an h x w image; n // 25 exact repeats and n // 50 boxes within 2 px of another."""
    dup, near = n // 25, n // 50
    m = n - dup - near
    side = np.exp(rng.uniform(np.log(16), np.log(0.8 * max(h, w)), m))
    ar = np.exp(rng.uniform(np.log(1 / 3.), np.log(3.), m))
    bw, bh = np.minimum(side * np.sqrt(ar), w - 1), np.minimum(side / np.sqrt(ar), h - 1)
    x1, y1 = rng.uniform(0, w - bw), rng.uniform(0, h - bh)
    b = np.stack([x1, y1, x1 + bw, y1 + bh], 1)
    nb = b[rng.choice(m, near)] + rng.uniform(-2, 2, (near, 4))
    nb[:, 2:] = np.maximum(nb[:, 2:], nb[:, :2])
    return np.concatenate([b, b[rng.choice(m, dup)], nb])[rng.permutation(n)].astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=48)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--passes", type=int, default=5, help="timed passes over all images, per arm")
    ap.add_argument("--proposals", type=int, default=1000, help="proposals per image (at most 1000)")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    from detectorch_b200.utils import result_utils
    from detectorch_b200.utils.preprocess_sample import preprocess_sample
    from oracle import network as net

    dev = torch.device("cuda:0")
    params = net.synthetic_params("resnet50", fpn=True, rpn=False, mask=False)
    batched, single = make_model(params), make_model(params)

    rng = np.random.RandomState(a.seed)
    shapes = [PHOTO_SIZES[i] for i in rng.randint(0, len(PHOTO_SIZES), a.images)]
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    props = [roidb_boxes(rng, a.proposals, h, w) for h, w in shapes]
    groups = {"landscape": [i for i, (h, w) in enumerate(shapes) if h <= w], "portrait": [i for i, (h, w) in enumerate(shapes) if h > w]}
    batches = []
    for g, idx in groups.items():
        for s in range(0, len(idx) - a.batch + 1, a.batch):           # full batches only
            part = idx[s:s + a.batch]
            batches.append(([ims[i] for i in part], [props[i] for i in part], CANVAS[g]))
    n = sum(len(b[0]) for b in batches)
    prep = preprocess_sample(target_sizes=[800], fpn_on=True)

    def arm_detect_images():
        res = []
        for part, pp, canvas in batches:
            res += [r[:3] for r in batched.detect_images(part, canvas=canvas, proposals=pp)]
        return res

    def arm_notebook():
        res = []
        for part, pp, _ in batches:
            for im, p in zip(part, pp):
                s = prep({'image': im, 'dbentry': {'boxes': p}})
                lst = [s['rois_fpn%d' % l].to(dev) for l in range(2, 6)]
                with torch.no_grad():
                    cls, box, _, _ = single(s['image'], lst, roi_original_idx=s['rois_idx_restore_int32'].long().to(dev))
                res.append(result_utils.postprocess_output(s['rois'], s['scaling_factors'], s['original_im_size'], cls, box))
        return res

    def same(x, y):
        return len(x) == len(y) and all(np.array_equal(p[0], q[0]) and np.array_equal(p[1], q[1]) and
                                        all(np.array_equal(np.reshape(u, (-1, 5)), np.reshape(v, (-1, 5))) for u, v in zip(p[2][1:], q[2][1:]))
                                        for p, q in zip(x, y))

    arms = (("detect_images", arm_detect_images), ("notebook", arm_notebook))
    first = {name: fn() for name, fn in arms}          # builds the engines, warms every kernel and shape up
    torch.cuda.synchronize()
    agree = same(first["detect_images"], first["notebook"])
    rates = {name: [] for name, _ in arms}
    for _ in range(a.passes):                          # the arms alternate, so a drift of the clocks or of the host load hits both
        for name, fn in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            rates[name].append(n / (time.perf_counter() - t0))
    res = {name: float(np.median(r)) for name, r in rates.items()}
    print(json.dumps({"metric": "fast_rcnn_fpn_img_per_s", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "images": n, "batch": a.batch, "proposals_per_image": a.proposals, "passes": a.passes, "results_agree": bool(agree),
                      "detections": int(sum(len(r[0]) for r in first["detect_images"])),
                      **{name + "_img_per_s": round(v, 2) for name, v in res.items()},
                      **{name + "_img_per_s_each_pass": [round(v, 1) for v in r] for name, r in rates.items()},
                      "detect_images_vs_notebook": round(res["detect_images"] / res["notebook"], 3)}))


if __name__ == "__main__":
    main()

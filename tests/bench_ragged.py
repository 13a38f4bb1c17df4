"""Throughput of batches of differently-sized images (detect(..., image_sizes, original_sizes)) against running the same images one at a
time at their own sizes -- the only correct option without per-image sizes.  Mask R-CNN R-50-FPN with synthetic weights.

Inputs: a seeded list of original sizes typical of photo datasets, prepared with utils.blob.images_to_batch (short side 800, long side
<= 1333, /32), grouped by orientation into 800x1344 (landscape, square) and 1344x800 (portrait) canvases, `--batch` images per batch.
Prints one JSON line: img/s of both arms and the fraction of canvas pixels that are padding.

    python tests/bench_ragged.py [--images 64] [--batch 8] [--passes 3]
"""
import argparse
import json
import os
import subprocess
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--passes", type=int, default=3, help="timed passes over all images, per arm")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    from detectorch_b200.model.detector import detector
    from detectorch_b200.utils import blob
    from oracle import network as net

    dev = torch.device("cuda:0")
    model = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                     conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                     roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                     use_rpn_head=True, use_mask_head=True, mask_head_type='1up4convs')
    sd = model.state_dict()
    for k, v in net.synthetic_params("resnet50").items():
        sd[k].copy_(v)
    model = model.cuda()
    model.engine_defaults = dict(emit_full_masks=False, det_cap=100)
    model.max_cached_engines = 32                    # one batch-1 engine per distinct blob size stays alive while timing

    rng = np.random.RandomState(a.seed)
    shapes = [PHOTO_SIZES[i] for i in rng.randint(0, len(PHOTO_SIZES), a.images)]
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    groups = {"landscape": [i for i, (h, w) in enumerate(shapes) if h <= w], "portrait": [i for i, (h, w) in enumerate(shapes) if h > w]}
    batches, singles, used = [], [], []
    valid_px = canvas_px = 0
    for g, idx in groups.items():
        for s in range(0, len(idx) - a.batch + 1, a.batch):           # full batches only
            part = idx[s:s + a.batch]
            data, sizes, scales, orig = blob.images_to_batch([ims[i] for i in part], canvas=CANVAS[g])
            batches.append((data, sizes.tolist(), scales.tolist(), orig.tolist()))
            valid_px += int((sizes[:, 0] * sizes[:, 1]).sum())
            canvas_px += a.batch * CANVAS[g][0] * CANVAS[g][1]
            for j, i in enumerate(part):
                h, w = batches[-1][1][j]
                singles.append((data[j:j + 1, :, :h, :w].contiguous(), batches[-1][2][j], batches[-1][3][j]))
            used += part
    n = len(used)

    def ragged():
        for data, sizes, scales, orig in batches:
            model.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)

    def one_by_one():
        for data, sf, orig in singles:
            model.detect(data, scaling_factor=sf)

    res = {}
    for name, fn in (("ragged", ragged), ("batch1", one_by_one)):
        fn()                                          # builds the engines and warms every kernel up
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(a.passes):
            fn()
        t1.record()
        torch.cuda.synchronize()
        res[name] = n * a.passes / (t0.elapsed_time(t1) / 1000.0)
    print(json.dumps({"metric": "ragged_batch_img_per_s", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "images": n, "batch": a.batch, "passes": a.passes, "ragged_img_per_s": round(res["ragged"], 2),
                      "batch1_img_per_s": round(res["batch1"], 2), "speedup": round(res["ragged"] / res["batch1"], 3),
                      "padding_fraction": round(1.0 - valid_px / canvas_px, 4),
                      "distinct_sizes": sorted({tuple(s) for b in batches for s in b[1]})}))


if __name__ == "__main__":
    main()

"""Times proposal recall on the device (coco_eval.box_proposal_recall, Detectron's 8 combinations in one launch) against the reference's
evaluate_box_proposals on its compiled cython_bbox (8 calls), on ~5000 images x 1000 proposals x ~7 GT; and propose_images against the
batch-1 forward() loop.  Prints one JSON line; the card and its power limit go with the numbers.
    python tests/bench_proposal_recall.py [--images 5000] [--ref-images 5000]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--ref-images", type=int, default=5000)
    ap.add_argument("--propose-images", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_proposal_recall needs a GPU")
    import proposal_recall_cases as cases
    from detectorch_b200.utils import coco_eval
    rng = np.random.RandomState(0)
    roidb = [cases.random_entry(rng, 1000, int(rng.randint(1, 14)), jitter=12.0) for _ in range(a.images)]
    combos = [(x, l) for x in ('all', 'small', 'medium', 'large') for l in (100, 1000)]
    coco_eval.box_proposal_recall(roidb[:50])                          # warm-up
    torch.cuda.synchronize()
    dev_s = []
    for _ in range(3):
        t = time.perf_counter()
        got = coco_eval.box_proposal_recall(roidb)
        torch.cuda.synchronize()
        dev_s.append(time.perf_counter() - t)
    res = {"images": a.images, "device_recall_s": min(dev_s), "device_recall_runs_s": dev_s,
           "ar": {"%s@%s" % k: float(got[k]['ar']) for k in combos}}
    from oracle import cython_bbox
    if cython_bbox.available():
        jde, _ = cython_bbox.load()
        sub = roidb[:a.ref_images]
        t = time.perf_counter()
        ref = {k: jde.evaluate_box_proposals(None, sub, area=k[0], limit=k[1]) for k in combos}
        res["reference_recall_s"] = time.perf_counter() - t
        res["reference_images"] = len(sub)
        mine = coco_eval.box_proposal_recall(sub) if len(sub) != len(roidb) else got
        res["equal"] = all(np.array_equal(mine[k]['gt_overlaps'], ref[k]['gt_overlaps']) and np.array_equal(mine[k]['recalls'], ref[k]['recalls'])
                           for k in combos)
    # propose_images vs the batch-1 forward() loop on photo-sized images
    from oracle import network as net
    from detectorch_b200.model.detector import detector
    from detectorch_b200.utils import blob
    model = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                     conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                     roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                     use_rpn_head=True, use_mask_head=False)
    sd = model.state_dict()
    for k, v in net.synthetic_params("resnet50", mask=False).items():
        if k in sd:
            sd[k].copy_(v)
    model = model.cuda()
    prng = np.random.RandomState(1)
    ims = [prng.randint(0, 256, (480, 640, 3) if i % 4 else (640, 480, 3)).astype(np.uint8) for i in range(a.propose_images)]
    land = [im for im in ims if im.shape[0] < im.shape[1]]
    port = [im for im in ims if im.shape[0] >= im.shape[1]]
    groups = [(land[i:i + 8], (800, 1088)) for i in range(0, len(land), 8)] + [(port[i:i + 8], (1088, 800)) for i in range(0, len(port), 8)]
    for _ in range(2):
        for g, c in groups:
            model.propose_images(g, canvas=c)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for g, c in groups:
        model.propose_images(g, canvas=c)
    torch.cuda.synchronize()
    res["propose_images_img_s"] = len(ims) / (time.perf_counter() - t)

    def loop():
        for im in ims:
            d, s = blob.image_to_blob(im, fpn_on=True)
            r = model(d, scaling_factor=s)[2]
            (r / s).cpu()
    loop()
    torch.cuda.synchronize()
    t = time.perf_counter()
    loop()
    torch.cuda.synchronize()
    res["forward_loop_img_s"] = len(ims) / (time.perf_counter() - t)
    try:
        res["gpu"] = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception as e:          # the numbers still print; the card stays unnamed
        res["gpu"] = "unknown (%s)" % e
    print(json.dumps(res))


if __name__ == "__main__":
    main()

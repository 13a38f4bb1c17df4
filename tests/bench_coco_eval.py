"""COCO evaluation: the device path (detectorch_b200.utils.coco_eval) against the reference's pycocotools COCOeval (oracle/_ref, built
by oracle/build_cocoapi.sh), on a minival-sized synthetic workload: 5000 images of 480 x 640, ~7 rectangle-polygon GTs and 100
detections each (two near each GT) over 80 categories, for 'bbox' and 'segm'.  The two arms alternate; the device arm times the GT build (once per
dataset) apart from each evaluation, and the host-side results conversion inside an evaluation on its own; the oracle arm times loadRes and evaluate() + accumulate().  Every oracle run is also checked
bit for bit against the device run.  Prints one JSON line (with the card's name and power limit); writes nothing unless --out.
    python tests/bench_coco_eval.py [--images 5000] [--reps 2] [--oracle-reps 1] [--out FILE]"""
import argparse
import contextlib
import copy
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

H, W, NGT, NDET, NCAT = 480, 640, 7, 100, 80


def _rect_string(x0, x1, y0, y1):
    """rleToString of the column-major RLE of the rectangle [x0, x1) x [y0, y1) on an H x W canvas: counts [x0 H + y0, h, H - h, h, ...,
    rest]; past the third count every delta against counts[i - 2] is 0 except the last."""
    from oracle import ref
    h, n = y1 - y0, x1 - x0
    head = [x0 * H + y0, h, H - h]
    last = H * W - (x0 * H + y0) - n * h - (n - 1) * (H - h)
    if n == 1:
        return ref.rle_to_string([head[0], h, last])
    body = ref.rle_to_string(head) + b"0" * (2 * n - 1 - 3 + 1)
    return body + ref.rle_to_string([0, 0, 0, last - (H - h)])[3:]     # counts[2 n - 2] is a gap of H - h


def make_workload(n_img, seed=0):
    rng = np.random.RandomState(seed)
    images = [dict(id=i + 1, height=H, width=W) for i in range(n_img)]
    anns, boxes = [], [[[] for _ in range(n_img)] for _ in range(NCAT + 1)]
    segms = [[[] for _ in range(n_img)] for _ in range(NCAT + 1)]
    for i in range(n_img):
        x0, y0 = rng.randint(0, W - 100, NDET), rng.randint(0, H - 100, NDET)
        x1, y1 = x0 + rng.randint(10, 100, NDET), y0 + rng.randint(10, 100, NDET)
        sc = rng.rand(NDET).astype(np.float32)
        cls = rng.randint(1, NCAT + 1, NDET)
        for g in range(NGT):
            x, y = rng.uniform(0, W - 100), rng.uniform(0, H - 100)
            w, h = rng.uniform(10, 100), rng.uniform(10, 100)
            c = int(rng.randint(1, NCAT + 1))
            anns.append(dict(id=len(anns) + 1, image_id=i + 1, category_id=c, bbox=[x, y, w, h], area=w * h,
                             iscrowd=0, segmentation=[[x, y, x + w, y, x + w, y + h, x, y + h]]))
            # two detections per GT lie near it (the rest are false positives), so matching does real work
            for d in (2 * g, 2 * g + 1):
                x0[d], y0[d] = int(x) + rng.randint(-4, 5), int(y) + rng.randint(-4, 5)
                x1[d], y1[d] = x0[d] + max(int(w) + rng.randint(-4, 5), 1), y0[d] + max(int(h) + rng.randint(-4, 5), 1)
                x0[d], y0[d] = max(x0[d], 0), max(y0[d], 0)
                x1[d], y1[d] = min(x1[d], W), min(y1[d], H)
                cls[d] = c
        for j in np.unique(cls):
            m = np.flatnonzero(cls == j)
            boxes[j][i] = np.stack([x0[m], y0[m], x1[m] - 1, y1[m] - 1, sc[m]], 1).astype(np.float32)
            segms[j][i] = [dict(size=[H, W], counts=_rect_string(x0[k], x1[k], y0[k], y1[k]).decode()) for k in m]
    ds = dict(images=images, annotations=anns, categories=[dict(id=c, name="c%d" % c) for c in range(1, NCAT + 1)])
    return ds, boxes, segms


def _check_rect_strings():
    from oracle import ref
    rng = np.random.RandomState(1)
    for _ in range(50):
        x0, y0 = rng.randint(0, W - 100), rng.randint(0, H - 100)
        x1, y1 = x0 + rng.randint(1, 100), y0 + rng.randint(1, 100)
        m = np.zeros((H, W), np.uint8)
        m[y0:y1, x0:x1] = 1
        assert _rect_string(x0, x1, y0, y1) == ref.rle_to_string(ref.rle_encode(m))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        name, pl = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, pl
    except Exception as e:          # noqa: BLE001 - reported, not fatal
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=2, help="device evaluations per iou type and round")
    ap.add_argument("--oracle-reps", type=int, default=1, help="rounds of (device, oracle) alternation; 0 skips the oracle arm")
    ap.add_argument("--out", help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_coco_eval: needs a CUDA device")
    from detectorch_b200.utils import coco_eval
    import coco_eval_cases as cc
    from oracle import cocoapi
    _check_rect_strings()
    t0 = time.perf_counter()
    ds, boxes, segms = make_workload(args.images)
    gen_s = time.perf_counter() - t0
    torch.cuda.synchronize()
    # warm-up on a small slice (module load, first launches), then the timed GT build
    wds, wb, ws = make_workload(20, seed=9)
    wg = coco_eval.CocoGroundTruth(wds)
    coco_eval.evaluate(wg, wb, 'bbox'); coco_eval.evaluate(wg, wb, 'segm', ws)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gt = coco_eval.CocoGroundTruth(ds)
    torch.cuda.synchronize()
    gt_s = time.perf_counter() - t0
    res = dict(workload="%d images %dx%d, %d GTs + %d detections each, %d categories" % (args.images, H, W, NGT, NDET, NCAT),
               gpu=card()[0], power_limit=card()[1], generate_s=round(gen_s, 2), device_gt_build_s=round(gt_s, 4))
    have_oracle = args.oracle_reps > 0 and cocoapi.available()
    mods = cocoapi.load() if have_oracle else None
    for t in ('bbox', 'segm'):
        dev_s, orc = [], []
        rounds = max(args.oracle_reps, 1)
        for r in range(rounds):
            for _ in range(args.reps):
                t0 = time.perf_counter()
                E = coco_eval.evaluate(gt, boxes, t, segms if t == 'segm' else None)
                dev_s.append(time.perf_counter() - t0)
            if have_oracle:
                COCO, COCOeval, _ = mods
                res_list = cc.results_file(ds, boxes, segms, t)
                with contextlib.redirect_stdout(io.StringIO()):
                    g = COCO(); g.dataset = copy.deepcopy(ds); g.createIndex()
                    t0 = time.perf_counter(); dt = g.loadRes(res_list); t1 = time.perf_counter()
                    O = COCOeval(g, dt, t); O.evaluate(); t2 = time.perf_counter(); O.accumulate(); t3 = time.perf_counter()
                    O.summarize()
                orc.append(dict(loadRes_s=round(t1 - t0, 3), evaluate_s=round(t2 - t1, 3), accumulate_s=round(t3 - t2, 3)))
                same = all(np.array_equal(E.eval[k], O.eval[k]) for k in ('precision', 'recall', 'scores')) and \
                    np.array_equal(E.stats, np.array(O.stats))
                res[t + "_bit_identical"] = bool(same) and res.get(t + "_bit_identical", True)
        t0 = time.perf_counter()
        coco_eval._flatten_results(gt, boxes, segms if t == 'segm' else None, t, gt.category_ids)
        res[t + "_host_conversion_s"] = round(time.perf_counter() - t0, 4)      # part of each device evaluation above
        res[t + "_AP"] = float(E.stats[0])
        res[t + "_device_eval_s"] = [round(x, 4) for x in dev_s]
        if orc:
            res[t + "_oracle"] = orc
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

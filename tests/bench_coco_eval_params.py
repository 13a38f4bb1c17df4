"""COCO evaluation with COCOeval's Params on the device (evaluate(..., params=)) against the reference's pycocotools COCOeval
(oracle/_ref, built by oracle/build_cocoapi.sh) run with the same Params, on tests/bench_coco_eval.py's workload (5000 images x 100
detections, 80 categories): the default Params, a 500-image subset and useCats = 0, for 'bbox' and 'segm'.  Device and reference runs
alternate; each device run is checked bit for bit against the reference run of its round.  Prints one JSON line with the card's name and
power limit and the median time of each arm (progress lines before it start with '#'); writes nothing.
    python tests/bench_coco_eval_params.py [--images 5000] [--reps 3] [--oracle-reps 1]"""
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench_coco_eval as bce  # noqa: E402
import coco_eval_cases as cc  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-reps", type=int, default=1)
    a = ap.parse_args()
    from detectorch_b200.utils import coco_eval
    from oracle import cocoapi
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    ds, boxes, segms = bce.make_workload(a.images)
    gt = coco_eval.CocoGroundTruth(ds)
    rng = np.random.RandomState(0)
    subset = sorted(int(v) for v in rng.choice(gt.img_ids, min(500, len(gt.img_ids)), replace=False))
    variants = {"default": (gt.img_ids, gt.cat_ids, 1), "500 images": (subset, gt.cat_ids, 1), "useCats 0": (gt.img_ids, gt.cat_ids, 0)}
    COCO, COCOeval, _ = cocoapi.load()
    times, out = {}, dict(card=_card(), images=a.images, detections_per_image=bce.NDET, categories=bce.NCAT)
    for t in ('bbox', 'segm'):
        res = cc.results_file(ds, boxes, segms, t)
        s = segms if t == 'segm' else None
        for name, (imgs, cats, uc) in variants.items():
            p = coco_eval.Params(gt, t)
            p.imgIds, p.catIds, p.useCats = list(imgs), list(cats), uc
            coco_eval.evaluate(gt, boxes, t, s, params=p)                   # warm-up
            for r in range(max(a.reps, a.oracle_reps)):
                if r < a.reps:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    got = coco_eval.evaluate(gt, boxes, t, s, params=p)
                    torch.cuda.synchronize()
                    times.setdefault((t, name, "device"), []).append(time.perf_counter() - t0)
                    print("# %s %s device %.3f s" % (t, name, times[(t, name, "device")][-1]), flush=True)
                if r < a.oracle_reps:
                    with contextlib.redirect_stdout(io.StringIO()):
                        g = COCO()
                        g.dataset = copy.deepcopy(ds)
                        g.createIndex()
                        t0 = time.perf_counter()
                        E = COCOeval(g, g.loadRes(copy.deepcopy(res)), t)
                        E.params.imgIds, E.params.catIds, E.params.useCats = list(imgs), list(cats), uc
                        E.evaluate()
                        E.accumulate()
                        times.setdefault((t, name, "reference"), []).append(time.perf_counter() - t0)
                    print("# %s %s reference %.1f s" % (t, name, times[(t, name, "reference")][-1]), flush=True)
                    for k in ('precision', 'recall', 'scores'):
                        assert np.array_equal(got.eval[k], E.eval[k]), (t, name, k)
    out["seconds"] = {"%s %s %s" % k: float(np.median(v)) for k, v in times.items()}
    out["runs"] = {"%s %s %s" % k: len(v) for k, v in times.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

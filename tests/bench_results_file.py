"""Reading and evaluating COCO results files: bench_device_results' workload A (5000 images x 100 detections, 80 categories, fed as
detect()-shaped batches of 8 to a DeviceResults), written by write_results as the 'bbox' and the 'segm' results file, then three arms
on each file:
  load       coco_eval.load_results(gt, file), ending in a device synchronise
  device     load_results + evaluate(gt, loaded, t)
  ref        the reference's pycocotools (oracle/_ref): COCO.loadRes(file) + COCOeval(G, ., t).evaluate() + accumulate()
The arms alternate; medians of --reps runs; every run checks the device evaluation equal (np.array_equal) to the reference's.
Files go to a temporary directory.  Prints one JSON line with the card's name and power limit and the file sizes.
    python tests/bench_results_file.py [--images 5000] [--reps 3] [--types bbox segm]"""
import argparse
import contextlib
import copy
import io
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench_coco_eval as bce              # noqa: E402
import bench_device_results as bdr         # noqa: E402
from bench_results_json import card        # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--types", nargs="+", default=["bbox", "segm"], choices=["bbox", "segm"])
    a = ap.parse_args()
    from detectorch_b200.utils import coco_eval
    from oracle import cocoapi
    COCO, COCOeval, _ = cocoapi.load()
    dev = torch.device("cuda:0")
    B = bdr.BATCH
    ds, boxes, scores, classes = bdr.workload_a(a.images)
    gt = coco_eval.CocoGroundTruth(ds)
    with contextlib.redirect_stdout(io.StringIO()):
        G = COCO()
        G.dataset = copy.deepcopy(ds)
        G.createIndex()
    bx, sc, cl = (torch.from_numpy(x).to(dev) for x in (boxes, scores, classes))
    counts = torch.full((B,), bce.NDET, dtype=torch.int32, device=dev)
    ones = torch.ones((B, bce.NDET, 28, 28), dtype=torch.float32, device=dev)
    orig = np.array([[bce.H, bce.W]] * B, np.float64)

    def acc_of(t):
        acc = coco_eval.DeviceResults(dev)
        for s in range(0, a.images - a.images % B, B):
            out = {"boxes": bx[s:s + B], "scores": sc[s:s + B], "classes": cl[s:s + B], "counts": counts}
            if t == 'segm':
                out["masks"] = ones
            acc.add(out, list(range(s + 1, s + B + 1)), original_sizes=orig)
        return acc

    out = dict(card=card(), images=a.images, dets_per_image=bce.NDET, reps=a.reps)
    with tempfile.TemporaryDirectory() as tmp:
        for t in a.types:
            path = os.path.join(tmp, "%s.json" % t)
            size = coco_eval.write_results(gt, acc_of(t), t, path)
            got = {}

            def load():
                coco_eval.load_results(gt, path)
                torch.cuda.synchronize()

            def device():
                got['E'] = coco_eval.evaluate(gt, coco_eval.load_results(gt, path), t)

            def ref():
                with contextlib.redirect_stdout(io.StringIO()):
                    E = COCOeval(G, G.loadRes(path), t)
                    E.evaluate()
                    E.accumulate()
                got['R'] = E
            arms = dict(load=load, device=device, ref=ref)
            load(), device()                # warm-up (the reference arm has no device state to warm)
            times = {k: [] for k in arms}
            for _ in range(a.reps):
                for k, fn in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times[k].append(time.perf_counter() - t0)
                for k in ('precision', 'recall', 'scores'):
                    assert np.array_equal(got['E'].eval[k], got['R'].eval[k]), (t, k)
            out[t] = dict(file_bytes=size, records=len(coco_eval.load_results(gt, path)),
                          **{k + "_s": round(float(np.median(v)), 4) for k, v in times.items()},
                          device_speedup_vs_ref=round(float(np.median(times['ref']) / np.median(times['device'])), 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()

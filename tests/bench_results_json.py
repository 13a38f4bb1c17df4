"""The COCO results json of bench_device_results' workload A (5000 images x 100 detections, 80 categories, detect()-shaped batches
of 8), 'bbox' and 'segm', three arms:
  device   DeviceResults.add per batch (untimed), then write_results(gt, acc, ...)
  list     batch_results per batch (untimed), then write_results(gt, per_image_results, ...)
  ref      batch_results per batch (untimed), then the reference writers' list of dicts + json.dump
The arms alternate; medians of --reps runs; the three files are compared byte for byte on every run.  Files go to a temporary
directory.  Prints one JSON line with the card's name and power limit and the file sizes.
    python tests/bench_results_json.py [--images 5000] [--reps 3]"""
import argparse
import json
import os
import subprocess
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
import results_json_cases as rj            # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not measured"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from detectorch_b200.utils import coco_eval, result_utils
    dev = torch.device("cuda:0")
    B = bdr.BATCH
    ds, boxes, scores, classes = bdr.workload_a(a.images)
    gt = coco_eval.CocoGroundTruth(ds)
    bx, sc, cl = (torch.from_numpy(x).to(dev) for x in (boxes, scores, classes))
    counts = torch.full((B,), bce.NDET, dtype=torch.int32, device=dev)
    ones = torch.ones((B, bce.NDET, 28, 28), dtype=torch.float32, device=dev)
    orig = np.array([[bce.H, bce.W]] * B, np.float64)
    starts = range(0, a.images - a.images % B, B)
    empty = (np.zeros(0, np.float32), np.zeros((0, 4), np.float32), [[]] * 81, [[]] * 81)

    def batch(s, masks):
        out = {"boxes": bx[s:s + B], "scores": sc[s:s + B], "classes": cl[s:s + B], "counts": counts}
        if masks:
            out["masks"] = ones
        return out

    def per_image(t):
        res = []
        for s in starts:
            res += result_utils.batch_results(batch(s, t == 'segm'), orig)
        return res + [empty] * (a.images % B)

    def acc_of(t):
        acc = coco_eval.DeviceResults(dev)
        for s in starts:
            acc.add(batch(s, t == 'segm'), list(range(s + 1, s + B + 1)), original_sizes=orig)
        torch.cuda.synchronize()
        return acc

    out = dict(card=card(), images=a.images, dets_per_image=bce.NDET, reps=a.reps)
    with tempfile.TemporaryDirectory() as tmp:
        for t in ('bbox', 'segm'):
            acc, res = acc_of(t), per_image(t)
            all_boxes, all_segms = rj.per_class(res, gt.num_images)
            cats = gt.category_ids
            paths = {k: os.path.join(tmp, "%s_%s.json" % (t, k)) for k in ('device', 'list', 'ref')}

            def ref_arm():
                text = rj.reference_text(gt.img_ids, cats, all_boxes, all_segms, t)
                with open(paths['ref'], 'wb') as f:
                    f.write(text)
            arms = dict(device=lambda: coco_eval.write_results(gt, acc, t, paths['device']),
                        list=lambda: coco_eval.write_results(gt, res, t, paths['list']), ref=ref_arm)
            for fn in arms.values():        # warm-up
                fn()
            times = {k: [] for k in arms}
            for _ in range(a.reps):
                for k, fn in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times[k].append(time.perf_counter() - t0)
                data = [open(p, 'rb').read() for p in paths.values()]
                assert data[0] == data[1] == data[2], t
            out[t] = dict(bytes=len(data[0]), records=int(sum(len(r[0]) for r in res)),
                          **{k + "_s": round(float(np.median(v)), 4) for k, v in times.items()},
                          device_speedup_vs_ref=round(float(np.median(times['ref']) / np.median(times['device'])), 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()

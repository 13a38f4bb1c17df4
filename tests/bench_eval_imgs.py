"""Per-image records (evaluate(..., keep_eval_imgs=True)) on bench_coco_eval's workload: 5000 images of 480 x 640, ~7 GTs and 100
detections each over 80 categories, 'bbox' and 'segm'.  Three device arms alternate in each round: evaluate() without records,
with records kept as columns (.eval_imgs), and with the list of dicts materialised (.evalImgs read); the time of the
dt_coco_eval_imgs launch (CUDA events) and of the host's column assembly are recorded apart.  The oracle arm times the reference's
COCOeval.evaluate() on the same results and checks its evalImgs against the device's, record by record.  Prints one JSON line (with the
card's name and power limit); writes nothing unless --out.
    python tests/bench_eval_imgs.py [--images 5000] [--rounds 3] [--oracle 1] [--out FILE]"""
import argparse
import contextlib
import copy
import io
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_coco_eval import NCAT, NDET, NGT, H, W, card, make_workload  # noqa: E402


class _Timed:
    """The loaded library with dt_coco_eval_imgs bracketed by CUDA events (kernel time, read when the evaluation has finished)."""

    def __init__(self, L):
        self.L, self.events = L, []

    def __getattr__(self, name):
        f = getattr(self.L, name)
        if name != "dt_coco_eval_imgs":
            return f

        def timed(*a):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = f(*a)
            e1.record()
            self.events.append((e0, e1))
            return r
        return timed


def _same(got, want):
    """-> number of records compared; raises on the first difference."""
    assert len(got) == len(want)
    n = 0
    for a, b in zip(got, want):
        assert (a is None) == (b is None)
        if a is None:
            continue
        assert a.keys() == b.keys()
        for k in ('image_id', 'category_id', 'aRng', 'maxDet', 'dtIds', 'gtIds', 'dtScores'):
            assert a[k] == b[k], k
        for k in ('dtMatches', 'gtMatches', 'gtIgnore', 'dtIgnore'):
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), k
        n += 1
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--rounds", type=int, default=3, help="rounds of the three alternating device arms per iou type")
    ap.add_argument("--oracle", type=int, default=1, help="1: time COCOeval.evaluate() once per iou type and compare its evalImgs")
    ap.add_argument("--out", help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_imgs: needs a CUDA device")
    from detectorch_b200 import _lib
    from detectorch_b200.utils import coco_eval
    import coco_eval_cases as cc
    from oracle import cocoapi
    ds, boxes, segms = make_workload(args.images)
    wds, wb, ws = make_workload(20, seed=9)                 # warm-up: module load, first launches of every arm
    wg = coco_eval.CocoGroundTruth(wds)
    for t in ('bbox', 'segm'):
        coco_eval.evaluate(wg, wb, t, ws if t == 'segm' else None, keep_eval_imgs=True).evalImgs
    gt = coco_eval.CocoGroundTruth(ds)
    torch.cuda.synchronize()
    lib = _Timed(_lib.lib())
    _lib.lib, plain_lib = (lambda: lib), _lib.lib
    columns_s = []
    plain_columns = coco_eval._eval_imgs_columns

    def timed_columns(*a):
        t0 = time.perf_counter()
        r = plain_columns(*a)
        columns_s.append(time.perf_counter() - t0)
        return r
    coco_eval._eval_imgs_columns = timed_columns
    name, power = card()
    res = dict(workload="%d images %dx%d, %d GTs + %d detections each, %d categories" % (args.images, H, W, NGT, NDET, NCAT),
               gpu=name, power_limit=power)
    have_oracle = args.oracle > 0 and cocoapi.available()
    mods = cocoapi.load() if have_oracle else None
    try:
        for t in ('bbox', 'segm'):
            s = segms if t == 'segm' else None
            arms = dict(plain=[], columns=[], materialised=[])
            lib.events.clear(); columns_s.clear()
            base = None
            for _ in range(args.rounds):
                t0 = time.perf_counter()
                E0 = coco_eval.evaluate(gt, boxes, t, s)
                arms['plain'].append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                E1 = coco_eval.evaluate(gt, boxes, t, s, keep_eval_imgs=True)
                arms['columns'].append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                E2 = coco_eval.evaluate(gt, boxes, t, s, keep_eval_imgs=True)
                recs = E2.evalImgs
                arms['materialised'].append(time.perf_counter() - t0)
                base = base or E0
                assert all(np.array_equal(E.eval[k], base.eval[k]) for E in (E0, E1, E2) for k in ('precision', 'recall', 'scores'))
            kernel_ms = [e0.elapsed_time(e1) for e0, e1 in lib.events]
            med = lambda v: round(float(np.median(v)), 4)
            res[t] = dict({k + "_s": [round(x, 4) for x in v] for k, v in arms.items()}, **{k + "_median_s": med(v) for k, v in arms.items()},
                          eval_imgs_kernel_ms=[round(x, 3) for x in kernel_ms], columns_host_s=[round(x, 4) for x in columns_s],
                          records=int(len(E1.eval_imgs['index'])), list_length=len(recs), AP=float(E0.stats[0]))
            if have_oracle:
                COCO, COCOeval, _ = mods
                with contextlib.redirect_stdout(io.StringIO()):
                    g = COCO(); g.dataset = copy.deepcopy(ds); g.createIndex()
                    O = COCOeval(g, g.loadRes(cc.results_file(ds, boxes, segms, t)), t)
                    t0 = time.perf_counter(); O.evaluate(); res[t]["cocoeval_evaluate_s"] = round(time.perf_counter() - t0, 2)
                res[t]["records_equal_cocoeval"] = _same(recs, O.evalImgs)
                del O, g
    finally:
        _lib.lib, coco_eval._eval_imgs_columns = plain_lib, plain_columns
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""COCO evaluation of detect() batches: per-image host results (batch_results + evaluate) against results kept on the device
(DeviceResults.add + evaluate), bit-identical on every run.
  A  bench_coco_eval's minival-sized workload (5000 images of 480 x 640, 7 rectangle-polygon GTs and 100 detections each over 80
     categories) fed as detect()-shaped device batches of 8; the masks are all-ones 28 x 28 maps, so each paste covers its box.
     host arm: batch_results per batch, then evaluate(gt, results, t); device arm: acc.add per batch, then evaluate(gt, acc, t).
     'bbox' feeds the batches without masks.  The arms alternate; medians of --reps runs.
  B  the synthetic-weight Mask R-CNN R-50-FPN on photo-sized images in 800 x 1344 / 1344 x 800 canvases (as tests/bench_results.py):
     detect_images + evaluate (bbox and segm) against images_to_batch + detect + add + evaluate, in img/s.
Prints one JSON line with the card's name and power limit; writes nothing unless --out.
    python tests/bench_device_results.py [--images 5000] [--reps 3] [--photos 48] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench_coco_eval as bce          # noqa: E402
import bench_results as br             # noqa: E402

BATCH = 8


def workload_a(n_img, seed=0):
    """bench_coco_eval.make_workload's images, GTs and detections, the detections as one detect()-shaped slot table per image (classes
    ascending, each class's detections in generation order)."""
    rng = np.random.RandomState(seed)
    H, W, NGT, NDET, NCAT = bce.H, bce.W, bce.NGT, bce.NDET, bce.NCAT
    images = [dict(id=i + 1, height=H, width=W) for i in range(n_img)]
    anns = []
    boxes = np.zeros((n_img, NDET, 4), np.float32)
    scores = np.zeros((n_img, NDET), np.float32)
    classes = np.zeros((n_img, NDET), np.int32)
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
            for d in (2 * g, 2 * g + 1):
                x0[d], y0[d] = int(x) + rng.randint(-4, 5), int(y) + rng.randint(-4, 5)
                x1[d], y1[d] = x0[d] + max(int(w) + rng.randint(-4, 5), 1), y0[d] + max(int(h) + rng.randint(-4, 5), 1)
                x0[d], y0[d] = max(x0[d], 0), max(y0[d], 0)
                x1[d], y1[d] = min(x1[d], W), min(y1[d], H)
                cls[d] = c
        o = np.argsort(cls, kind='stable')
        boxes[i] = np.stack([x0, y0, x1 - 1, y1 - 1], 1)[o]
        scores[i], classes[i] = sc[o], cls[o]
    ds = dict(images=images, annotations=anns, categories=[dict(id=c, name="c%d" % c) for c in range(1, NCAT + 1)])
    return ds, boxes, scores, classes


def same(a, b):
    return all(np.array_equal(a.eval[k], b.eval[k]) for k in ('precision', 'recall', 'scores')) and np.array_equal(a.stats, b.stats)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def bench_a(n_img, reps):
    from detectorch_b200.utils import coco_eval, result_utils
    dev = torch.device("cuda:0")
    ds, boxes, scores, classes = workload_a(n_img)
    gt = coco_eval.CocoGroundTruth(ds)
    bx, sc, cl = (torch.from_numpy(x).to(dev) for x in (boxes, scores, classes))
    counts = torch.full((BATCH,), bce.NDET, dtype=torch.int32, device=dev)
    ones = torch.ones((BATCH, bce.NDET, 28, 28), dtype=torch.float32, device=dev)
    orig = np.array([[bce.H, bce.W]] * BATCH, np.float64)
    starts = range(0, n_img - n_img % BATCH, BATCH)

    def batch(s, masks):
        out = {"boxes": bx[s:s + BATCH], "scores": sc[s:s + BATCH], "classes": cl[s:s + BATCH], "counts": counts}
        if masks:
            out["masks"] = ones
        return out

    def host(t):
        res = []
        for s in starts:
            res += result_utils.batch_results(batch(s, t == 'segm'), orig)
        res += [(np.zeros(0, np.float32), np.zeros((0, 4), np.float32), [[]] * 81, [[]] * 81)] * (n_img % BATCH)
        t0 = time.perf_counter()
        E = coco_eval.evaluate(gt, res, t)
        return E, time.perf_counter() - t0

    def device(t):
        acc = coco_eval.DeviceResults(dev)
        for s in starts:
            acc.add(batch(s, t == 'segm'), list(range(s + 1, s + BATCH + 1)), original_sizes=orig)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        E = coco_eval.evaluate(gt, acc, t)
        return E, time.perf_counter() - t0

    for t in ('bbox', 'segm'):                        # warm-up: every kernel and allocation once
        assert same(host(t)[0], device(t)[0])
    res = {}
    for t in ('bbox', 'segm'):
        hs, ds_, he, de = [], [], [], []
        for _ in range(reps):
            th, (Eh, eh) = timed(lambda: host(t))
            td, (Ed, ed) = timed(lambda: device(t))
            assert same(Eh, Ed), t
            hs.append(th); ds_.append(td); he.append(eh); de.append(ed)
        res[t] = dict(host_s=round(float(np.median(hs)), 4), device_s=round(float(np.median(ds_)), 4),
                      host_evaluate_s=round(float(np.median(he)), 4), device_evaluate_s=round(float(np.median(de)), 4),
                      speedup=round(float(np.median(hs) / np.median(ds_)), 2), AP=float(Ed.stats[0]),
                      host_each_s=[round(x, 4) for x in hs], device_each_s=[round(x, 4) for x in ds_])
    return res


def bench_b(n_photos, reps):
    from detectorch_b200.utils import blob, coco_eval
    from oracle import network as net
    model = br.make_model(net.synthetic_params("resnet50"), emit_full_masks=False, det_cap=100)
    rng = np.random.RandomState(0)
    shapes = [br.PHOTO_SIZES[i] for i in rng.randint(0, len(br.PHOTO_SIZES), n_photos)]
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    batches = []
    for g in ("landscape", "portrait"):
        idx = [i for i, (h, w) in enumerate(shapes) if (h <= w) == (g == "landscape")]
        for s in range(0, len(idx) - BATCH + 1, BATCH):
            batches.append((idx[s:s + BATCH], br.CANVAS[g]))
    used = sorted(i for part, _ in batches for i in part)

    def host():
        res = {}
        for part, canvas in batches:
            res.update(zip(part, model.detect_images([ims[i] for i in part], canvas=canvas)))
        results = [res[i] for i in used]
        return [coco_eval.evaluate(gt, results, t) for t in ('bbox', 'segm')], results

    def device():
        acc = coco_eval.DeviceResults()
        for part, canvas in batches:
            data, sizes, scales, orig = blob.images_to_batch([ims[i] for i in part], canvas=canvas)
            out = model.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
            acc.add(out, [i + 1 for i in part], original_sizes=orig)
        return [coco_eval.evaluate(gt, acc, t) for t in ('bbox', 'segm')]

    # the ground truth: jittered copies of the first pass's detections (three per image and class), so that matching does real work
    gt = None
    res = {}
    for part, canvas in batches:
        res.update(zip(part, model.detect_images([ims[i] for i in part], canvas=canvas)))
    anns = []
    for i in used:
        for j in range(1, 81):
            for b in np.asarray(res[i][2][j]).reshape(-1, 5)[:3]:
                x, y = float(b[0]) + rng.uniform(-3, 3), float(b[1]) + rng.uniform(-3, 3)
                w, h = float(b[2] - b[0]) + rng.uniform(-3, 3), float(b[3] - b[1]) + rng.uniform(-3, 3)
                anns.append(dict(id=len(anns) + 1, image_id=i + 1, category_id=j, bbox=[x, y, w, h], area=max(w * h, 0.), iscrowd=0,
                                 segmentation=[[x, y, x + w, y, x + w, y + h, x, y + h]]))
    ds = dict(images=[dict(id=i + 1, height=shapes[i][0], width=shapes[i][1]) for i in used], annotations=anns,
              categories=[dict(id=c, name="c%d" % c) for c in range(1, 81)])
    gt = coco_eval.CocoGroundTruth(ds)
    (hb, hs), _ = host()
    db, dsg = device()
    assert same(hb, db) and same(hs, dsg)
    th, td = [], []
    for _ in range(reps):
        t, ((hb, hs), _) = timed(host)
        th.append(t)
        t, (db, dsg) = timed(device)
        td.append(t)
        assert same(hb, db) and same(hs, dsg)
    n = len(used)
    return dict(images=n, batch=BATCH, detections=int(sum(len(res[i][0]) for i in used)), bbox_AP=float(db.stats[0]), segm_AP=float(dsg.stats[0]),
                detect_images_evaluate_img_per_s=round(n / float(np.median(th)), 2), detect_add_evaluate_img_per_s=round(n / float(np.median(td)), 2),
                speedup=round(float(np.median(th) / np.median(td)), 3),
                host_each_s=[round(x, 4) for x in th], device_each_s=[round(x, 4) for x in td])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000, help="workload A images")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--photos", type=int, default=48, help="workload B images (0 skips it)")
    ap.add_argument("--out", help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_results: needs a CUDA device")
    name, pl = bce.card()
    res = dict(gpu=name, power_limit=pl, workload_a=dict(images=a.images, batch=BATCH, **bench_a(a.images, a.reps)))
    if a.photos:
        res["workload_b"] = bench_b(a.photos, a.reps)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

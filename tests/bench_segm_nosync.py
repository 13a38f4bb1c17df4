"""Masked DeviceResults.add with and without a host synchronisation per batch, alternated in one session, results bit-identical.
  sync arm    the add of the previous release: ops.segm_rle_batch_device reads the run overflow and the string offsets back (one
              synchronisation per batch), the strings are copied into the char buffer at the host-known length
  nosync arm  DeviceResults.add: ops.segm_rle_batch_append at the device cursor, overflows settled later from a ring of batches
  A  tests/bench_device_results.py's workload A, 'segm': 5000 images of 480 x 640 with 100 detections of all-ones 28 x 28 masks, added
     in device batches of 8, then evaluate(gt, acc, 'segm'); seconds for adds + evaluate.
  B  its workload B: the synthetic-weight Mask R-CNN R-50-FPN on photo-sized images, images_to_batch + detect + add per batch of 8, then
     evaluate 'bbox' and 'segm'; img/s.
Medians of --reps runs per arm; prints one JSON line with the card's name and power limit; writes nothing unless --out.
    python tests/bench_segm_nosync.py [--images 5000] [--reps 5] [--photos 48] [--out FILE]"""
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
import bench_device_results as bdr     # noqa: E402
import bench_results as br             # noqa: E402


def sync_results_class():
    from detectorch_b200 import _lib, ops
    from detectorch_b200.utils import coco_eval

    class SyncResults(coco_eval.DeviceResults):
        """DeviceResults whose masked add synchronises once per batch, as the previous release's did."""

        def add(self, out, image_ids, original_sizes=None, num_classes=81):
            if out.get('masks') is None:
                return super().add(out, image_ids, original_sizes, num_classes)
            boxes, scores, classes, counts, masks = out['boxes'], out['scores'], out['classes'], out['counts'], out['masks']
            B, cap = int(boxes.size(0)), int(boxes.size(1))
            ids = [int(v) for v in image_ids]
            sizes = ops.segm_image_sizes(original_sizes, B)
            o0, n0, base = len(self.image_ids), self._num_records, self._chars_used
            L = _lib.lib()
            with torch.cuda.device(self.device):
                strings, host = ops.segm_rle_batch_device(masks, None, boxes, counts, sizes)
                nch = int(host[0][-1])
                self._reserve(n0 + B * cap)
                if nch and (self._chars is None or base + nch > self._chars.shape[0]):
                    c = torch.empty((max(base + nch, 2 * (0 if self._chars is None else self._chars.shape[0]), self._MIN_CHARS),),
                                    dtype=torch.uint8, device=self.device)
                    if base:
                        c[:base].copy_(self._chars[:base])
                    self._chars = c
                if nch:
                    self._chars[base:base + nch].copy_(strings[:nch])
                offs_d = coco_eval._pinned_upload(host[0].astype(np.int64), self.device)
                table = np.concatenate([np.arange(o0, o0 + B, dtype=np.int64)[:, None], sizes.astype(np.int64)], 1)
                img_d = coco_eval._pinned_upload(table, self.device)
                bx, sc = boxes.contiguous().float(), scores.contiguous().float()
                cl, ct = classes.contiguous().to(torch.int32), counts.contiguous().to(torch.int32)
                _lib.check(L.dt_coco_results_append(B, cap, num_classes, coco_eval._p(bx), coco_eval._p(sc), coco_eval._p(cl), coco_eval._p(ct),
                                                    coco_eval._p(img_d), coco_eval._p(offs_d), base, coco_eval._p(self._rec_f[n0:]),
                                                    coco_eval._p(self._rec_i[n0:]), coco_eval._p(self._err), coco_eval._stream(self.device)),
                           "dt_coco_results_append")
            for b, v in enumerate(ids):
                self._ordinal[v] = o0 + b
                self._where.append((b, num_classes))
            self.image_ids += ids
            self._num_records += B * cap
            self._chars_used += nch
            self._num_classes = max(self._num_classes, num_classes)

    return SyncResults


def bench_a(n_img, reps, arms):
    from detectorch_b200.utils import coco_eval
    dev = torch.device("cuda:0")
    ds, boxes, scores, classes = bdr.workload_a(n_img)
    gt = coco_eval.CocoGroundTruth(ds)
    bx, sc, cl = (torch.from_numpy(x).to(dev) for x in (boxes, scores, classes))
    B = bdr.BATCH
    counts = torch.full((B,), bce.NDET, dtype=torch.int32, device=dev)
    ones = torch.ones((B, bce.NDET, 28, 28), dtype=torch.float32, device=dev)
    orig = np.array([[bce.H, bce.W]] * B, np.float64)
    starts = range(0, n_img - n_img % B, B)

    def run(cls):
        acc = cls(dev)
        t0 = time.perf_counter()
        for s in starts:
            acc.add({"boxes": bx[s:s + B], "scores": sc[s:s + B], "classes": cl[s:s + B], "counts": counts, "masks": ones},
                    list(range(s + 1, s + B + 1)), original_sizes=orig)
        t_add = time.perf_counter() - t0
        E = coco_eval.evaluate(gt, acc, 'segm')
        torch.cuda.synchronize()
        return time.perf_counter() - t0, t_add, E, acc._num_chars

    ref = None
    for name, cls in arms:                                  # warm-up, and the arms agree
        _, _, E, nch = run(cls)
        ref = ref or (E, nch)
        assert bdr.same(E, ref[0]) and nch == ref[1], name
    t = {name: [] for name, _ in arms}
    ta = {name: [] for name, _ in arms}
    for _ in range(reps):
        for name, cls in arms:
            torch.cuda.synchronize()
            dt, dt_add, E, nch = run(cls)
            assert bdr.same(E, ref[0]) and nch == ref[1], name
            t[name].append(dt); ta[name].append(dt_add)
    res = {name: dict(total_s=round(float(np.median(t[name])), 4), add_loop_s=round(float(np.median(ta[name])), 4),
                      each_s=[round(x, 4) for x in t[name]]) for name, _ in arms}
    res["speedup"] = round(float(np.median(t["sync"]) / np.median(t["nosync"])), 3)
    res["AP"] = float(ref[0].stats[0])
    return res


def bench_b(n_photos, reps, arms):
    from detectorch_b200.utils import blob, coco_eval
    from oracle import network as net
    model = br.make_model(net.synthetic_params("resnet50"), emit_full_masks=False, det_cap=100)
    rng = np.random.RandomState(0)
    shapes = [br.PHOTO_SIZES[i] for i in rng.randint(0, len(br.PHOTO_SIZES), n_photos)]
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    batches = []
    for g in ("landscape", "portrait"):
        idx = [i for i, (h, w) in enumerate(shapes) if (h <= w) == (g == "landscape")]
        for s in range(0, len(idx) - bdr.BATCH + 1, bdr.BATCH):
            batches.append((idx[s:s + bdr.BATCH], br.CANVAS[g]))
    used = sorted(i for part, _ in batches for i in part)
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

    def run(cls):
        acc = cls()
        for part, canvas in batches:
            data, sizes, scales, orig = blob.images_to_batch([ims[i] for i in part], canvas=canvas)
            out = model.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
            acc.add(out, [i + 1 for i in part], original_sizes=orig)
        return [coco_eval.evaluate(gt, acc, t) for t in ('bbox', 'segm')]

    ref = None
    for name, cls in arms:
        E = run(cls)
        ref = ref or E
        assert all(bdr.same(a, b) for a, b in zip(E, ref)), name
    t = {name: [] for name, _ in arms}
    for _ in range(reps):
        for name, cls in arms:
            dt, E = bdr.timed(lambda: run(cls))
            assert all(bdr.same(a, b) for a, b in zip(E, ref)), name
            t[name].append(dt)
    n = len(used)
    out = {name: dict(img_per_s=round(n / float(np.median(t[name])), 2), each_s=[round(x, 4) for x in t[name]]) for name, _ in arms}
    out.update(images=n, batch=bdr.BATCH, speedup=round(float(np.median(t["sync"]) / np.median(t["nosync"])), 3),
               bbox_AP=float(ref[0].stats[0]), segm_AP=float(ref[1].stats[0]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000, help="workload A images")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--photos", type=int, default=48, help="workload B images (0 skips it)")
    ap.add_argument("--out", help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_segm_nosync: needs a CUDA device")
    from detectorch_b200.utils import coco_eval
    arms = [("sync", sync_results_class()), ("nosync", coco_eval.DeviceResults)]
    name, pl = bce.card()
    res = dict(gpu=name, power_limit=pl, reps=a.reps, workload_a=dict(images=a.images, batch=bdr.BATCH, **bench_a(a.images, a.reps, arms)))
    if a.photos:
        res["workload_b"] = bench_b(a.photos, a.reps, arms)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

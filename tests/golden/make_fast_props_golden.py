"""Regenerates tests/golden/fast_props_golden.npz by running the REFERENCE's own Fast R-CNN proposal preparation (needs the reference tree
and oracle/_ref, see oracle/build_ref.sh; run from the repository root: python tests/golden/make_fast_props_golden.py).

For each seeded case of float32 roidb boxes and a scaling factor it applies what preprocess_sample.__call__ does with fpn_on=True
(preprocess_sample.py:36-45): proposals = boxes * scale, remove_dup_prop (spatial scale 1/16), add_multilevel_rois_for_test.  Stored per
case <c>:
  * <c>_boxes    float32 [n, 4] original-image boxes          <c>_scale     float64 scaling factor
  * <c>_props    float32 [m, 4] deduplicated proposals (hash order, what forward() gets back through roi_original_idx)
  * <c>_levels   int32 [m] FPN level (2..5) of each row of <c>_props
  * <c>_restore  int32 [m] rois_idx_restore_int32
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import reference_shim as rs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fast_props_golden.npz")


def boxes_wh(rng, n, lo, hi, extent=1200.0):
    """n boxes with sides log-uniform in [lo, hi] and aspect ratios in [1/3, 3], anywhere in an extent x extent image."""
    side = np.exp(rng.uniform(np.log(lo), np.log(hi), n))
    ar = np.exp(rng.uniform(np.log(1 / 3.), np.log(3.), n))
    w, h = side * np.sqrt(ar), side / np.sqrt(ar)
    x1, y1 = rng.uniform(0, extent, n), rng.uniform(0, extent, n)
    return np.stack([x1, y1, x1 + w, y1 + h], 1).astype(np.float32)


def cases():
    rng = np.random.RandomState(0)
    c = {}
    # exact duplicates: every third box repeated (some of them twice), shuffled
    b = boxes_wh(rng, 60, 16, 400)
    b = np.concatenate([b, b[::3], b[::9]])[rng.permutation(60 + 20 + 7)]
    c["dups"] = (b, 800 / 480.)
    # near-duplicates: jitter of up to 3 px after scaling, so most of them round to the same /16 cell and some do not
    b = boxes_wh(rng, 40, 32, 300)
    s = 1.25
    j = np.concatenate([b] + [b + (rng.uniform(-3, 3, b.shape) / s).astype(np.float32) for _ in range(3)])
    c["near"] = (np.maximum(j, 0)[rng.permutation(len(j))], s)
    # p / 16 exactly at k + 0.5 for even and odd k (scale 2: box = 8k + 4): 8 -> 0, 24 -> 2, 40 -> 2, 56 -> 4 (round half to even)
    k = np.arange(0, 40)
    half = (8 * k + 4).astype(np.float32)
    rows = []
    for i in range(len(k) - 3):
        rows.append([half[i], half[i + 1], half[i + 2] + 64, half[i + 3] + 64])
        rows.append([half[i] + 8, half[i + 1], half[i + 2] + 64, half[i + 3] + 64])     # one cell over: same hash only for an odd k
    c["half"] = (np.array(rows, np.float32), 2.0)
    # every FPN level and past both clip bounds: sides from 2 px to 2000 px
    c["levels"] = (boxes_wh(rng, 120, 2, 2000), 1.0)
    c["single"] = (boxes_wh(rng, 1, 40, 200), 800 / 612.)
    # a full image: 1000 boxes, a few percent of them duplicates after scaling
    b = boxes_wh(rng, 960, 8, 700, extent=900)
    d = b[rng.choice(960, 40, replace=False)] + (rng.uniform(-2, 2, (40, 4))).astype(np.float32)
    c["full"] = (np.maximum(np.concatenate([b, d]), 0)[rng.permutation(1000)].astype(np.float32), 800 / 375.)
    for name, (b, _) in c.items():
        assert b.dtype == np.float32 and np.all(b[:, 2] >= b[:, 0]) and np.all(b[:, 3] >= b[:, 1]), name
    return c


def main():
    rs.install()
    from utils.multilevel_rois import add_multilevel_rois_for_test
    from utils.preprocess_sample import preprocess_sample
    prep = preprocess_sample(target_sizes=[800], fpn_on=True)
    out = {}
    for name, (boxes, scale) in cases().items():
        proposals = boxes * scale                                       # preprocess_sample.py:36
        proposals, _ = prep.remove_dup_prop(proposals)                  # :38
        blobs = add_multilevel_rois_for_test({'rois': proposals}, 'rois')   # :43
        lv = np.concatenate([np.full(len(blobs['rois_fpn%d' % l]), l) for l in range(2, 6)]).astype(np.int32)
        restore = blobs['rois_idx_restore_int32']
        assert proposals.dtype == np.float32 and len(restore) == len(proposals)
        out[name + "_boxes"], out[name + "_scale"] = boxes, np.float64(scale)
        out[name + "_props"], out[name + "_levels"], out[name + "_restore"] = proposals, lv[restore], restore.astype(np.int32)
        print("%-7s %4d boxes -> %4d unique, levels %s" % (name, len(boxes), len(proposals), np.bincount(lv, minlength=6)[2:]))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()

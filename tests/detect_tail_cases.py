"""Adversarial and randomised inputs for the device detection tail (ST_DETECT: det_class_kernel + det_limit_kernel, the port of
postprocess_output / box_results_with_nms_and_limit, result_utils.py:76-168), one generator per family of inputs where the port
can go wrong, so that a failure names its family:

  threshold  scores at float32(0.05) and one ulp either side: only the upper one passes the strict score > 0.05
  iou        integer RoIs with zero deltas (decoded exactly): pairs whose fp32 IoU is exactly 0.5 in the oracle's operation order
             (suppressed) next to pairs one step below (kept), a pair whose true IoU is below 0.5 but whose fp32 IoU rounds to 0.5,
             greedy chains (A suppresses B, B would suppress C, C survives), many identical boxes
  decode     dw / dh above BBOX_XFORM_CLIP, strongly negative dw (pw -> 0, x2 < x1), boxes decoded wholly outside the image (clipped
             to width-1 lines on the border)
  limit      99 / 100 / 101 kept, ties at rank 100 that fit in det_cap, ties that overflow det_cap while an above-threshold
             detection sits in a later class, one class holding all R candidates
  batch      B = 3 with roi_counts 0, 1 and R, poisoned rows (NaN, 1e30) past roi_counts, scaling factors that are not powers of
             two and distinct original sizes
  sizes      R in {1, 31, 32, 33, 1000, 1024} (1024 fills the class kernel's bitonic sort and its 16-word NMS mask), and every
             class x 1024 RoIs above the threshold (~80k keys in the limit's radix sort)
  classes    num_classes 2 and 128 (the bound of the limit kernel's per-class table)
  fuzz       clustered boxes with scores from a small set of fp32 values: ties within and across classes

Every case is a Case: the teacher-forced inputs of ST_DETECT (rois [B,R,5] at network scale, roi_counts [B], cls_prob [B*R,NC],
bbox_pred [B*R,4NC]), each image's scaling factor and original size, and the properties it is built to have (`claims`), which
tests/test_detect_tail_host.py checks under the oracle.  oracle/ref.expected_device turns a case into the device's expected rows."""
import numpy as np

F32 = np.float32
THRESH = F32(0.05)
BELOW, ABOVE = np.nextafter(THRESH, F32(0)), np.nextafter(THRESH, F32(1))
POISON = (np.nan, F32(1e30), -np.inf, F32(-1e30))


class Case:
    """claims: list of tuples, checked under the stable-order oracle by the host test:
         ("kept", b, j, rois) / ("dropped", b, j, rois)   those RoIs are / are not among class j's detections of image b
         ("iou", b, j, ri, rk, "eq" | "below")            fp32 IoU of the decoded boxes == 0.5 / just below 0.5
         ("iou_rounds", b, j, ri, rk)                     fp32 IoU == 0.5 while the exact IoU is below 0.5
         ("count", b, n)                                  the reference returns n detections
         ("tie_at_limit", b)                              the image threshold is tied: several detections score exactly it
         ("overflow", b)                                  the reference returns more than det_cap and cutting its list at det_cap
                                                          would lose a detection scoring above the threshold
         ("poison", b)                                    every row past roi_counts[b] is non-finite or huge
       exact: zero deltas everywhere, so the device's boxes equal the oracle's bit for bit; otherwise expf against numpy's exp,
       and every same-class IoU keeps 1e-5 away from 0.5.  tie_free: the oracle's result does not depend on the NMS tie order."""

    def __init__(self, family, name, R, NC=81, B=1, det_cap=100, exact=True, tie_free=True, orig_hw=(600, 800)):
        self.family, self.name = family, name
        self.B, self.R, self.NC, self.det_cap = B, R, NC, det_cap
        self.exact, self.tie_free = exact, tie_free
        self.rois = np.zeros((B, R, 5), F32)
        self.rois[:, :, 0] = np.arange(B, dtype=F32)[:, None]
        self.roi_counts = np.full((B,), R, np.int32)
        self.cls_prob = np.zeros((B * R, NC), F32)
        self.bbox_pred = np.zeros((B * R, 4 * NC), F32)
        self.scale = np.ones((B,), F32)
        self.orig_hw = np.tile(np.asarray(orig_hw, F32), (B, 1))
        self.claims = []

    @property
    def id(self):
        return "%s-%s" % (self.family, self.name)

    @property
    def group(self):
        """Cases of one group run on one engine."""
        return (self.B, self.R, self.NC, self.det_cap)

    def box(self, i, xyxy, b=0):
        self.rois[b, i, 1:5] = np.asarray(xyxy, F32)

    def score(self, i, j, s, b=0):
        self.cls_prob[b * self.R + i, j] = F32(s)

    def delta(self, i, j, d, b=0):
        self.bbox_pred[b * self.R + i, 4 * j:4 * j + 4] = np.asarray(d, F32)

    def poison(self, b, rng):
        """Rows at and past roi_counts[b] hold NaN, infinities and huge values, which the device must never read."""
        n, R = int(self.roi_counts[b]), self.R
        if n == R:
            return
        pick = lambda shape: np.asarray(POISON, F32)[rng.randint(0, len(POISON), shape)]
        self.rois[b, n:, 1:5] = pick((R - n, 4))
        self.cls_prob[b * R + n:(b + 1) * R] = pick((R - n, self.NC))
        self.cls_prob[b * R + n:(b + 1) * R:2] = F32(1e30)           # a score the strict > 0.05 would take
        self.bbox_pred[b * R + n:(b + 1) * R] = pick((R - n, 4 * self.NC))
        self.claims.append(("poison", b))


def grid_box(i, size=20, step=30, cols=16, x0=0, y0=0):
    """Non-overlapping integer boxes (step > size)."""
    x, y = x0 + (i % cols) * step, y0 + (i // cols) * step
    return [x, y, x + size - 1, y + size - 1]


def distinct_scores(rng, n, lo=0.06, hi=0.98):
    """n distinct fp32 scores in (lo, hi), shuffled."""
    s = np.linspace(lo, hi, n).astype(F32)
    assert len(np.unique(s)) == n
    return s[rng.permutation(n)]


def clustered_boxes(rng, n, clusters, jitter=3, extent=(560, 760)):
    """Integer boxes around a few centres: heavy overlap, IoUs on and around 0.5."""
    cen = np.stack([rng.randint(0, extent[1] - 120, clusters), rng.randint(0, extent[0] - 120, clusters),
                    rng.randint(12, 100, clusters), rng.randint(12, 100, clusters)], 1)
    c = cen[rng.randint(0, clusters, n)]
    j = rng.randint(-jitter, jitter + 1, (n, 4))
    x1, y1 = c[:, 0] + j[:, 0], c[:, 1] + j[:, 1]
    return np.stack([x1, y1, x1 + np.maximum(c[:, 2] + j[:, 2], 1), y1 + np.maximum(c[:, 3] + j[:, 3], 1)], 1).astype(F32)


# ------------------------------------------------------------------------------------------------ families
def threshold_cases():
    c = Case("threshold", "ulp", 64)
    kept, dropped = {}, {}
    for i in range(48):
        j = 1 + i % 16
        c.box(i, grid_box(i))
        s = (BELOW, THRESH, ABOVE)[i % 3]
        c.score(i, j, s)
        (kept if s == ABOVE else dropped).setdefault(j, []).append(i)
    # three identical boxes in one class: only the one above the threshold is a candidate, so nothing suppresses it
    for k, s in zip(range(48, 51), (THRESH, ABOVE, BELOW)):
        c.box(k, [500, 500, 539, 539])
        c.score(k, 20, s)
    kept[20], dropped[20] = [49], [48, 50]
    for j in kept:
        c.claims += [("kept", 0, j, kept[j]), ("dropped", 0, j, dropped[j])]
    c.claims.append(("count", 0, 17))
    return [c]


def iou_cases():
    out = []
    c = Case("iou", "half_and_below", 64)
    pairs = [  # (class, A, B, relation): A scores higher
        (1, [0, 0, 29, 9], [10, 0, 39, 9], "eq"),              # side by side: inter 200 / union 400
        (2, [0, 0, 19, 9], [0, 0, 9, 9], "eq"),                # nested: 100 / 200
        (3, [0, 0, 9, 9], [0, 0, 19, 9], "eq"),                # nested, the smaller one scores higher
        (4, [0, 0, 76, 12], [0, 0, 49, 9], "below"),           # 500 / 1001: kept
        (5, [300, 200, 349, 209], [300, 200, 376, 212], "below"),
        (6, [0, 0, 26, 36], [0, 0, 19, 24], "above"),          # 500 / 999: suppressed
        (7, [100, 100, 129, 109], [110, 100, 139, 109], "eq"),
        (8, [100, 100, 109, 129], [100, 110, 109, 139], "eq"),  # stacked vertically
    ]
    for k, (j, a, bb, rel) in enumerate(pairs):
        ia, ib = 2 * k, 2 * k + 1
        c.box(ia, a); c.box(ib, bb)
        c.score(ia, j, 0.9 - 0.01 * k); c.score(ib, j, 0.5 - 0.01 * k)
        if rel in ("eq", "below"):
            c.claims.append(("iou", 0, j, ia, ib, rel))
        c.claims.append(("kept", 0, j, [ia, ib] if rel == "below" else [ia]))
        if rel != "below":
            c.claims.append(("dropped", 0, j, [ib]))
    out.append(c)

    # true IoU 2^25 / (2^26 + 1) < 0.5, but the fp32 area of A (8321 x 8065 = 2^26 + 1) rounds to 2^26 and the IoU to exactly 0.5
    c = Case("iou", "fp32_rounds_to_half", 64, orig_hw=(9000, 9000))
    c.box(0, [0, 0, 8320, 8064]); c.box(1, [0, 0, 8191, 4095])
    c.score(0, 1, 0.9); c.score(1, 1, 0.8)
    c.box(2, [0, 0, 8191, 4095]); c.box(3, [0, 0, 8320, 8064])    # the same pair with the smaller box first and higher
    c.score(2, 2, 0.9); c.score(3, 2, 0.8)
    c.claims += [("iou_rounds", 0, 1, 0, 1), ("kept", 0, 1, [0]), ("dropped", 0, 1, [1]),
                 ("iou_rounds", 0, 2, 2, 3), ("kept", 0, 2, [2]), ("dropped", 0, 2, [3])]
    out.append(c)

    # greedy chains: box k = [10k, 0, 10k + 29, 9]; IoU(k, k+1) = 0.5, IoU(k, k+2) = 0.2
    c = Case("iou", "chains", 64)
    rng = np.random.RandomState(3)
    n = 9
    chain = [[10 * k, 0, 10 * k + 29, 9] for k in range(n)]
    for k in range(n):                                   # class 1: scores fall along the chain -> even positions kept
        c.box(k, chain[k]); c.score(k, 1, 0.9 - 0.05 * k)
    c.claims += [("kept", 0, 1, list(range(0, n, 2))), ("dropped", 0, 1, list(range(1, n, 2))), ("iou", 0, 1, 1, 2, "eq")]
    m = n - 1
    for k in range(m):                                   # class 2: scores rise along an even chain -> odd positions kept
        c.box(16 + k, [v + (0, 100)[t % 2] for t, v in enumerate(chain[k])])
        c.score(16 + k, 2, 0.4 + 0.05 * k)
    c.claims += [("kept", 0, 2, [16 + k for k in range(m - 1, -1, -2)]), ("dropped", 0, 2, [16 + k for k in range(m - 2, -1, -2)])]
    perm = rng.permutation(n)                            # class 3: the chain on shuffled RoI indices
    for k in range(n):
        c.box(32 + perm[k], [v + (0, 200)[t % 2] for t, v in enumerate(chain[k])])
        c.score(32 + perm[k], 3, 0.9 - 0.05 * k)
    c.claims += [("kept", 0, 3, [32 + perm[k] for k in range(0, n, 2)]), ("dropped", 0, 3, [32 + perm[k] for k in range(1, n, 2)])]
    out.append(c)

    # many identical boxes (IoU 1): distinct scores keep the best one wherever it sits
    c = Case("iou", "identical", 64)
    s = distinct_scores(rng, 40)
    for i in range(40):
        c.box(i, [40, 50, 139, 129]); c.score(i, 1, s[i])
    best = int(np.argmax(s))
    c.claims += [("kept", 0, 1, [best]), ("dropped", 0, 1, [i for i in range(40) if i != best]), ("count", 0, 1)]
    out.append(c)

    # identical boxes with tied scores: the result depends on the visiting order; (score desc, RoI asc) keeps the first
    c = Case("iou", "identical_tied", 64, tie_free=False)
    for i in range(40):
        c.box(i, [40, 50, 139, 129]); c.score(i, 1, 0.5)
    for i in range(40, 60):                              # two score values, the best ones from RoI 45 on
        c.box(i, [200, 50, 239, 99]); c.score(i, 2, 0.75 if i >= 45 else 0.25)
    c.claims += [("kept", 0, 1, [0]), ("dropped", 0, 1, list(range(1, 40))), ("kept", 0, 2, [45]), ("count", 0, 2)]
    out.append(c)
    return out


def decode_cases():
    c = Case("decode", "clip_and_degenerate", 64, exact=False, orig_hw=(800, 800))
    rng = np.random.RandomState(5)
    s = distinct_scores(rng, 64, 0.1, 0.95)
    kinds = [(0, 0, 30, 0.5),          # dw / 5 = 6 > BBOX_XFORM_CLIP: w grows 62.5x and clips on both sides
             (0, 0, 40, 40),           # both clipped
             (0, 0, -100, 0),          # pw = exp(-20) w ~ 0: x2 = x1 - 1
             (0, 0, -100, -100),
             (1000, 0, 0, 0),          # decoded wholly right of the image: a width-1 line on x = W - 1
             (-1000, 1000, 0, 0)]      # left and below: the corner line x = 0, y = H - 1
    for i in range(60):
        c.box(i, grid_box(i, size=30, step=100, cols=8, x0=10, y0=10))
        c.score(i, 1 + i, s[i])
        c.delta(i, 1 + i, kinds[i % len(kinds)])
    # two boxes decoded outside the image into the same border line (IoU 1) and two on disjoint stretches of it (IoU 0)
    for i, (j, y) in zip(range(60, 64), ((70, 100), (70, 100), (71, 100), (71, 400))):
        c.box(i, [300, y, 339, y + 49])
        c.score(i, j, s[i])
        c.delta(i, j, (1000, 0, 0, 0))
    hi70 = 60 if s[60] > s[61] else 61
    c.claims += [("kept", 0, 70, [hi70]), ("dropped", 0, 70, [121 - hi70]), ("kept", 0, 71, [62, 63]), ("count", 0, 63)]
    return [c]


def _spread(c, rng, scores, first_cls=1, last_cls=80, avoid=()):
    """Detections (RoI, class) on distinct grid boxes, so that none suppresses another; returns [(roi, class)]."""
    slots = [(i, j) for j in range(first_cls, last_cls + 1) for i in range(c.R) if (i, j) not in avoid]
    pick = rng.permutation(len(slots))[:len(scores)]
    out = []
    for k, p in enumerate(pick):
        i, j = slots[p]
        c.box(i, grid_box(i))
        c.score(i, j, scores[k])
        out.append((i, j))
    return out


def limit_cases():
    out = []
    rng = np.random.RandomState(11)
    for n in (99, 100, 101):
        c = Case("limit", "kept_%d" % n, 64)
        _spread(c, rng, distinct_scores(rng, n))
        c.claims.append(("count", 0, min(n, 100)))
        out.append(c)

    # ranks 98..100 tied, rank 101 below: exactly 100 come out
    c = Case("limit", "tie_fills_100", 64)
    t = F32(0.3)
    _spread(c, rng, np.concatenate([distinct_scores(rng, 97, 0.4, 0.95), [t] * 3, distinct_scores(rng, 6, 0.1, 0.25)]))
    c.claims += [("count", 0, 100), ("tie_at_limit", 0)]
    out.append(c)

    # 99 above and 5 tied at rank 100: 104 fit in det_cap 128
    c = Case("limit", "tie_fits_cap", 64, det_cap=128)
    _spread(c, rng, np.concatenate([distinct_scores(rng, 99, 0.4, 0.95), [t] * 5, distinct_scores(rng, 10, 0.1, 0.25)]))
    c.claims += [("count", 0, 104), ("tie_at_limit", 0)]
    out.append(c)

    # the engine default det_cap = 100: one extra tie at rank 100 in class 1 and a 0.99 in class 80, the last class
    c = Case("limit", "tie_overflows_cap_100", 64)
    c.box(0, grid_box(0)); c.score(0, 1, t)
    c.box(1, grid_box(1)); c.score(1, 1, t)
    c.box(2, grid_box(2)); c.score(2, 80, 0.99)
    _spread(c, rng, np.concatenate([distinct_scores(rng, 98, 0.4, 0.95), distinct_scores(rng, 8, 0.1, 0.25)]), 2, 79)
    c.claims += [("count", 0, 101), ("tie_at_limit", 0), ("overflow", 0), ("kept", 0, 80, [2])]
    out.append(c)

    # det_cap 128: 40 ties spread over the classes (class 80 included) and above-threshold detections after them
    c = Case("limit", "tie_overflows_cap_128", 64, det_cap=128)
    used = [(i, 80) for i in range(0, 64, 9)]
    for k, (i, j) in enumerate(used):
        c.box(i, grid_box(i)); c.score(i, j, t if k % 2 == 0 else 0.97 - 0.001 * k)
    n_tied = 40 - sum(1 for k in range(len(used)) if k % 2 == 0)
    n_above = 99 - sum(1 for k in range(len(used)) if k % 2 == 1)
    _spread(c, rng, np.concatenate([distinct_scores(rng, n_above, 0.4, 0.95), [t] * n_tied, distinct_scores(rng, 12, 0.1, 0.25)]),
            avoid=set(used))
    c.claims += [("count", 0, 139), ("tie_at_limit", 0), ("overflow", 0)]
    out.append(c)

    # one class holds all R candidates: distinct scores, and all tied
    c = Case("limit", "one_class", 256)
    s = distinct_scores(rng, 256)
    for i in range(256):
        c.box(i, grid_box(i)); c.score(i, 1, s[i])
    c.claims.append(("count", 0, 100))
    out.append(c)
    c = Case("limit", "one_class_tied", 256)
    for i in range(256):
        c.box(i, grid_box(i)); c.score(i, 7, 0.5)
    c.claims += [("count", 0, 256), ("tie_at_limit", 0)]
    out.append(c)
    return out


def batch_cases():
    rng = np.random.RandomState(17)
    c = Case("batch", "counts_0_1_R", 64, B=3)
    c.scale[:] = [0.8, 1.37, 2.2]
    c.orig_hw[:] = [[480, 640], [333, 517], [250, 190]]
    c.roi_counts[:] = [0, 1, 64]
    # image 1: one RoI scoring in several classes
    c.box(0, [13, 27, 211, 190], b=1)
    for j, s in ((3, 0.7), (9, 0.2), (80, ABOVE), (40, THRESH)):
        c.score(0, j, s, b=1)
    # image 2: overlapping boxes at network scale, distinct scores
    bx = clustered_boxes(rng, 64, 6, extent=(540, 410))
    s = distinct_scores(rng, 64 * 8)
    for i in range(64):
        c.box(i, bx[i], b=2)
        for k, j in enumerate(rng.choice(np.arange(1, 81), 8, replace=False)):
            c.score(i, j, s[i * 8 + k], b=2)
    for b in range(3):
        c.poison(b, rng)
    c.claims.append(("count", 0, 0))
    c.claims.append(("count", 1, 3))
    return [c]


def size_cases():
    out = []
    for R in (1, 31, 32, 33, 1000, 1024):
        rng = np.random.RandomState(R)
        c = Case("sizes", "R%d" % R, R)
        bx = clustered_boxes(rng, R, max(1, R // 24))
        on = rng.rand(R, 81) < 0.1
        on[:, 0] = False
        on[:, 1] = True                                  # class 1 holds all R candidates
        s = distinct_scores(rng, int(on.sum()))
        c.cls_prob[on] = s
        for i in range(R):
            c.box(i, bx[i])
        out.append(c)
    c = Case("sizes", "all_classes_R1024", 1024, orig_hw=(700, 700))
    for i in range(1024):
        c.box(i, grid_box(i, size=10, step=20, cols=32))
    c.cls_prob[:, 1:] = distinct_scores(np.random.RandomState(1), 1024 * 80).reshape(1024, 80)
    c.claims.append(("count", 0, 100))
    out.append(c)
    return out


def class_cases():
    out = []
    rng = np.random.RandomState(23)
    c = Case("classes", "nc2", 64, NC=2)
    bx = clustered_boxes(rng, 64, 4)
    s = distinct_scores(rng, 64)
    for i in range(64):
        c.box(i, bx[i]); c.score(i, 1, s[i])
    out.append(c)
    c = Case("classes", "nc128", 64, NC=128)
    _spread(c, rng, distinct_scores(rng, 150), 1, 127)
    c.box(63, grid_box(63)); c.score(63, 127, 0.999)
    c.claims += [("count", 0, 100), ("kept", 0, 127, [63])]
    out.append(c)
    c = Case("classes", "nc128_tied", 64, NC=128, tie_free=False)
    bx = clustered_boxes(rng, 64, 5)
    for i in range(64):
        c.box(i, bx[i])
    c.cls_prob[:, 1:] = np.asarray([0, 0, 0.2, 0.4, 0.4, 0.6], F32)[rng.randint(0, 6, (64, 127))]
    c.score(int(rng.randint(64)), 127, 0.95)
    out.append(c)
    return out


def fuzz_case(seed):
    rng = np.random.RandomState(1000 + seed)
    c = Case("fuzz", "seed%d" % seed, 256, tie_free=False)
    c.scale[0] = F32((1.0, 0.5, 1.6, 2.3)[seed % 4])
    if seed % 3 == 1:
        c.roi_counts[0] = rng.randint(128, 256)
    bx = clustered_boxes(rng, 256, int(rng.randint(2, 12)), jitter=int(rng.randint(1, 6)))
    vals = np.asarray([BELOW, THRESH, ABOVE, 0.1, 0.25, 0.5, 0.5, 0.75, 0.9, 1.0], F32)
    on = rng.rand(256, 81) < rng.uniform(0.002, 0.3)
    on[:, 0] = False
    c.cls_prob[on] = vals[rng.randint(0, len(vals), int(on.sum()))]
    for i in range(256):
        c.box(i, bx[i] * c.scale[0])                     # network scale
    c.poison(0, rng)
    return c


FAMILIES = {"threshold": threshold_cases, "iou": iou_cases, "decode": decode_cases, "limit": limit_cases,
            "batch": batch_cases, "sizes": size_cases, "classes": class_cases,
            "fuzz": lambda: [fuzz_case(s) for s in range(20)]}


def all_cases():
    return [c for f in FAMILIES.values() for c in f()]

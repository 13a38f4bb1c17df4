"""Randomised and adversarial COCO cases for the device evaluation (detectorch_b200.utils.coco_eval), one generator per family of
inputs where a restatement of COCOeval can go wrong, so that a failure names its family:

  poly       polygons: simple and self-intersecting with 3..500 vertices, degenerate ones, tenth-pixel and (-1, 0) coordinates where
             (int)(5 x + .5) truncates, vertices ~1e4 px outside every side and exactly on w - 1 / h - 1 / w / h, identical, nested
             and disjoint parts, a 2000 x 3000 image with a long boundary
  rle_gt     uncompressed counts with a leading zero and zero-length runs, compressed strings with 6-char values, crowd regions,
             RLEs whose size is not the image's
  matching   101..3000 detections in a pair, score ties at ranks 1 / 10 / 100 and across images and categories, zero and negative
             scores, w or h <= 0, areas of exactly 0 / 32^2 / 96^2 / 1e10, IoUs of k/20, a crowd GT hit by several detections, a GT of
             id 0, categories all crowd or all outside an area range, detections without GT and GT without detections
  segm_dets  all-zero detection masks, masks of another size than their image, masks with many runs
  rank       one category holding most of a few thousand detections (coco_rank_kernel)
  wide       ~80 categories x ~50 images

make_case(family, seed, encode) builds one family; make_mixed_case(seed, encode) a random mix of all of them at a smaller scale.
Both return (dataset, all_boxes [class][image], all_segms [class][image]) as coco_eval_cases.make_case does; encode(mask uint8
[h, w]) -> RLE string is pycocotools' mask.encode.  GT strings are written from counts by oracle/ref.rle_to_string, which
tests/test_coco_eval_host.py pins to mask.encode."""
import numpy as np

from oracle import ref

CAT_IDS = [5, 2, 9, 1, 7, 3, 11, 4]       # dataset order != sorted order


class Case:
    def __init__(self, rng, cat_ids=CAT_IDS, encode=None):
        self.rng, self.cat_ids, self.encode = rng, list(cat_ids), encode
        self.images, self.anns, self.dets = [], [], {}
        self.next_id = 1

    def image(self, h, w):
        i = 1000 - 7 * len(self.images)       # ids not in creation order
        self.images.append(dict(id=i, height=int(h), width=int(w)))
        return i

    def hw(self, img):
        im = next(m for m in self.images if m['id'] == img)
        return im['height'], im['width']

    def gt(self, img, cat, seg, bbox, area, crowd=0, aid=None):
        if aid is None:
            aid, self.next_id = self.next_id, self.next_id + 1
        self.anns.append(dict(id=int(aid), image_id=img, category_id=int(cat), segmentation=seg, bbox=[float(v) for v in bbox],
                              area=float(area), iscrowd=int(crowd)))

    def poly_gt(self, img, cat, parts, area=None, crowd=0, aid=None):
        parts = [[float(v) for v in p] for p in parts]
        xy = np.concatenate([np.array(p).reshape(-1, 2) for p in parts])
        lo, hi = xy.min(0), xy.max(0)
        if area is None:
            area = self.rng.choice([0., 32. ** 2, 96. ** 2, float((hi - lo).prod()), float(self.rng.uniform(0, 2e4))])
        self.gt(img, cat, parts, [lo[0], lo[1], hi[0] - lo[0], hi[1] - lo[1]], area, crowd, aid)

    def counts_gt(self, img, cat, counts, size, compressed, area=None, crowd=0):
        seg = dict(size=list(size), counts=ref.rle_to_string(counts).decode() if compressed else [int(c) for c in counts])
        ys, xs = np.nonzero(ref.rle_decode(counts, size[0], size[1]))
        bb = [xs.min(), ys.min(), xs.max() - xs.min() + 1, ys.max() - ys.min() + 1] if len(xs) else [0, 0, 0, 0]
        self.gt(img, cat, seg, bb, float(np.sum(counts[1::2])) if area is None else area, crowd)

    def det(self, img, cat, box, score, mask=None):
        """box xyxy (float32 as detections are); mask: uint8 array of any size (default: the box clipped to the image)."""
        self.dets.setdefault((img, cat), []).append((np.array(list(box) + [score], np.float32), mask))

    def near(self, img, cat, bb, n, jitter=2.0):
        x, y, w, h = bb
        for _ in range(n):
            j = self.rng.uniform(-jitter, jitter, 4)
            self.det(img, cat, [x + j[0], y + j[1], x + w - 1 + j[2], y + h - 1 + j[3]], self.score())

    def score(self):
        return float(np.round(self.rng.uniform(0, 1) * 16) / 16)      # few distinct values: ties within and across pairs

    def build(self):
        ds = dict(images=list(self.images), annotations=list(self.anns),
                  categories=[dict(id=c, name="c%d" % c) for c in self.cat_ids])
        img_ids = sorted(im['id'] for im in self.images)
        J = len(self.cat_ids) + 1
        all_boxes = [[[] for _ in img_ids] for _ in range(J)]
        all_segms = [[[] for _ in img_ids] for _ in range(J)] if self.encode is not None else None
        for (img, cat), ds_ in self.dets.items():
            i, j = img_ids.index(img), self.cat_ids.index(cat) + 1
            all_boxes[j][i] = np.stack([d for d, _ in ds_]).astype(np.float32)
            if all_segms is not None:
                h, w = self.hw(img)
                segs = []
                for d, m in ds_:
                    if m is None:
                        m = np.zeros((h, w), np.uint8)
                        x1, y1 = int(min(max(d[0], 0), w - 1)), int(min(max(d[1], 0), h - 1))
                        x2, y2 = int(min(max(d[2], 0), w - 1)), int(min(max(d[3], 0), h - 1))
                        m[y1:y2 + 1, x1:x2 + 1] = 1
                    segs.append(dict(size=[int(m.shape[0]), int(m.shape[1])], counts=self.encode(m)))
                all_segms[j][i] = segs
        return ds, all_boxes, all_segms


def _bbox_of(parts):
    xy = np.concatenate([np.array(p, np.float64).reshape(-1, 2) for p in parts])
    lo, hi = xy.min(0), xy.max(0)
    return [lo[0], lo[1], hi[0] - lo[0], hi[1] - lo[1]]


def _star(rng, cx, cy, r, k, jag=0.3):
    t = np.sort(rng.uniform(0, 2 * np.pi, k))
    rr = r * (1 - jag * rng.rand(k))
    return list(np.stack([cx + rr * np.cos(t), cy + rr * np.sin(t)], 1).reshape(-1))


def fam_poly(c, scale=1.0):
    rng = c.rng
    cats = c.cat_ids[:4]
    for n in range(max(1, int(12 * scale))):
        h, w = int(rng.randint(12, 160)), int(rng.randint(12, 160))
        img = c.image(h, w)
        for g in range(int(rng.randint(3, 9))):
            cat = int(rng.choice(cats))
            kind = int(rng.randint(0, 9))
            cx, cy = rng.uniform(-5, w + 5), rng.uniform(-5, h + 5)
            if kind == 0:                     # simple (star-shaped), 3..500 vertices
                parts = [_star(rng, cx, cy, rng.uniform(1, max(h, w) / 2), int(rng.randint(3, 500)))]
            elif kind == 1:                   # self-intersecting: random vertex order in a small region
                k = int(rng.randint(3, 500))
                s = rng.uniform(2, 40)
                parts = [list((np.stack([cx, cy]) + rng.uniform(-s, s, (k, 2))).reshape(-1))]
            elif kind == 2:                   # degenerate: all vertices equal, collinear, a zero-area triangle
                parts = [[[cx, cy] * int(rng.randint(3, 6)), [cx, cy, cx + 7, cy + 3, cx + 14, cy + 6, cx + 3.5, cy + 1.5],
                          [cx, cy, cx + 10, cy, cx + 5, cy]][int(rng.randint(0, 3))]]
            elif kind == 3:                   # tenth-pixel coordinates: 5 x + .5 exactly on an integer; (-1, 0) truncates to 0
                k = int(rng.randint(3, 12))
                xs = np.round(rng.uniform(-1, w + 1, k) * 10) / 10
                ys = np.round(rng.uniform(-1, h + 1, k) * 10) / 10
                xs[0], ys[1] = rng.choice([-0.15, -0.1, -0.9, -0.5, -0.05]), rng.choice([-0.15, -0.3, -0.7, -0.1])
                parts = [list(np.stack([xs, ys], 1).reshape(-1))]
            elif kind == 4:                   # vertices far outside every side
                far = 1e4 * rng.uniform(0.3, 1)
                parts = [[cx, -far, w + far, cy, cx, h + far, -far, cy], [-far, -far, w / 2, h / 3, w / 3, h / 2]]
            elif kind == 5:                   # vertices exactly on the last pixel row / column and on the image edge
                parts = [[w - 1, h - 1, w - 1, 0, rng.uniform(0, w - 1), rng.uniform(0, h - 1)],
                         [w, h, w, h / 2, w / 2, h], [0, h - 1, w - 1, h - 1, w / 2, h / 2]]
            elif kind == 6:                   # identical parts
                p = _star(rng, cx, cy, rng.uniform(2, 30), int(rng.randint(3, 12)))
                parts = [p, list(p)]
            elif kind == 7:                   # nested parts
                r = rng.uniform(6, 40)
                parts = [_star(rng, cx, cy, r, 9, 0.1), _star(rng, cx, cy, r / 3, 5, 0.1)]
            else:                             # disjoint and overlapping parts
                parts = [_star(rng, cx, cy, 5, 6), _star(rng, cx + 20, cy, 5, 6), _star(rng, cx + 23, cy + 2, 6, 7)]
            c.poly_gt(img, cat, parts)
            c.near(img, cat, _bbox_of(parts), int(rng.randint(0, 4)))
        for _ in range(int(rng.randint(0, 6))):
            x, y = rng.uniform(-4, w), rng.uniform(-4, h)
            c.det(img, int(rng.choice(cats)), [x, y, x + rng.uniform(0, w / 2), y + rng.uniform(0, h / 2)], c.score())
    # a large image with a long boundary: many upsampled points over many threads, one part much larger than the others
    h, w = 2000, 3000
    img = c.image(h, w)
    t = np.linspace(0, 2 * np.pi, 401)[:-1]
    r = 900 + 40 * (np.arange(400) % 2)
    big = list(np.stack([1500 + 1.4 * r * np.cos(t), 1000 + r * np.sin(t)], 1).reshape(-1))
    c.poly_gt(img, cats[0], [big, _star(rng, 400, 300, 200, 300)])
    c.near(img, cats[0], _bbox_of([big]), 3, jitter=30)


def _runs(m):
    return [int(v) for v in ref.rle_encode(m)]


def fam_rle_gt(c, scale=1.0):
    rng = c.rng
    cats = c.cat_ids[:3]
    for n in range(max(1, int(10 * scale))):
        h, w = int(rng.randint(8, 90)), int(rng.randint(8, 90))
        img = c.image(h, w)
        for g in range(int(rng.randint(2, 7))):
            cat = int(rng.choice(cats))
            m = np.zeros((h, w), np.uint8)
            y, x = int(rng.randint(0, h)), int(rng.randint(0, w))
            m[y:y + int(rng.randint(1, h)), x:x + int(rng.randint(1, w))] = 1
            if g % 3 == 0:
                m[0, 0] = 1                   # leading zero count
            if g % 3 == 1:
                m ^= (rng.rand(h, w) < .05).astype(np.uint8)
            cnt = _runs(m)
            if g % 2 == 0 and len(cnt) > 2:   # zero-length runs inside
                i = int(rng.randint(0, len(cnt)))
                a = int(rng.randint(0, cnt[i] + 1))
                cnt = cnt[:i] + [a, 0, cnt[i] - a] + cnt[i + 1:]
            size = (h, w)
            if g % 4 == 3:                    # an RLE of another size than the image
                size = (h + int(rng.randint(1, 5)), w)
                cnt = cnt[:-1] + [cnt[-1] + (size[0] - h) * w] if len(cnt) % 2 else cnt + [(size[0] - h) * w]
            crowd = int(rng.rand() < .35)
            c.counts_gt(img, cat, cnt, size, compressed=bool(rng.rand() < .5), crowd=crowd)
            ys, xs = np.nonzero(m)
            if len(ys):
                bb = [xs.min(), ys.min(), xs.max() - xs.min() + 1, ys.max() - ys.min() + 1]
                c.near(img, cat, bb, int(rng.randint(1, 5 if crowd else 3)))
    # values of 6 chars: counts of 2^24 and more, on an image of 4200 x 4100 (17.2 M pixels)
    h, w = 4200, 4100
    img = c.image(h, w)
    m = np.zeros((h, w), np.uint8)
    m[100:900, w - 40:w - 3] = 1
    m[3000:3100, 5:9] = 1
    c.counts_gt(img, cats[0], _runs(m), (h, w), compressed=True)
    c.counts_gt(img, cats[1], _runs(m[:, ::-1]), (h, w), compressed=True, crowd=1)
    c.counts_gt(img, cats[0], _runs(m), (h, w), compressed=False)
    c.det(img, cats[0], [w - 41, 90, w - 2, 905], .9)
    c.det(img, cats[1], [0, 90, 45, 910], .6)
    c.det(img, cats[0], [0, 2990, 12, 3110], .3)


def fam_matching(c, scale=1.0):
    rng = c.rng
    K = c.cat_ids
    # exact IoUs k/20: GT 20 x 10, detections k x 10 at the same corner, every threshold (the oracle decides each side)
    img = c.image(60, 80)
    c.poly_gt(img, K[0], [[5, 5, 25, 5, 25, 15, 5, 15]], area=200.)
    for k in range(9, 21):
        c.det(img, K[0], [5, 5, 5 + k - 1, 14], 1 - k / 40)
    c.poly_gt(img, K[1], [[40, 30, 60, 30, 60, 40, 40, 40]], area=200.)
    for k in range(9, 21):                    # the same IoUs, all at one score
        c.det(img, K[1], [40, 30, 40 + k - 1, 39], .5)
    # a pair with many detections and ties straddling ranks 1, 10 and 100
    img = c.image(120, 160)
    n = int(rng.randint(101, int(101 + 2900 * scale) + 1))
    s = np.sort(rng.uniform(0.05, 1, n))[::-1].copy()
    for a, b in ((0, 2), (8, 12), (98, 103)):
        s[a:b] = s[a]
    for g in range(6):
        x, y = rng.uniform(0, 120), rng.uniform(0, 80)
        c.poly_gt(img, K[2], [[x, y, x + 30, y, x + 30, y + 30, x, y + 30]], area=[0., 1024., 9216., 1e10, 500., 1023.9][g],
                  crowd=int(g == 5))
    for i in rng.permutation(n):
        x, y = rng.uniform(-2, 150), rng.uniform(-2, 110)
        c.det(img, K[2], [x, y, x + rng.uniform(-3, 40), y + rng.uniform(-3, 40)], s[i])
    # zero and negative scores, w or h <= 0 and zero area, det areas of exactly 0 / 32^2 / 96^2 / 1e10
    img = c.image(200, 200)
    c.poly_gt(img, K[3], [[10, 10, 50, 10, 50, 50, 10, 50]], area=1600.)
    c.poly_gt(img, K[3], [[0, 0, 200, 0, 200, 200, 0, 200]], area=1e10)
    for box, sc in (([10, 10, 41, 41], 0.), ([10, 10, 105, 105], -.25), ([12, 12, 11, 40], .7), ([12, 12, 40, 11], .7),
                    ([12, 12, 5, 3], .6), ([0, 0, 99999, 99999], .2), ([20, 20, 51, 51], -0.), ([10, 10, 49, 49], 0.)):
        c.det(img, K[3], box, sc)
    # a crowd GT hit by several detections and a GT of id 0
    img = c.image(100, 100)
    c.poly_gt(img, K[4], [[0, 0, 60, 0, 60, 60, 0, 60]], area=3600., crowd=1)
    c.poly_gt(img, K[4], [[10, 10, 30, 10, 30, 30, 10, 30]], area=400., aid=0)
    c.poly_gt(img, K[4], [[70, 70, 95, 70, 95, 95, 70, 95]], area=625.)
    for k in range(6):
        c.det(img, K[4], [2 + 8 * k, 2, 10 + 8 * k, 40], .3 + .1 * (k % 3))
    c.near(img, K[4], [10, 10, 20, 20], 3, jitter=1.5)
    c.near(img, K[4], [70, 70, 25, 25], 2)
    # categories all crowd, all outside one area range (all large), detections without any GT of their category
    for n_img in range(3):
        img = c.image(150, 150)
        c.poly_gt(img, K[5], [[5, 5, 60, 5, 60, 60, 5, 60]], area=3025., crowd=1)
        c.near(img, K[5], [5, 5, 55, 55], 2)
        c.poly_gt(img, K[6], [[20, 20, 140, 20, 140, 140, 20, 140]], area=14400.)
        c.near(img, K[6], [20, 20, 120, 120], 2, jitter=6)
        c.det(img, K[6], [0, 0, 10, 10], c.score())
        c.det(img, K[7], [30, 30, 70, 70], c.score())
    # an image with GT but no detections, and one with detections but no GT
    img = c.image(50, 50)
    c.poly_gt(img, K[0], [[5, 5, 20, 5, 20, 20]], area=120.)
    img = c.image(50, 50)
    c.det(img, K[0], [5, 5, 20, 20], .75)
    # random pairs with tied scores across images and categories
    for n_img in range(max(1, int(12 * scale))):
        h, w = int(rng.randint(40, 120)), int(rng.randint(40, 120))
        img = c.image(h, w)
        for g in range(int(rng.randint(1, 8))):
            cat = int(rng.choice(K[:5]))
            x, y = rng.uniform(-3, w - 4), rng.uniform(-3, h - 4)
            bw, bh = rng.uniform(1, w / 2), rng.uniform(1, h / 2)
            c.poly_gt(img, cat, [[x, y, x + bw, y, x + bw, y + bh, x, y + bh]], crowd=int(rng.rand() < .15))
            c.near(img, cat, [x, y, bw, bh], int(rng.randint(0, 4)), jitter=3)
        for _ in range(int(rng.randint(0, 15))):
            x, y = rng.uniform(-3, w), rng.uniform(-3, h)
            c.det(img, int(rng.choice(K[:5])), [x, y, x + rng.uniform(-2, w / 2), y + rng.uniform(-2, h / 2)], c.score())


def fam_segm_dets(c, scale=1.0):
    rng = c.rng
    cats = c.cat_ids[:3]
    for n in range(max(1, int(10 * scale))):
        h, w = int(rng.randint(10, 80)), int(rng.randint(10, 80))
        img = c.image(h, w)
        boxes = []
        for g in range(int(rng.randint(1, 5))):
            cat = int(rng.choice(cats))
            x, y = rng.uniform(0, w - 4), rng.uniform(0, h - 4)
            bw, bh = rng.uniform(2, w - x), rng.uniform(2, h - y)
            c.poly_gt(img, cat, [[x, y, x + bw, y, x + bw, y + bh, x, y + bh]], crowd=int(rng.rand() < .2))
            boxes.append((cat, [x, y, x + bw, y + bh]))
        for cat, b in boxes:
            for kind in range(int(rng.randint(1, 5))):
                k = int(rng.randint(0, 4))
                if k == 0:
                    m = np.zeros((h, w), np.uint8)                              # all zero
                elif k == 1:
                    m = np.zeros((h + int(rng.randint(-3, 4)), w + int(rng.randint(1, 4))), np.uint8)   # another size
                    m[int(b[1]):int(b[3]), int(b[0]):int(b[2])] = 1
                elif k == 2:
                    m = (rng.rand(h, w) < .5).astype(np.uint8)                 # many runs
                    m[:int(b[1])] = 0
                else:
                    m = None
                c.det(img, cat, b, c.score(), m)


def fam_rank(c, scale=1.0):
    """One category holding most of a few thousand detections: 100 kept per image over many images, few distinct scores."""
    rng = c.rng
    n_img = max(2, int(30 * scale))
    for n in range(n_img):
        img = c.image(64, 64)
        for g in range(int(rng.randint(0, 4))):
            x, y = rng.uniform(0, 40), rng.uniform(0, 40)
            bw, bh = rng.uniform(4, 24), rng.uniform(4, 24)
            c.poly_gt(img, c.cat_ids[0], [[x, y, x + bw, y, x + bw, y + bh, x, y + bh]], area=float(bw * bh))
            c.near(img, c.cat_ids[0], [x, y, bw, bh], 2)
        for _ in range(int(rng.randint(95, 130))):
            x, y = rng.uniform(0, 60), rng.uniform(0, 60)
            c.det(img, c.cat_ids[0], [x, y, x + rng.uniform(1, 30), y + rng.uniform(1, 30)], float(rng.randint(0, 5)) / 4)
        if n % 5 == 0:
            c.near(img, c.cat_ids[1], [10, 10, 20, 20], 3)
            c.poly_gt(img, c.cat_ids[1], [[10, 10, 30, 10, 30, 30, 10, 30]], area=400.)


def fam_wide(c, scale=1.0):
    rng = c.rng
    for n in range(max(2, int(50 * scale))):
        h, w = int(rng.randint(30, 90)), int(rng.randint(30, 90))
        img = c.image(h, w)
        for g in range(int(rng.randint(0, 6))):
            cat = int(rng.choice(c.cat_ids))
            x, y = rng.uniform(-2, w - 4), rng.uniform(-2, h - 4)
            bw, bh = rng.uniform(1, w / 2), rng.uniform(1, h / 2)
            c.poly_gt(img, cat, [[x, y, x + bw, y, x + bw / 2, y + bh]], crowd=int(rng.rand() < .1))
            c.near(img, cat, [x, y, bw, bh], int(rng.randint(0, 3)), jitter=3)
        for _ in range(int(rng.randint(0, 8))):
            x, y = rng.uniform(-2, w), rng.uniform(-2, h)
            c.det(img, int(rng.choice(c.cat_ids)), [x, y, x + rng.uniform(0, w / 2), y + rng.uniform(0, h / 2)], c.score())


FAMILIES = dict(poly=fam_poly, rle_gt=fam_rle_gt, matching=fam_matching, segm_dets=fam_segm_dets, rank=fam_rank, wide=fam_wide)
WIDE_CATS = [int(v) for v in np.random.RandomState(80).permutation(np.arange(1, 91))[:80]]


def make_case(family, seed=0, encode=None):
    rng = np.random.RandomState(1000 * (list(FAMILIES).index(family) + 1) + seed)
    c = Case(rng, WIDE_CATS if family == 'wide' else CAT_IDS, encode)
    FAMILIES[family](c)
    return c.build()


def make_mixed_case(seed, encode=None):
    """A random mix of the families at a small scale (no 4200 x 4100 / 2000 x 3000 images unless the seed picks poly / rle_gt)."""
    rng = np.random.RandomState(seed)
    c = Case(rng, CAT_IDS, encode)
    names = [n for n in FAMILIES if n != 'wide']
    for name in rng.choice(names, int(rng.randint(1, 4)), replace=False):
        FAMILIES[name](c, scale=float(rng.uniform(.1, .4)))
    return c.build()

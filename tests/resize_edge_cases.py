"""Seeded edge cases of the two OpenCV-exact resizes, shared by tests/test_resize_edges_host.py, tests/test_gpu_resize_edges.py and
tests/golden/make_resize_edges_golden.py (which runs the reference's own blob.py and segm_results on them and stores what it computed
in tests/golden/resize_edges_golden.npz).  Importable without the reference.

  prep   (H, W, target_size, max_size) through prep_im_for_blob + im_list_to_blob (prep_image_kernel / dt_prep_image): exact 2x
         down-scales with an odd side whose half rounds up (n % 4 == 3: cvRound(n / 2) = (n + 1) / 2, a partial last column / row of
         OpenCV's area-fast kernel) or down (n % 4 == 1), the max_size cap landing on exactly 0.5, 1xN / Nx1 / 1x1 images, large
         up-scales, ordinary down-scales
  fx     (H, W, fx) straight through cv2.resize(fx=fy=fx) after the mean subtraction: both sides odd at fx = 0.5 (no target / max
         size gives that), fx a few ulp either side of 0.5 (1 / fx is then not 2: the bilinear kernel, not the area-fast one), and
         factors other than 1 that keep the size (OpenCV copies the image then)
  masks  mask paste + RLE (segm_results; segm_rle_kernel, segm_paste_kernel) for M = 28 and 14, class-specific
         [D, K, M, M] stacks with one class per detection, on images of 1x1, 1xN, Nx1, 2x2, odd sizes (23x37, 31x17, 47x45), 13x1500 and 600x11; boxes of
         every family in `FAMILIES`, clipped to the image (the reference raises on boxes outside it); masks uniform random, in
         multiples of 1/8 (interpolated values land exactly on the 0.5 threshold), constant 0.5, ones, zeros and a checkerboard."""
import zlib

import numpy as np

F32 = np.float32
MEANS = (122.7717, 115.9465, 102.9801)

PREP_CASES = [
    # exact 2x down-scale, one odd side: half rounding up (23 -> 12, 35 -> 18, 7 -> 4, 19 -> 10, 3 -> 2) and down (21 -> 10, 17 -> 8, 5 -> 2)
    (16, 23, 8, 1333), (16, 21, 8, 1333), (23, 16, 8, 1333), (21, 16, 8, 1333), (16, 19, 8, 1333), (16, 17, 8, 1333),
    (22, 35, 11, 1333), (2, 7, 1, 1333), (7, 2, 1, 1333), (2, 5, 1, 1333), (2, 3, 1, 1333), (18, 16, 8, 1333),
    # the max_size cap landing on exactly 0.5: the min side odd, rounding up (11 -> 6) and down (13 -> 6)
    (11, 30, 8, 15), (30, 11, 8, 15), (13, 30, 50, 15), (9, 18, 50, 9),
    # 1xN, Nx1, 1x1 and large up-scales
    (1, 37, 50, 84), (41, 1, 50, 84), (1, 1, 50, 1333), (2, 3, 40, 1333), (3, 2, 60, 1333), (1, 4, 3, 1333),
    # ordinary down-scales and a non-integer up-scale
    (37, 53, 20, 1333), (64, 48, 30, 40), (45, 100, 30, 50), (17, 29, 40, 1333),
]
HALF = 0.5
FX_CASES = [(9, 11, HALF), (15, 13, HALF), (3, 3, HALF), (11, 5, HALF), (7, 7, HALF), (19, 23, HALF)]
for _k in (1, 3):
    _up, _dn = HALF, HALF
    for _ in range(_k):
        _up, _dn = float(np.nextafter(_up, 1.0)), float(np.nextafter(_dn, 0.0))
    FX_CASES += [(16, 23, _up), (9, 11, _dn), (23, 16, _dn), (11, 9, _up)]
# dsize == ssize with fx != 1: cv::resize copies the image
FX_CASES += [(1, 1, float(np.nextafter(HALF, 1.0))), (1, 1, 0.75), (5, 7, 1.05)]
# full-size exact 2x down-scales with an odd side whose half rounds up (checked against the oracle computed live)
FULL_CASES = [(1600, 2003, 800, 1333), (2666, 1003, 800, 1333)]


def prep_image(i, h, w, seed=0):
    """The uint8 BGR image of prep / fx / full case i (seed 0: the fixture's; other seeds: fresh inputs of the same shape)."""
    return np.random.RandomState(1000 + 7919 * seed + i).randint(0, 256, (h, w, 3)).astype(np.uint8)


def fx_input(im):
    """prep_im_for_blob's float32 image before the resize: im.astype(float32) -= pixel_means."""
    x = im.astype(np.float32, copy=True)
    x -= list(MEANS)
    return x


def cv_round(v):
    """cvRound of a double: round half to even (the size cv2.resize(fx=...) produces)."""
    return int(np.rint(v))


# ------------------------------------------------------------------------------------------------ masks
MASK_SIZES = (28, 14)
NUM_CLASSES = {28: 4, 14: 3}
IMAGES = [(1, 1), (1, 37), (41, 1), (2, 2), (23, 37), (31, 17), (47, 45), (13, 1500), (600, 11)]
KINDS = ("uniform", "eighths", "half", "ones", "zeros", "checker")
FAMILIES = ("full", "point", "corner", "row", "col", "trunc", "neg", "area2", "half_x", "half_y", "exact", "big")


def expand(M, boxes):
    """boxes.expand_boxes by (M + 2) / M, truncated to int32 (result_utils.segm_results)."""
    from oracle import ref
    return ref.expand_boxes(np.asarray(boxes, F32).reshape(-1, 4), (M + 2.0) / M).astype(np.int32)


def axis_span(M, want, start, limit):
    """float32 (a, b), start <= a <= b <= limit, whose expanded int32 extent e2 - e0 + 1 is `want` cells; None if there is none.
    Found by search: the expansion is fp32 arithmetic followed by truncation, so the span is not a closed form."""
    L = np.arange(0, limit + 1, 0.0625, dtype=np.float64)
    for a in start + np.arange(0, 1, 0.125):
        b = a + L
        b = b[b <= limit]
        if len(b) == 0:
            break
        bx = np.stack([np.full_like(b, a), np.full_like(b, a), b, b], 1)
        e = expand(M, bx)
        hit = np.flatnonzero(e[:, 2] - e[:, 0] + 1 == want)
        if len(hit):
            return F32(a), F32(b[hit[0]])
    return None


def mask_boxes(M, H, W):
    """[(family, box)] for one image: every family that fits, clipped to the image."""
    S = M + 2
    X, Y = W - 1, H - 1
    out = [("full", [0, 0, X, Y]), ("full", [0, 0, X, Y]),
           ("point", [0, 0, 0, 0]), ("point", [X, Y, X, Y]), ("point", [X * .5 + .25, Y * .5 + .25] * 2)]
    c, r = min(X, 5.5), min(Y, 4.25)
    out += [("corner", [0, 0, c, r]), ("corner", [X - c, 0, X, r]), ("corner", [0, Y - r, c, Y]), ("corner", [X - c, Y - r, X, Y])]
    out += [("row", [min(1.5, X), Y // 2, X, Y // 2]), ("row", [0, Y, X, Y]), ("col", [X // 2, min(.5, Y), X // 2, Y]), ("col", [X, 0, X, Y])]
    # the expanded origin -s / M: in (-1, 0) (truncated to 0, not floored to -1) and <= -1
    out += [("trunc", [0, 0, min(3.5, X), min(2.5, Y)]), ("trunc", [0, min(1.0, Y), min(M - .5, X), min(M + 1.0, Y)]),
            ("neg", [0, 0, min(M + 3.5, X), min(M + 1.5, Y)]), ("neg", [0, 0, min(3 * M + .5, X), min(2 * M, Y)])]
    spans = {}
    for want in sorted({S // 2, S // 2 + 3, S}):
        for name, start in (("in", 2.0), ("origin", 0.0), ("end", None)):
            for ax, lim in (("x", X), ("y", Y)):
                st = start if start is not None else max(0.0, lim - want + 2.0)
                spans[(want, name, ax)] = axis_span(M, want, st, lim)

    def span_box(fam, wx, wy, name):
        sx, sy = spans[(wx, name, "x")], spans[(wy, name, "y")]
        if sx is not None and sy is not None:
            out.append((fam, [sx[0], sy[0], sx[1], sy[1]]))
    for name in ("in", "origin", "end"):
        span_box("area2", S // 2, S // 2, name)
        span_box("half_x", S // 2, S // 2 + 3, name)
        span_box("half_y", S // 2 + 3, S // 2, name)
        span_box("exact", S, S, name)
    # boxes 10 to 50 times the mask size along the long side of the image
    for k in (10, 23, 50):
        if W >= 10 * M:
            out.append(("big", [min(2.5, X), 0, min(2.5 + k * M, X), Y]))
        if H >= 10 * M:
            out.append(("big", [0, min(1.5, Y), X, min(1.5 + k * M, Y)]))
    b = np.asarray([bx for _, bx in out], F32)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, X)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, Y)
    assert np.all(b[:, 2] >= b[:, 0]) and np.all(b[:, 3] >= b[:, 1])
    return [f for f, _ in out], b


def make_mask(kind, M, rng):
    if kind == "uniform":
        return rng.rand(M, M).astype(F32)
    if kind == "eighths":
        return (rng.randint(0, 9, (M, M)) / 8.0).astype(F32)
    if kind == "half":
        return np.full((M, M), .5, F32)
    if kind == "ones":
        return np.ones((M, M), F32)
    if kind == "zeros":
        return np.zeros((M, M), F32)
    return (np.add.outer(np.arange(M), np.arange(M)) % 2).astype(F32)


class MaskSet:
    """One image of one mask size: boxes [D, 4] fp32 (image pixels, within the image), cls [D] int32 sorted ascending in [1, K)
    (segm_results visits the detections class by class), masks [D, K, M, M] fp32; families[d] and kinds[d] name what each is."""

    def __init__(self, M, H, W, seed=0):
        self.M, self.K, self.H, self.W = M, NUM_CLASSES[M], H, W
        self.tag = "m%d_%dx%d" % (M, H, W)
        rng = np.random.RandomState(zlib.crc32(self.tag.encode()) + 7919 * seed)
        self.families, self.boxes = mask_boxes(M, H, W)
        D = len(self.boxes)
        self.cls = np.sort(rng.randint(1, self.K, D)).astype(np.int32)
        # the first full-image box is all ones (runs touch the top and bottom rows, end at the last column, set pixel (0, 0)), the
        # second a checkerboard (the most runs); the other detections cycle through the kinds
        self.kinds = [KINDS[(d + seed) % len(KINDS)] for d in range(D)]
        self.kinds[0], self.kinds[1] = "ones", "checker"
        self.masks = np.zeros((D, self.K, M, M), F32)
        for d in range(D):
            for k in range(self.K):
                self.masks[d, k] = make_mask(self.kinds[d], M, rng)

    @property
    def D(self):
        return len(self.boxes)

    def cls_boxes(self):
        cb = [[] for _ in range(self.K)]
        for j in range(1, self.K):
            sel = self.cls == j
            cb[j] = np.hstack([self.boxes[sel], np.ones((int(sel.sum()), 1), F32)])
        return cb

    def selected(self):
        """[D, M, M]: each detection's own class plane."""
        return self.masks[np.arange(self.D), self.cls]

    def digest(self):
        return np.uint32(zlib.crc32(self.boxes.tobytes() + self.cls.tobytes() + self.masks.tobytes()))


def mask_sets(seed=0):
    return [MaskSet(M, H, W, seed) for M in MASK_SIZES for (H, W) in IMAGES]


# ------------------------------------------------------------------------------------------------ running the reference
def reference_prep(rb, im, ts, ms):
    """The reference's blob.prep_im_for_blob + im_list_to_blob(fpn_on=False) -> (blob [1, 3, h, w], im_scale); also checks that its
    fpn_on=True blob is that blob zero-padded to the stride."""
    ims, scales = rb.prep_im_for_blob(im.copy(), target_sizes=[ts], max_size=ms)
    blob = rb.im_list_to_blob(ims, fpn_on=False)
    fpn = rb.im_list_to_blob(ims, fpn_on=True)
    h, w = blob.shape[2:]
    assert fpn.shape[2] == -(-h // 32) * 32 and fpn.shape[3] == -(-w // 32) * 32
    assert np.array_equal(fpn[:, :, :h, :w], blob) and not fpn[:, :, h:].any() and not fpn[:, :, :, w:].any()
    return np.ascontiguousarray(blob), scales[0]


def reference_segm(ru, s):
    """The reference's segm_results on mask set s -> (pasted masks [D, H, W] uint8 it hands to mask_util.encode, RLE strings).
    pycocotools is not importable with the reference: mask_util.encode is replaced for the call by a recorder that encodes with the
    oracle's restatement of maskApi."""
    from oracle import ref
    captured = []

    def encode(arr):
        captured.append(np.ascontiguousarray(arr[:, :, 0]))
        return [{'size': list(arr.shape[:2]), 'counts': ref.rle_to_string(ref.rle_encode(arr[:, :, 0]))}]
    had = hasattr(ru.mask_util, "encode")
    old = getattr(ru.mask_util, "encode", None)
    ru.mask_util.encode = encode
    try:
        segms = ru.segm_results(s.cls_boxes(), s.masks, s.boxes, s.H, s.W, num_classes=s.K, M=s.M)
    finally:
        if had:
            ru.mask_util.encode = old
        else:
            del ru.mask_util.encode
    strings = [d['counts'] for j in range(1, s.K) for d in segms[j]]
    assert len(captured) == s.D and all(d['size'] == [s.H, s.W] for j in range(1, s.K) for d in segms[j])
    return np.stack(captured), strings


def oracle_segm(s):
    """oracle.segm_results on mask set s -> (pasted masks [D, H, W] uint8, RLE strings)."""
    from oracle import ref
    exp = expand(s.M, s.boxes)
    pasted = np.stack([ref.paste_mask(s.masks[d, s.cls[d]], exp[d], s.H, s.W) for d in range(s.D)])
    segms = ref.segm_results(s.cls_boxes(), s.masks, s.boxes, s.H, s.W, num_classes=s.K, M=s.M)
    return pasted, [d['counts'] for j in range(1, s.K) for d in segms[j]]

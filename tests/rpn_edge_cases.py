"""Adversarial inputs for the device RPN proposal stage (ST_PROPOSALS: rpn_select_{keys,hist2,count,scatter}_kernel,
rpn_proposals_kernel, nms_mask_kernel, rpn_nms_scan_kernel) and the collect step (ST_COLLECT: collect_kernel), one generator per
family of inputs where the port can go wrong, so that a failure names its family:

  select    every branch of the top-k: a level with n <= 8192 anchors (sorted whole), 8192 < n <= 4K (sorted whole), the two-level
            11+11-bit radix select that narrows the level, and its fall-back to a whole sort when the boundary sub-bin holds more than
            8192 keys; the K-th key at the first and at the last slot of its 11-bit digit bin and of its 22-bit sub-bin; a boundary
            total of exactly 8192 and 8193; pre_nms of 1, 63, 64, 65, 127, 128, 129, 3071, 3072 and 8192 (>= n on the coarse levels);
            runs of equal scores straddling the cut and a level of one score
  mixed     one launch of two images on a ragged canvas, one image's P2 selecting and the other's not (n just below and above 8192)
  filter    zero size deltas (boxes bit-exact): widths and heights exactly min_size * scale next to one pixel less, anchors pushed far
            outside the image (clipped to points and lines on the border, xc = im_w - 0.5, the largest a clipped box reaches), a
            level whose candidates are all filtered out, and size deltas above log(1000 / 16) (compared within 2e-4)
  nms       fp32 IoU of exactly 0.7 (suppressed: the reference tests ovr >= thresh) next to 0.65, every candidate the same box, more
            survivors than post_nms, post_nms of 1
  collect   scores equal across levels, empty levels, more candidates than top_n

Every case is a Case: per image, per level, the RPN maps (objectness [A, h, w] and deltas [4A, h, w] over the image's own extent
of the level) that are teacher-forced into rpn_out*, each image's network size and scaling factor, the engine configuration
(pre_nms, post_nms, min_size), and the properties it is built to have (`claims`), which tests/test_rpn_edge_cases_host.py checks
with a numpy mirror of the device's selection and with the oracle."""
import numpy as np

F32 = np.float32
CANVAS = 256                       # engine canvas (H = W); P2 then holds 64 * 64 * 3 = 12288 anchors
A = 3
LEVELS = 5                         # P2..P6
NMS = 0.7
SEL_MAX = 8192                     # largest boundary total the narrowed sort takes (rpn_select_count_kernel)


def stride(l):
    return 4 << l


def extent(net, l):
    """Cells of level l covered by an image of net pixels (image_info: ceil(net / stride), within the canvas map)."""
    return min(-(-net // stride(l)), -(-CANVAS // stride(l)))


def desc_key(s):
    """float_desc_key (sort_nms.cuh): ascending key == descending score."""
    b = np.asarray(s, F32).view(np.uint32)
    b = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000))
    return (~b).astype(np.uint32)


def from_key(k):
    """The positive score whose desc_key is k (k in [0x00000000, 0x7fffffff])."""
    k = np.asarray(k, np.int64)
    assert np.all((k >= 0) & (k <= 0x7fffffff))
    return (0x7fffffff - k).astype(np.uint32).view(F32)


def select_stats(scores, pre):
    """The device's top-k plan for one (image, level), mirrored in numpy: n, K, whether the level selects
    (rpn_level_selects: n > 4K and n > 8192), the boundary digit b1, sub-digit b2 and the boundary total, and the branch:
    "small" (n <= 8192, whole sort), "k4" (8192 < n <= 4K, whole sort), "narrowed", "fallback" (total > 8192, whole sort)."""
    keys = np.sort(desc_key(np.asarray(scores).reshape(-1)))
    n = len(keys)
    K = n if pre <= 0 or pre >= n else pre
    kth = int(keys[K - 1])
    b1, b2 = kth >> 21, (kth >> 10) & 2047
    d1, d2 = keys >> 21, (keys >> 10) & 2047
    total = int(np.count_nonzero((d1 < b1) | ((d1 == b1) & (d2 <= b2))))
    selects = n > 4 * K and n > SEL_MAX
    branch = ("narrowed" if total <= SEL_MAX else "fallback") if selects else ("small" if n <= SEL_MAX else "k4")
    return dict(n=n, K=K, b1=b1, b2=b2, total=total, branch=branch, keys=keys)


def base_anchors(l):
    """Level l's base anchors (ratio-major, one size), float64 as generate_anchors gives them."""
    from oracle import ref
    return ref.generate_anchors(stride=stride(l), sizes=(32 << l,))


class Case:
    """claims: list of tuples checked by the host test:
         ("branch", b, l, name)       select_stats(...)["branch"] == name
         ("slot", b, l, where)        the K-th key is the first / last key present in its digit bin ("bin_first", "bin_last") or
                                      sub-bin ("sub_first", "sub_last"), and it sits on that edge of the bin's key range
         ("total", b, l, t)           the boundary total is t
         ("tie_cut", b, l)            a run of equal scores straddles the top-K cut
         ("iou", b, l, i, j, v)       anchors i (higher score) and j decode to boxes whose fp32 IoU is v; with v >= 0.7, j is
                                      suppressed, else both are kept
         ("filtered_all", b, l)       no candidate of the level passes filter_boxes
         ("cands", b, l, c)           exactly c candidates pass the filter
         ("edge", b, l, what, i)      anchor i's clipped box sits on a filter edge: "ws_eq" / "hs_eq" (== min_size * scale, kept),
                                      "ws_below" / "hs_below" (one less, dropped), "xc_max" / "yc_max" (xc == im_w - 0.5 / yc == im_h - 0.5)
         ("survivors", b, l, c)       c candidates survive the NMS (before the post_nms cut)
         ("survivors_over", b, l, c)  more than c candidates survive the NMS, so that post_nms = c cuts them
         ("collect_cut", b)           more proposals than top_n reach the collect
         ("cross_level_tie", b)       equal scores on different levels reach the collect
       exact: zero size deltas everywhere, so the device's boxes equal the oracle's bit for bit (otherwise expf against torch.exp,
       and every candidate pair keeps its IoU 1e-5 away from the NMS threshold)."""

    def __init__(self, family, name, net_hw=((CANVAS, CANVAS),), pre=1000, post=1000, min_size=0.0, scale=None, seed=0):
        self.family, self.name = family, name
        self.net_hw = [tuple(int(v) for v in hw) for hw in net_hw]
        self.B = len(self.net_hw)
        self.pre, self.post, self.min_size = pre, post, float(min_size)
        self.scale = np.ones(self.B, F32) if scale is None else np.asarray(scale, F32).reshape(self.B)
        self.exact = True
        self.claims = []
        rng = np.random.RandomState(seed)
        self.scores, self.deltas = [], []
        for b, (h, w) in enumerate(self.net_hw):
            sl, dl = [], []
            for l in range(LEVELS):
                eh, ew = extent(h, l), extent(w, l)
                n = A * eh * ew
                sl.append((0.9 * (rng.permutation(n) + 1) / (n + 1)).astype(F32).reshape(A, eh, ew))    # distinct, in (0, 0.9]
                d = np.zeros((4 * A, eh, ew), F32)
                d[0::4] = 0.3 * rng.randn(A, eh, ew)
                d[1::4] = 0.3 * rng.randn(A, eh, ew)
                dl.append(d)
            self.scores.append(sl)
            self.deltas.append(dl)

    @property
    def id(self):
        return "%s-%s" % (self.family, self.name)

    @property
    def group(self):
        """Cases of one group run on one engine."""
        return (self.B, self.pre, self.post, self.min_size)

    def dims(self, b, l):
        return self.scores[b][l].shape[1:]

    def set_scores(self, b, l, flat_scores):
        h, w = self.dims(b, l)
        self.scores[b][l] = np.asarray(flat_scores, F32).reshape(h, w, A).transpose(2, 0, 1).copy()

    def get_scores(self, b, l):
        return self.scores[b][l].transpose(1, 2, 0).reshape(-1)

    def anchor_box(self, l, i, w):
        """Unclipped anchor box of flat index i on level l of an image w cells wide (float32, as the oracle rounds them)."""
        a, cell = i % A, i // A
        y, x = cell // w, cell % w
        s = stride(l)
        return (base_anchors(l)[a] + np.array([x * s, y * s, x * s, y * s])).astype(F32)

    def place(self, b, l, i, box, score=None):
        """Move anchor i of (b, l) onto the integer box `box` (same size as the anchor) with zero size deltas: the decode is exact."""
        h, w = self.dims(b, l)
        anc = self.anchor_box(l, i, w)
        box = np.asarray(box, F32)
        aw, ah = anc[2] - anc[0] + 1, anc[3] - anc[1] + 1
        assert box[2] - box[0] + 1 == aw and box[3] - box[1] + 1 == ah, (box, anc)
        a, y, x = i % A, (i // A) // w, (i // A) % w
        self.deltas[b][l][4 * a:4 * a + 4, y, x] = [F32((box[0] - anc[0]) / aw), F32((box[1] - anc[1]) / ah), 0, 0]
        if score is not None:
            self.scores[b][l][a, y, x] = F32(score)

    def set_delta(self, b, l, i, d):
        h, w = self.dims(b, l)
        a, y, x = i % A, (i // A) // w, (i // A) % w
        self.deltas[b][l][4 * a:4 * a + 4, y, x] = np.asarray(d, F32)

    def rpn_out(self, b, l):
        """NHWC [h, w, 5A] block of rpn_out for (b, l): objectness then deltas."""
        return np.concatenate([self.scores[b][l], self.deltas[b][l]], 0).transpose(1, 2, 0).copy()

    def decoy(self, seed=1):
        """The same case with every level's scores shuffled across its anchors: another input of the same engine whose keys have the
        same histograms, run before the case so that the case is always a second run of its engine (stale selection histograms
        would double every count)."""
        d = Case.__new__(Case)
        d.__dict__.update(self.__dict__)
        rng = np.random.RandomState(seed)
        d.scores = [[s.reshape(-1)[rng.permutation(s.size)].reshape(s.shape) for s in sl] for sl in self.scores]
        d.name = self.name + "-decoy"
        d.claims = []
        return d


# ------------------------------------------------------------------------------------------------ helpers
def keys_to_level(c, b, l, below, above, kth, rng):
    """P-level scores whose sorted keys are `below` (K - 1 keys), kth, `above` (n - K keys), shuffled over the anchors."""
    keys = np.concatenate([below, [kth], above]).astype(np.int64)
    n = A * int(np.prod(c.dims(b, l)))
    assert len(keys) == n, (len(keys), n)
    c.set_scores(b, l, from_key(keys[rng.permutation(n)]))


def pick(rng, lo, hi, k):
    """k distinct integers in [lo, hi)."""
    assert hi - lo >= k
    return lo + rng.choice(hi - lo, k, replace=False)


B1 = 0x205          # a digit bin of scores in (0.5, 1)


# ------------------------------------------------------------------------------------------------ families
def select_cases():
    out = []
    K, n = 1000, A * 64 * 64
    # the K-th key on each edge of its digit bin / sub-bin; every key distinct
    for where in ("bin_first", "bin_last", "sub_first", "sub_last"):
        c = Case("select", where, pre=K, seed=10)
        rng = np.random.RandomState(11)
        lo = B1 << 21
        if where == "bin_first":
            kth = lo
            below, above = pick(rng, lo - (1 << 21), lo, K - 1), pick(rng, lo + 1, lo + (1 << 21), n - K)
        elif where == "bin_last":
            kth = lo | 0x1fffff
            below, above = pick(rng, lo, kth, K - 1), pick(rng, kth + 1, kth + 1 + (1 << 21), n - K)
        elif where == "sub_first":
            kth = lo | (700 << 10)
            below = pick(rng, lo, kth, K - 1)
            above = np.concatenate([pick(rng, kth + 1, kth + 1024, 300), pick(rng, lo + (1 << 21), lo + (2 << 21), n - K - 300)])
        else:
            kth = lo | (700 << 10) | 0x3ff
            below = np.concatenate([pick(rng, kth - 1023, kth, 300), pick(rng, lo, lo | (700 << 10), K - 1 - 300)])
            above = pick(rng, kth + 1, lo + (1 << 21), n - K)
        keys_to_level(c, 0, 0, below, above, kth, rng)
        c.claims += [("branch", 0, 0, "narrowed"), ("slot", 0, 0, where)]
        out.append(c)
    # boundary total of exactly 8192 (narrowed) and 8193 (whole-sort fall-back): the K-th key opens a sub-bin that also holds, after
    # it, repeated keys (ties, all past the cut)
    for total in (SEL_MAX, SEL_MAX + 1):
        c = Case("select", "total%d" % total, pre=K, seed=12)
        rng = np.random.RandomState(13)
        kth = (B1 << 21) | (300 << 10)
        below = pick(rng, B1 << 21, kth, K - 1)
        same = kth + 1 + rng.randint(0, 1023, total - K)
        above = np.concatenate([same, pick(rng, (B1 + 1) << 21, (B1 + 2) << 21, n - total)])
        keys_to_level(c, 0, 0, below, above, kth, rng)
        c.claims += [("branch", 0, 0, "narrowed" if total <= SEL_MAX else "fallback"), ("total", 0, 0, total), ("slot", 0, 0, "sub_first")]
        out.append(c)
    # fall-back: the level sits 1..K ulps above one score that fills the boundary sub-bin (the whole level is sorted)
    c = Case("select", "fallback", pre=K, seed=14)
    s = np.full(n, 0.75, F32)
    top = np.random.RandomState(15).permutation(n)[:K]
    s[top] = (0.75 + (K - np.arange(K)) * 2.0 ** -24).astype(F32)
    c.set_scores(0, 0, s)
    c.claims.append(("branch", 0, 0, "fallback"))
    out.append(c)
    # the selection thresholds: pre_nms around n / 4 and at the engine's largest
    for pre, br in ((3071, "narrowed"), (3072, "k4"), (8192, "k4")):
        c = Case("select", "pre%d" % pre, pre=pre, seed=16)
        c.claims.append(("branch", 0, 0, br))
        if pre == 8192:
            c.claims += [("branch", 0, 1, "small"), ("cands", 0, 0, 8192)]          # P3: pre_nms >= n
        out.append(c)
    for pre in (1, 63, 64, 65, 127, 128, 129):
        c = Case("select", "pre%d" % pre, pre=pre, seed=17)
        c.claims += [("branch", 0, 0, "narrowed"), ("cands", 0, 0, pre)]            # NMS over 1, 63, 64, ... candidates
        out.append(c)
    # ties: a run of 41 equal scores over ranks 980..1020 (the device keeps its lowest anchor indices), and a level of one score
    c = Case("select", "tie_cut", pre=K, seed=18)
    s = c.get_scores(0, 0).copy()
    order = np.argsort(-s, kind="stable")
    s[order[980:1021]] = s[order[980]]
    c.set_scores(0, 0, s)
    c.claims += [("branch", 0, 0, "narrowed"), ("tie_cut", 0, 0)]
    out.append(c)
    c = Case("select", "all_equal", pre=K, seed=19)
    for l in range(LEVELS):
        c.set_scores(0, l, np.full(A * int(np.prod(c.dims(0, l))), 0.5, F32))
    c.claims += [("branch", 0, 0, "fallback"), ("tie_cut", 0, 0), ("tie_cut", 0, 1)]
    out.append(c)
    return out


def mixed_cases():
    """One launch, two images: P2 of 42 x 64 cells (8064 anchors: sorted whole) and of 43 x 64 (8256: narrowed), then a full image
    whose P2 narrows next to one (64 x 48 cells) whose P2 falls back."""
    c = Case("mixed", "n8192", net_hw=((168, 256), (172, 256)), seed=20)
    c.claims += [("branch", 0, 0, "small"), ("branch", 1, 0, "narrowed")]
    d = Case("mixed", "narrow_fallback", net_hw=((256, 256), (256, 192)), seed=21)
    n = A * int(np.prod(d.dims(1, 0)))
    d.set_scores(1, 0, np.full(n, 0.625, F32))
    d.claims += [("branch", 0, 0, "narrowed"), ("branch", 1, 0, "fallback")]
    return [c, d]


def _far(c, b, l, i, dx, dy):
    c.set_delta(b, l, i, [dx, dy, 0, 0])


def filter_cases():
    out = []
    # min_size 16 at scale 0.75: widths / heights of exactly 12 are kept, 11 dropped.  32 x 32 anchors (a = 1) on P2 moved so
    # that the left / top border clips them to those sizes, with the top scores
    c = Case("filter", "min_size", net_hw=((256, 256),), min_size=16.0, scale=(0.75,), seed=30)
    h, w = c.dims(0, 0)
    top = 0.95
    for k, (what, wd, ht) in enumerate((("ws_eq", 12, 32), ("ws_below", 11, 32), ("hs_eq", 32, 12), ("hs_below", 32, 11))):
        for r in range(4):
            i = ((8 + 8 * k) * w + 4 + 12 * r) * A + 1
            o = 32 * (4 * (k % 2) + r) + 32          # disjoint: 8 boxes down the left border, 8 along the top
            box = [wd - 32, o, wd - 1, o + 31] if ht == 32 else [o, ht - 32, o + 31, ht - 1]
            c.place(0, 0, i, box, top - 0.001 * (4 * k + r))
            c.claims.append(("edge", 0, 0, what, i))
    out.append(c)
    # anchors pushed far outside the image: clipped to points and lines on the border.  xc < im_w holds for every clipped box
    # (x1, x2 <= im_w - 1 give xc = (x1 + x2 + 1) / 2 <= im_w - 0.5): the right / bottom border reaches the largest xc / yc
    c = Case("filter", "border", net_hw=((256, 256),), seed=31)
    h, w = c.dims(0, 0)
    for k in range(40):
        i = ((k % 8) * w + k) * A + k % 3
        dx, dy = ((50, 0), (0, 50), (50, 50), (-50, 0), (0, -50), (-50, -50), (50, -50), (-50, 50))[k % 8]
        _far(c, 0, 0, i, dx, dy)
        c.scores[0][0][k % 3, k % 8, k] = F32(0.99 - 0.001 * k)
        if dx > 0:
            c.claims.append(("edge", 0, 0, "xc_max", i))
        if dy > 0:
            c.claims.append(("edge", 0, 0, "yc_max", i))
    out.append(c)
    # a ragged pair: the second image (160 x 96) clips against its own size, not the canvas
    c = Case("filter", "border_ragged", net_hw=((256, 256), (160, 96)), seed=32)
    h, w = c.dims(1, 0)
    for k in range(20):
        i = ((k % 4) * w + k) * A + 1
        dx, dy = ((40, 40), (40, -40), (-40, 40), (-40, -40))[k % 4]
        _far(c, 1, 0, i, dx, dy)
        c.scores[1][0][1, k % 4, k] = F32(0.99 - 0.001 * k)
        if dx > 0:
            c.claims.append(("edge", 1, 0, "xc_max", i))
        if dy > 0:
            c.claims.append(("edge", 1, 0, "yc_max", i))
    out.append(c)
    # every candidate of P4 shrinks below min_size (dw = dh = -8: widths ~ 1 pixel), and all of P6
    c = Case("filter", "level_empty", net_hw=((256, 256),), min_size=16.0, scale=(0.75,), seed=33)
    for l in (2, 4):
        c.deltas[0][l][2::4] = -8
        c.deltas[0][l][3::4] = -8
        c.claims.append(("filtered_all", 0, l))
    out.append(c)                   # the inexact (expf(-8)) boxes are all filtered out: what remains is bit-exact
    # size deltas above the clip log(1000 / 16) on the 50 best anchors of P2: centres placed so that the right edge of each
    # 62.5x-wide box lands inside the image, where it depends on expf(clip) (compared within 2e-4)
    c = Case("filter", "dw_clip", net_hw=((256, 256),), seed=34)
    rng = np.random.RandomState(35)
    h, w = c.dims(0, 0)
    for i in np.argsort(-c.get_scores(0, 0), kind="stable")[:50]:
        anc = c.anchor_box(0, i, w).astype(np.float64)
        aw = anc[2] - anc[0] + 1
        target = rng.uniform(20, 230)
        pcx = target + 1 - 0.5 * aw * np.exp(4.135166556742356)
        c.set_delta(0, 0, i, [(pcx - (anc[0] + 0.5 * aw)) / aw, 0, rng.uniform(4.2, 6), 0])
    c.exact = False
    out.append(c)
    return out


def nms_cases():
    out = []
    # nested boxes clipped at the left / top border: 14 x 32 inside 20 x 32 has IoU 448 / 640 = 0.7 exactly (suppressed), 13 x 32 inside
    # 20 x 32 has 0.65 (kept)
    c = Case("nms", "iou_eq", seed=40)
    h, w = c.dims(0, 0)
    s = 0.99
    for k in range(6):
        y = 10 + 40 * k
        i, j, m = [((4 * k + 2) * w + 10 + 4 * t) * A + 1 for t in range(3)]
        if k % 2 == 0:
            c.place(0, 0, i, [-12, y, 19, y + 31], s)
            c.place(0, 0, j, [-18, y, 13, y + 31], s - 0.001)
            c.place(0, 0, m, [-19, y + 0, 12, y + 31], s - 0.002)
        else:
            x = 40 * k
            c.place(0, 0, i, [x, -12, x + 31, 19], s)
            c.place(0, 0, j, [x, -18, x + 31, 13], s - 0.001)
            c.place(0, 0, m, [x, -19, x + 31, 12], s - 0.002)
        c.claims += [("iou", 0, 0, i, j, 0.7), ("iou", 0, 0, i, m, 0.65)]
        s -= 0.01
    out.append(c)
    # every candidate of P2 and P3 the same box (only the 32 x 32 / 64 x 64 anchors score): one survivor each
    c = Case("nms", "identical", seed=41)
    for l in (0, 1):
        h, w = c.dims(0, l)
        sc = c.get_scores(0, l).copy()
        sc[np.arange(len(sc)) % A != 1] *= 0.01
        c.set_scores(0, l, sc)
        side = 32 << l
        for i in np.flatnonzero(np.arange(len(sc)) % A == 1):
            c.place(0, l, i, [20, 30, 20 + side - 1, 30 + side - 1])
        c.claims.append(("survivors", 0, l, 1))
    out.append(c)
    # post_nms 100 and 1: more survivors than are kept
    for post in (100, 1):
        c = Case("nms", "post%d" % post, post=post, seed=42 + post)
        c.claims.append(("survivors_over", 0, 0, post))
        out.append(c)
    return out


def collect_cases():
    out = []
    # scores from four values on every level: ties within and across levels through the collect's top-1000 cut
    c = Case("collect", "cross_level_ties", seed=50)
    rng = np.random.RandomState(51)
    vals = np.array([0.875, 0.75, 0.625, 0.5], F32)
    for l in range(LEVELS):
        n = A * int(np.prod(c.dims(0, l)))
        c.set_scores(0, l, vals[rng.randint(0, 4, n)])
    c.claims += [("cross_level_tie", 0), ("collect_cut", 0), ("tie_cut", 0, 0)]
    out.append(c)
    # P3 and P5 empty (every candidate below min_size), the other levels more than top_n together
    c = Case("collect", "empty_levels", min_size=16.0, scale=(0.75,), seed=52)
    for l in (1, 3):
        c.deltas[0][l][2::4] = -8
        c.deltas[0][l][3::4] = -8
        c.claims.append(("filtered_all", 0, l))
    c.claims.append(("collect_cut", 0))
    out.append(c)
    return out


def all_cases():
    cases = select_cases() + mixed_cases() + filter_cases() + nms_cases() + collect_cases()
    assert len({c.id for c in cases}) == len(cases)
    return cases


# ------------------------------------------------------------------------------------------------ FPN level boundaries
# map_rois_to_fpn_levels: floor(4 + log2(sqrt(area) / 224 + 1e-6)) in float32 changes level at areas near 112^2, 224^2 and 448^2.
BOUNDARY_AREAS = (112 * 112, 224 * 224, 448 * 448)
BOUNDARY_ULPS = 4096
NAMED_AREAS = (12543.9453125, 12543.9462890625, 12543.947265625, 200703.71875, 200703.734375)


def boundary_areas():
    """Every float32 area within +-BOUNDARY_ULPS ulps of each boundary area."""
    out = []
    for a in BOUNDARY_AREAS:
        bits = np.array(a, F32).view(np.int32) + np.arange(-BOUNDARY_ULPS, BOUNDARY_ULPS + 1, dtype=np.int32)
        out.append(bits.view(F32))
    return np.concatenate(out)


def boundary_boxes(areas, canvas=512):
    """One box per area whose (x2 - x1 + 1) * (y2 - y1 + 1) is exactly that area in float32 and which fits a canvas x canvas
    image: the height is the power of two 128 / 256 / 512 nearest above sqrt(area), the width area / height (exact in
    float32), x1 = y1 = 0."""
    areas = np.asarray(areas, F32)
    h = (2.0 ** np.ceil(np.log2(np.sqrt(areas.astype(np.float64)) * 1.01))).astype(F32)
    wd = (areas / h).astype(F32)
    boxes = np.zeros((len(areas), 4), F32)
    boxes[:, 2] = wd - F32(1)
    boxes[:, 3] = h - F32(1)
    assert np.all(boxes[:, 2:] < canvas)
    return boxes


def box_areas(boxes):
    boxes = np.asarray(boxes, F32)
    return ((boxes[:, 2] - boxes[:, 0] + F32(1)) * (boxes[:, 3] - boxes[:, 1] + F32(1))).astype(F32)


# ------------------------------------------------------------------------------------------------ oracle
def oracle_level(case, b, l, tie_order="stable", post=None):
    """generate_proposals_level on image b, level l of `case`: (props [k, 4], scores [k, 1], stages) as torch / numpy."""
    import torch
    from oracle import ref
    h, w = case.net_hw[b]
    return ref.generate_proposals_level(torch.from_numpy(case.scores[b][l][None]), torch.from_numpy(case.deltas[b][l][None]), h, w,
                                        float(case.scale[b]), 1.0 / stride(l), (32 << l,), pre_nms_top_n=case.pre,
                                        post_nms_top_n=case.post if post is None else post, nms_thresh=NMS, min_size=case.min_size,
                                        return_stages=True, tie_order=tie_order)


def expected(case, tie_order="stable"):
    """Per image: ([(props, scores, stages)] per level, (collected rois [n, 4] numpy, their levels)) under the oracle with
    `tie_order` (the collect sorts stably when it is "stable")."""
    from oracle import ref
    out = []
    for b in range(case.B):
        lv = [oracle_level(case, b, l, tie_order) for l in range(LEVELS)]
        _, _, rois, lvls = ref.collect_and_distribute([p for p, _, _ in lv], [s for _, s, _ in lv], post_nms_top_n=case.post,
                                                      stable=tie_order == "stable")
        out.append((lv, (rois.numpy(), lvls)))
    return out

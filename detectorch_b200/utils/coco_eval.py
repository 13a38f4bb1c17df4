"""COCO box and mask evaluation on the device: pycocotools' COCOeval ('bbox' / 'segm'; its default thresholds, area ranges and maxDets,
any imgIds / catIds / useCats) without its per-(image, category) Python loops.  Precision, recall and scores are bit-identical to COCOeval.evaluate() + accumulate() run on the results
file that lib/utils/json_dataset_evaluator.py would write; no file is written.

    gt = CocoGroundTruth("instances_minival2014.json")   # or the annotation dict; GT masks are built once, on the device
    E = evaluate(gt, detector.detect_images(ims), "segm")  # or evaluate(gt, all_boxes, "bbox") / evaluate(gt, all_boxes, "segm", all_segms)
    E.stats, E.eval["precision"]                          # summarize()'s 12 numbers, [T, R, K, A, M]
    acc = DeviceResults(); acc.add(detector.detect(...), image_ids, original_sizes=orig); evaluate(gt, acc, "segm")   # no host copy
    p = Params(gt, "bbox"); p.imgIds = ids[:500]; p.useCats = 0; E = evaluate(gt, results, "bbox", params=p)   # subsets, class-agnostic
    E = evaluate(gt, results, "bbox", keep_eval_imgs=True)  # + COCOeval's per-image records:
    E.eval_imgs["dtMatches"], E.evalImgs[n]               # as flat columns, or as COCOeval's list of dicts (built when first read)
    R = load_results(gt, "segm_results.json"); E = evaluate(gt, R, "segm")   # a results file, parsed on the device (COCO.loadRes)

keep_eval_imgs=True runs one more kernel after the evaluation, on the IoUs it kept; the records' detection ids are the ones loadRes
gives the rows of the results file (1 + the row's index), their GT ids the annotation ids.

The host only checks and flattens the annotations and results into arrays (csrc/coco_eval.cuh documents their layout); everything
numeric runs in the CUDA kernels of coco_eval.cuh.  Malformed annotations or results raise ValueError before the evaluation is
launched (segm results' run sums are checked by a small kernel first)."""
import collections
import json
import math

import numpy as np
import torch

from .. import _lib

# COCOeval's Params.setDetParams
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ['all', 'small', 'medium', 'large']
KIND_POLY, KIND_COUNTS, KIND_STRING = 0, 1, 2
_GT_BUDGET_INTS = 1 << 26        # GT masks are built in chunks of at most this much int32 workspace + output
_COORD_MAX = 1e8                 # polygon coordinates: x5 upsampled to int32 by maskApi


def _params():
    p = np.zeros(119, np.float64)
    p[0:8] = np.array(AREA_RNG, np.float64).reshape(-1)
    p[8:18] = [min([t, 1 - 1e-10]) for t in IOU_THRS]
    p[18:] = REC_THRS
    return p


def _p(t):
    return None if t is None else t.data_ptr()


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _int(v, what):
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
        raise ValueError("%s must be an integer, got %r" % (what, v))
    return int(v)


def _num(v, what):
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(float(v)):
        raise ValueError("%s must be a finite number, got %r" % (what, v))
    return float(v)


def _size(seg, what):
    sz = seg.get('size')
    if not isinstance(sz, (list, tuple)) or len(sz) != 2:
        raise ValueError("%s: RLE 'size' must be [h, w]" % what)
    h, w = _int(sz[0], what + " size"), _int(sz[1], what + " size")
    if h < 1 or w < 1 or h * w >= 2 ** 32:
        raise ValueError("%s: RLE size %dx%d outside [1, 2^32) pixels" % (what, h, w))
    return h, w


def _check_strings(buf, lens, what):
    """maskApi rleFrString reads 6-bit chars 48..111, a value ends on a char without bit 0x20; values are kept to <= 6 chars (< 2^30)."""
    if len(buf) == 0:
        return
    b = np.frombuffer(buf, np.uint8).astype(np.int32)
    if b.min() < 48 or b.max() > 111:
        raise ValueError("%s: RLE string with a character outside '0'..'o'" % what)
    cont = ((b - 48) & 0x20) != 0
    ends = np.cumsum(lens)[lens > 0] - 1
    if np.any(cont[ends]):
        raise ValueError("%s: RLE string ends inside a value" % what)
    stops = np.flatnonzero(~cont)
    if np.max(np.diff(np.concatenate([[-1], stops])) - 1) > 5:
        raise ValueError("%s: RLE string with a value longer than 6 characters" % what)


_SUM_BLOCK_CHARS = 1 << 20      # _string_sums works on blocks of whole strings of about this many chars (bounded temporaries)


def _string_sums(buf, lens):
    """The sum of the run lengths rleFrString decodes from each string (buf already passed _check_strings).  Linear in the chars,
    per-value temporaries only: chars 48..79 end a value; a value is its 5-bit groups, sign-extended from bit 4 of its last char;
    count m > 2 is its value plus count m - 2, in uint32."""
    lens = np.asarray(lens, np.int64)
    sums = np.zeros(len(lens), np.int64)
    if len(buf) == 0:
        return sums
    b = np.frombuffer(buf, np.uint8)
    ends = np.cumsum(lens)
    s0 = 0
    while s0 < len(lens):
        c0 = ends[s0] - lens[s0]
        s1 = max(int(np.searchsorted(ends, c0 + _SUM_BLOCK_CHARS, 'right')), s0 + 1)
        sums[s0:s1] = _string_sums_block(b[c0:ends[s1 - 1]], lens[s0:s1])
        s0 = s1
    return sums


def _string_sums_block(b, lens):
    """One block (< 2^31 chars): 32-bit arithmetic throughout, uint32 sums wrap as the C counts do."""
    stops = np.flatnonzero(b < 80).astype(np.int32)
    if len(stops) == 0:
        return np.zeros(len(lens), np.int64)
    nv = np.diff(np.searchsorted(stops, np.cumsum(lens)), prepend=0).astype(np.int32)     # values per string
    # the last char holds the top 5-bit group, sign-extended from its bit 4; the lower groups of the few longer values are added
    v = b[stops].astype(np.int32) - 48
    v -= (v & 0x10) << 1
    nch = np.diff(stops, prepend=np.int32(-1))
    i = np.flatnonzero(nch > 1)
    if len(i):
        n, s = nch[i], stops[i] - nch[i] + 1
        top = v[i] << (5 * (n - 1))
        for k in range(5):
            j = np.flatnonzero(n - 1 > k)
            top[j] += ((b[s[j] + k].astype(np.int32) - 48) & 0x1f) << (5 * k)
        v[i] = top
    u = v.view(np.uint32)
    vfirst = (np.cumsum(nv) - nv).astype(np.int32)
    first = np.repeat(vfirst, nv)                                            # each value's string's first value
    idx = np.arange(len(v), dtype=np.int32)
    odd, even = ((idx ^ first) & 1) == 1, ((idx ^ first) & 1) == 0
    even &= idx != first
    # counts 1, 3, 5.. and 2, 4, 6.. are running sums of their values, restarted at each string; count 0 stands alone
    p = np.zeros(len(v) + 1, np.uint32)
    q = np.zeros(len(v) + 1, np.uint32)
    np.cumsum(np.where(odd, u, np.uint32(0)), dtype=np.uint32, out=p[1:])
    np.cumsum(np.where(even, u, np.uint32(0)), dtype=np.uint32, out=q[1:])
    cnt = np.where(odd, p[1:] - p[first], np.where(even, q[1:] - q[first], u))
    out = np.zeros(len(lens), np.int64)
    full = nv > 0
    out[full] = np.add.reduceat(cnt, vfirst[full], dtype=np.int64)
    return out


def _check_sums(sums, h, w, what):
    """rleIou and rleMerge walk two masks' runs together until both end: runs that do not cover h * w pixels never end."""
    bad = np.flatnonzero(np.asarray(sums) != np.asarray(h, np.int64) * np.asarray(w, np.int64))
    if len(bad):
        raise ValueError("%s: RLE counts do not sum to h * w (mask %d)" % (what, bad[0]))


_MASK_PIXELS = 1 << 29           # pycocotools keeps GT masks as strings (polygons and uncompressed counts too): a count or count
                                 # difference outside [-2^29, 2^29) takes 7 chars, and rleFrString decodes some of those with int
                                 # shifts that overflow (-1 << 35 for negative ones, a last group of 2 or more << 30).  Masks of fewer
                                 # pixels never need 7 chars; larger polygon images are refused, larger counts checked one by one.


def _as_bytes(c, what):
    if isinstance(c, str):
        try:
            return c.encode('ascii')
        except UnicodeEncodeError:
            raise ValueError("%s: RLE string is not ASCII" % what) from None
    if isinstance(c, (bytes, bytearray)):
        return bytes(c)
    raise ValueError("%s: RLE 'counts' must be a string, bytes or a list of integers" % what)


def _upsampled_points(xy):
    """maskApi rleFrPoly's m: points of the x5 upsampled boundary ((int)(5 x + .5), then max(|dx|, |dy|) + 1 per edge)."""
    q = np.trunc(5.0 * xy + 0.5).astype(np.int64).reshape(-1, 2)
    d = np.abs(q - np.roll(q, -1, axis=0))
    return int(np.sum(np.maximum(d[:, 0], d[:, 1]) + 1))


class CocoGroundTruth:
    """The ground truth of a COCO annotation set (dict or json path) on the device, reusable across evaluations.  Images, categories
    and annotations are taken as pycocotools' COCO indexes them; annotations of unknown images or categories are left out, as
    COCOeval's getAnnIds does.  Polygon / uncompressed RLE / RLE masks are converted to RLE on the device (COCO.annToRLE)."""

    def __init__(self, annotations, device=None):
        if isinstance(annotations, str):
            with open(annotations) as f:
                annotations = json.load(f)
        if not isinstance(annotations, dict):
            raise ValueError("annotations must be a COCO annotation dict or the path of one")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        ds = annotations
        imgs, cats, anns = ds.get('images', []), ds.get('categories', []), ds.get('annotations', [])
        self.image_hw = {}
        for im in imgs:
            i = _int(im.get('id'), "image id")
            if i in self.image_hw:
                raise ValueError("duplicate image id %d" % i)
            h, w = _int(im.get('height'), "image %d height" % i), _int(im.get('width'), "image %d width" % i)
            if h < 1 or w < 1 or h * w >= 2 ** 32:
                raise ValueError("image %d: size %dx%d outside [1, 2^32) pixels" % (i, h, w))
            self.image_hw[i] = (h, w)
        self.category_ids = [_int(c.get('id'), "category id") for c in cats]       # dataset order: JsonDataset's contiguous classes
        if len(set(self.category_ids)) != len(self.category_ids):
            raise ValueError("duplicate category id")
        self.img_ids = sorted(self.image_hw)                                          # COCOeval params.imgIds / catIds
        self.cat_ids = sorted(self.category_ids)
        I, K = len(self.img_ids), len(self.cat_ids)
        img_index = {v: n for n, v in enumerate(self.img_ids)}
        cat_index = {v: n for n, v in enumerate(self.cat_ids)}
        seen, kept = set(), []
        for a in anns:
            aid = _int(a.get('id'), "annotation id")
            if aid in seen:
                raise ValueError("duplicate annotation id %d" % aid)
            seen.add(aid)
            i, k = img_index.get(a.get('image_id')), cat_index.get(a.get('category_id'))
            if i is not None and k is not None:
                kept.append((k * I + i, a))
        order = sorted(range(len(kept)), key=lambda n: kept[n][0])                  # stable: annotation order within a pair
        G = len(kept)
        self.num_images, self.num_cats, self.num_gts = I, K, G
        gt_f = np.zeros((G, 9), np.float64)
        gt_i = np.zeros((G, 6), np.int64)
        keys = np.zeros(G, np.int64)
        segs = []
        for n, o in enumerate(order):
            key, a = kept[o]
            what = "annotation %r" % a['id']
            keys[n] = key
            bb = a.get('bbox')
            if not isinstance(bb, (list, tuple)) or len(bb) != 4:
                raise ValueError("%s: bbox must be [x, y, w, h]" % what)
            gt_f[n, :4] = [_num(v, what + " bbox") for v in bb]
            gt_f[n, 4] = _num(a.get('area'), what + " area")
            crowd = a.get('iscrowd')
            if crowd not in (0, 1) or isinstance(crowd, float):
                raise ValueError("%s: iscrowd must be 0 or 1, got %r" % (what, crowd))
            h, w = self.image_hw[self.img_ids[key % I]]
            gt_i[n, 2:6] = [h, w, int(crowd), int(a['id'] != 0)]
            segs.append((a.get('segmentation'), h, w, what))
        self.keys = keys
        self.ann_ids = [kept[o][1]['id'] for o in order]                             # annotation ids in pair order
        self.cat_gt = np.searchsorted(keys // max(I, 1), np.arange(K + 1)).astype(np.int64) if I else np.zeros(K + 1, np.int64)
        self.has_masks = all(s[0] is not None for s in segs)
        self._gt_f, self._gt_i = gt_f, gt_i
        self.gt_counts = torch.zeros((1,), dtype=torch.int32, device=self.device)
        if self.has_masks and G:
            self._build_masks(segs)
        self.gt_f = torch.from_numpy(self._gt_f).to(self.device)
        self.gt_i = torch.from_numpy(self._gt_i).to(self.device)
        self.keys_d = torch.from_numpy(keys).to(self.device)                        # DeviceResults looks pairs' gts up on the device

    def _build_masks(self, segs):
        """Flatten every mask into the annotation / part tables, check it, then convert on the device in bounded chunks."""
        G = len(segs)
        ann = np.zeros((G, 6), np.int64)
        parts, xy, ucounts, chars = [], [], [], []
        nxy = ncnt = nch = 0
        ws_ints, out_cap = np.zeros(G, np.int64), np.zeros(G, np.int64)
        for n, (seg, h, w, what) in enumerate(segs):
            if isinstance(seg, list):
                if len(seg) == 0 or not all(isinstance(p, (list, tuple)) for p in seg):
                    raise ValueError("%s: polygon segmentation must be a non-empty list of coordinate lists" % what)
                # maskUtils.frPyObjects takes a first entry of 4 numbers for a box list and fails on it (frBbox wants an array)
                polys = []
                for p in seg:
                    if len(p) < 6 or len(p) % 2:
                        raise ValueError("%s: a polygon needs an even number (>= 6) of coordinates" % what)
                    polys.append(np.array([_num(v, what + " polygon") for v in p], np.float64))
                if h * w >= _MASK_PIXELS:
                    raise ValueError("%s: polygon on an image of %dx%d, 2^29 pixels or more" % (what, h, w))
                ann[n, :5] = [KIND_POLY, h, w, len(parts), len(polys)]
                for q in polys:
                    if np.abs(q).max() > _COORD_MAX:
                        raise ValueError("%s: polygon coordinate beyond %g" % (what, _COORD_MAX))
                    k, m = len(q) // 2, _upsampled_points(q)
                    if m >= 2 ** 31 // 4:
                        raise ValueError("%s: polygon too long" % what)
                    parts.append([nxy, k, int(ws_ints[n]), m])
                    ws_ints[n] += k + 4 * m + 3
                    out_cap[n] += m + 2
                    xy.append(q); nxy += k
                out_cap[n] += len(polys)
            elif isinstance(seg, dict) and 'counts' in seg and 'size' in seg:
                rh, rw = _size(seg, what)
                c = seg['counts']
                if isinstance(c, list):
                    v = np.array([_int(x, what + " counts") for x in c], np.int64)
                    if v.size and (v.min() < 0 or v.max() >= 2 ** 32):
                        raise ValueError("%s: RLE count outside [0, 2^32)" % what)
                    _check_sums([v.sum()], rh, rw, what)
                    # frPyObjects stores them as a string: count m > 2 as its difference to count m - 2, in at most 6 chars
                    d = np.concatenate([v[:3], v[3:] - v[1:-2]])
                    if d.size and (d.max() >= _MASK_PIXELS or d.min() < -_MASK_PIXELS):
                        raise ValueError("%s: RLE count difference outside [-2^29, 2^29)" % what)
                    ann[n, :5] = [KIND_COUNTS, rh, rw, len(parts), 1]
                    parts.append([ncnt, len(v), 0, 0]); ucounts.append(v.astype(np.uint32)); ncnt += len(v)
                    out_cap[n] = max(len(v), 1)
                else:
                    s = _as_bytes(c, what)
                    _check_strings(s, np.array([len(s)]), what)
                    _check_sums(_string_sums(s, np.array([len(s)])), rh, rw, what)
                    ann[n, :5] = [KIND_STRING, rh, rw, len(parts), 1]
                    parts.append([nch, len(s), 0, 0]); chars.append(s); nch += len(s)
                    out_cap[n] = max(len(s), 1)
                self._gt_i[n, 2:4] = [rh, rw]
            else:
                raise ValueError("%s: segmentation must be polygons or an RLE dict with 'size' and 'counts'" % what)
        parts = np.array(parts, np.int64).reshape(-1, 4)
        dev = self.device
        L = _lib.lib()
        xy_d = torch.from_numpy(np.concatenate(xy) if xy else np.zeros(2)).to(dev)
        uc_d = torch.from_numpy((np.concatenate(ucounts) if ucounts else np.zeros(1, np.uint32)).view(np.int32)).to(dev)
        ch_d = torch.from_numpy(np.frombuffer(b"".join(chars) or b"\0", np.uint8).copy()).to(dev)
        # chunks of annotations whose workspace + 2 output buffers fit the budget (a single larger annotation gets a chunk of its own)
        cost = ws_ints + 2 * out_cap
        self._mask_cost = cost
        lens, outs = np.zeros(G, np.int64), []
        n0 = 0
        while n0 < G:
            n1 = n0 + 1
            tot = cost[n0]
            while n1 < G and tot + cost[n1] <= _GT_BUDGET_INTS:
                tot += cost[n1]; n1 += 1
            a = ann[n0:n1].copy()
            a[:, 5] = np.concatenate([[0], np.cumsum(out_cap[n0:n1])[:-1]])
            p0, p1 = a[0, 3], (a[-1, 3] + a[-1, 4])
            pt = parts[p0:p1].copy()
            a[:, 3] -= p0
            poly = a[:, 0] == KIND_POLY
            # workspace offsets of the chunk's polygon parts: per annotation, after the previous annotations'
            wbase = np.concatenate([[0], np.cumsum(ws_ints[n0:n1])[:-1]])
            for r in np.flatnonzero(poly):
                pt[a[r, 3]:a[r, 3] + a[r, 4], 2] += wbase[r]
            ncap = int(out_cap[n0:n1].sum())
            ws = torch.empty((max(int(ws_ints[n0:n1].sum()), 1),), dtype=torch.int32, device=dev)
            out = torch.empty((ncap,), dtype=torch.int32, device=dev)
            tmp = torch.empty((ncap,), dtype=torch.int32, device=dev)
            olen = torch.empty((n1 - n0,), dtype=torch.int64, device=dev)
            obox = torch.empty((n1 - n0, 4), dtype=torch.float64, device=dev)
            a_d, p_d = torch.from_numpy(a).to(dev), torch.from_numpy(pt).to(dev)
            _lib.check(L.dt_coco_gt_build(n1 - n0, _p(a_d), _p(p_d), _p(xy_d), _p(uc_d), _p(ch_d), _p(ws), _p(out), _p(tmp), _p(olen), _p(obox),
                                          _stream(dev)), "dt_coco_gt_build")
            ln = olen.cpu().numpy()
            lens[n0:n1] = ln
            self._gt_f[n0:n1, 5:9] = obox.cpu().numpy()
            starts = torch.from_numpy(a[:, 5]).to(dev)
            ln_d = torch.from_numpy(ln).to(dev)
            idx = torch.repeat_interleave(starts, ln_d) + (torch.arange(int(ln.sum()), device=dev) -
                                                           torch.repeat_interleave(torch.cumsum(ln_d, 0) - ln_d, ln_d))
            outs.append(out[idx])
            n0 = n1
        self._gt_i[:, 0] = np.concatenate([[0], np.cumsum(lens)[:-1]])
        self._gt_i[:, 1] = lens
        self.gt_counts = torch.cat(outs) if int(lens.sum()) else torch.zeros((1,), dtype=torch.int32, device=dev)

    def rles(self):
        """The GT masks as pycocotools would hold them after COCO.annToRLE, in pair order: uint32 run lengths per annotation."""
        c = self.gt_counts.cpu().numpy().view(np.uint32)
        return [c[o:o + n].copy() for o, n in self._gt_i[:, :2]]


class Params:
    """COCOeval's Params for 'bbox' / 'segm', with gt's images and categories.  evaluate(..., params=) takes one edited as on a COCOeval
    object: imgIds (a subset of the images), catIds (a subset of the categories) and useCats (0: class-agnostic matching).  iouThrs,
    recThrs, maxDets, areaRng and areaRngLbl must keep their defaults."""

    def __init__(self, gt, iou_type):
        self.imgIds, self.catIds = list(gt.img_ids), list(gt.cat_ids)
        self.iouThrs, self.recThrs = IOU_THRS.copy(), REC_THRS.copy()
        self.maxDets, self.areaRng, self.areaRngLbl = list(MAX_DETS), [list(a) for a in AREA_RNG], list(AREA_LBL)
        self.useCats, self.iouType = 1, iou_type


def _id_list(v, what, known):
    if isinstance(v, (str, bytes)) or not hasattr(v, '__len__'):
        raise ValueError("params.%s must be a list of ids" % what)
    ids = [_int(x, "params.%s entry" % what) for x in v]
    if not ids:
        raise ValueError("params.%s is empty" % what)
    bad = [x for x in ids if x not in known]
    if bad:
        raise ValueError("params.%s: %d is not in the ground truth" % (what, bad[0]))
    return ids


def _same(a, b):
    try:
        a = np.asarray(a, np.float64)
    except (TypeError, ValueError):
        return False
    return a.shape == np.shape(b) and np.array_equal(a, b)


def _normalised_params(gt, params, iou_type):
    """Checks params on the host and returns a copy normalised as COCOeval.evaluate() normalises it: imgIds unique and sorted, catIds
    too when useCats is 1 (with useCats 0 their order is the order in which each image's categories are concatenated), maxDets sorted."""
    if not isinstance(params, Params):
        raise ValueError("params must be a coco_eval.Params")
    if params.iouType != iou_type:
        raise ValueError("params.iouType is %r, the evaluation is %r" % (params.iouType, iou_type))
    if not _same(params.iouThrs, IOU_THRS):
        raise ValueError("params.iouThrs: only COCOeval's default IoU thresholds are supported")
    if not _same(params.recThrs, REC_THRS):
        raise ValueError("params.recThrs: only COCOeval's default recall thresholds are supported")
    if not (isinstance(params.maxDets, (list, tuple)) and _same(sorted(params.maxDets), MAX_DETS)):
        raise ValueError("params.maxDets: only COCOeval's default [1, 10, 100] is supported")
    if not _same(params.areaRng, AREA_RNG) or list(params.areaRngLbl) != AREA_LBL:
        raise ValueError("params.areaRng / areaRngLbl: only COCOeval's default area ranges are supported")
    if isinstance(params.useCats, float) or params.useCats not in (0, 1):
        raise ValueError("params.useCats must be 0 or 1, got %r" % (params.useCats,))
    p = Params(gt, iou_type)
    p.useCats = int(params.useCats)
    p.imgIds = [int(v) for v in np.unique(_id_list(params.imgIds, 'imgIds', gt.image_hw))]
    cats = _id_list(params.catIds, 'catIds', set(gt.cat_ids))
    if p.useCats:
        cats = [int(v) for v in np.unique(cats)]
    elif len(set(cats)) != len(cats):
        raise ValueError("params.catIds: a category is repeated (with useCats 0 its ground truth would count twice)")
    p.catIds = cats
    return p


def _is_default(gt, p):
    return p.useCats == 1 and p.imgIds == list(gt.img_ids) and p.catIds == list(gt.cat_ids)


class _GtView:
    """The ground truth re-indexed for a Params: the evaluated images and categories (one category, -1, when useCats is 0), pair keys
    over them, and the gt rows of those pairs gathered on the device (the masks stay where CocoGroundTruth built them).  It has the
    attributes of CocoGroundTruth that the evaluation reads.  per: category slots per pair (with useCats 0 the evaluated categories, in
    the order COCOeval concatenates them per image; else 1); cat_slot / img_slot: each category / image index of gt to its slot / index
    here, -1 when it takes no part."""

    def __init__(self, gt, p):
        self.device, self.has_masks, self.gt_counts = gt.device, gt.has_masks, gt.gt_counts
        self.img_ids = list(p.imgIds)
        self.cat_ids = list(p.catIds) if p.useCats else [-1]
        self.num_images, self.num_cats = len(self.img_ids), len(self.cat_ids)
        self.per = 1 if p.useCats else len(p.catIds)
        cat_index = {v: n for n, v in enumerate(gt.cat_ids)}
        img_index = {v: n for n, v in enumerate(gt.img_ids)}
        self.cat_slot = np.full(gt.num_cats, -1, np.int64)
        self.cat_slot[[cat_index[c] for c in p.catIds]] = np.arange(len(p.catIds))
        self.img_slot = np.full(gt.num_images, -1, np.int64)
        self.img_slot[[img_index[i] for i in p.imgIds]] = np.arange(self.num_images)
        self.I0 = gt.num_images
        rows, fine = self.select(gt.keys)
        self.rows = rows
        self.keys = fine // self.per
        self.num_gts = len(rows)
        self.ann_ids = [gt.ann_ids[r] for r in rows]
        self.cat_gt = np.searchsorted(self.keys // max(self.num_images, 1), np.arange(self.num_cats + 1)).astype(np.int64)
        rows_d = torch.from_numpy(rows).to(gt.device)
        self.gt_f, self.gt_i = gt.gt_f.index_select(0, rows_d), gt.gt_i.index_select(0, rows_d)
        self.keys_d = torch.from_numpy(self.keys).to(gt.device)

    def fine_key(self, k, i):
        """(category slot, image index) -> fine bin (csrc/coco_eval.cuh): pairs in a row, each pair's slots in concatenation order."""
        return i * self.per + k if self.per > 1 else k * self.num_images + i

    def select(self, key):
        """Rows keyed as gt keys them (category index * images + image index, sorted; rows of a key in their order) -> the rows that take
        part, in this view's order (stable), and their fine bins."""
        I0 = max(self.I0, 1)
        k, i = self.cat_slot[key // I0], self.img_slot[key % I0]
        rows = np.flatnonzero((k >= 0) & (i >= 0))
        fine = self.fine_key(k[rows], i[rows])
        o = np.argsort(fine, kind='stable')
        return rows[o], fine[o]


class CocoEvalResult:
    """What a COCOeval object holds after evaluate() + accumulate() (+ summarize() for .stats): .params, .eval, .stats; with
    evaluate(..., keep_eval_imgs=True) also .evalImgs, built from the columns .eval_imgs when first read."""
    eval_imgs = None

    def __init__(self, params, precision, recall, scores):
        self.params = params
        T, R, K, A, M = precision.shape
        self.eval = {'params': params, 'counts': [T, R, K, A, M], 'precision': precision, 'recall': recall, 'scores': scores}
        self.stats = self._stats(verbose=False)
        self._eval_imgs_list = None

    @property
    def evalImgs(self):
        if self.eval_imgs is None:
            raise AttributeError("evalImgs: evaluate(..., keep_eval_imgs=True) keeps the per-image records")
        if self._eval_imgs_list is None:
            self._eval_imgs_list = _eval_imgs_list(self.params, self.eval_imgs)
        return self._eval_imgs_list

    def summarize(self):
        self.stats = self._stats(verbose=True)

    def _stats(self, verbose):
        p = self.params

        def one(ap=1, iouThr=None, areaRng='all', maxDets=100):
            aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
            s = self.eval['precision'] if ap == 1 else self.eval['recall']
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
            mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
            if verbose:
                iouStr = '{:0.2f}:{:0.2f}'.format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else '{:0.2f}'.format(iouThr)
                print(' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'.format(
                    'Average Precision' if ap == 1 else 'Average Recall', '(AP)' if ap == 1 else '(AR)', iouStr, areaRng, maxDets, mean_s))
            return mean_s
        m = p.maxDets
        stats = np.zeros((12,))
        stats[0] = one(1)
        stats[1] = one(1, iouThr=.5, maxDets=m[2])
        stats[2] = one(1, iouThr=.75, maxDets=m[2])
        stats[3] = one(1, areaRng='small', maxDets=m[2])
        stats[4] = one(1, areaRng='medium', maxDets=m[2])
        stats[5] = one(1, areaRng='large', maxDets=m[2])
        stats[6] = one(0, maxDets=m[0])
        stats[7] = one(0, maxDets=m[1])
        stats[8] = one(0, maxDets=m[2])
        stats[9] = one(0, areaRng='small', maxDets=m[2])
        stats[10] = one(0, areaRng='medium', maxDets=m[2])
        stats[11] = one(0, areaRng='large', maxDets=m[2])
        return stats


def _per_class(gt, results, all_segms, iou_type):
    """results -> (all_boxes, all_segms) indexed [contiguous class][image]: detect_images / batch_results' per-image tuples are filed
    the way extend_results files them."""
    if isinstance(results, (list, tuple)) and len(results) and isinstance(results[0], tuple):
        if all_segms is not None:
            raise ValueError("per-image results carry their masks; all_segms is for all_boxes input")
        if len(results) != gt.num_images:
            raise ValueError("%d per-image results for %d images" % (len(results), gt.num_images))
        if any(len(r) != 4 for r in results):
            raise ValueError("per-image results are (scores, boxes, boxes_per_class, segms_per_class) tuples")
        nc = max(len(r[2]) for r in results)
        boxes = [[[] for _ in results] for _ in range(nc)]
        segms = [[[] for _ in results] for _ in range(nc)]
        for i, r in enumerate(results):
            for j in range(1, len(r[2])):
                boxes[j][i] = r[2][j]
                if r[3] is not None:
                    segms[j][i] = r[3][j]
                elif iou_type == 'segm':
                    raise ValueError("segm evaluation of results without masks")
        return boxes, segms
    if iou_type == 'segm' and all_segms is None:
        raise ValueError("segm evaluation of all_boxes needs all_segms")
    return results, all_segms


def _flatten_results(gt, all_boxes, all_segms, iou_type, category_ids, with_ids=False):
    """_write_coco_{bbox,segms}_results_file + COCO.loadRes, as arrays: one row per result in the file's order (class-major, images in
    sorted-id order), bbox = xyxy_to_xywh of the float64 boxes (+1 width), score = the float64 of the stored value.  Rows come back
    sorted by key (category index, image index); with_ids adds each row's loadRes id (1 + its index in the file) as a fifth value."""
    I = gt.num_images
    cat_index = {v: n for n, v in enumerate(gt.cat_ids)}
    segm = iou_type == 'segm'
    keys, dets, strs, hw = [], [], [], []
    for j in range(1, len(category_ids) + 1):
        if j >= len(all_boxes):
            break
        k = cat_index[category_ids[j - 1]]
        per_img = all_boxes[j]
        if len(per_img) != I:
            raise ValueError("class %d: %d entries for %d images" % (j, len(per_img), I))
        if segm and (j >= len(all_segms) or len(all_segms[j]) != I):
            raise ValueError("class %d: all_segms does not have one entry per image" % j)
        for i in range(I):
            d = per_img[i]
            if isinstance(d, list) and len(d) == 0:
                continue
            d = np.asarray(d)
            if d.ndim != 2 or d.shape[1] != 5:
                raise ValueError("class %d image %d: detections must be an N x 5 array" % (j, i))
            n = d.shape[0]
            keys.append((k * I + i, n))
            dets.append(d)
            if segm:
                rles = all_segms[j][i]
                if len(rles) < n:
                    raise ValueError("class %d image %d: %d masks for %d detections" % (j, i, len(rles), n))
                for r in rles[:n]:
                    if not isinstance(r, dict) or 'counts' not in r or 'size' not in r:
                        raise ValueError("class %d image %d: RLE dicts with 'size' and 'counts' expected" % (j, i))
                    sz, c = r['size'], r['counts']
                    hw.append(sz)
                    strs.append(c.encode() if isinstance(c, str) else _as_bytes(c, "class %d image %d mask" % (j, i)))
    # the float64 view of each stored value, then xyxy_to_xywh (+1) -- elementwise, so done once over the concatenation
    d = np.concatenate([x.astype(np.float64) for x in dets]) if dets else np.zeros((0, 5))
    if not np.all(np.isfinite(d)):
        raise ValueError("non-finite box or score in the results")
    N = len(d)
    key = np.repeat(np.array([a for a, _ in keys], np.int64), [n for _, n in keys]) if keys else np.zeros(0, np.int64)
    det_f = np.zeros((N, 5), np.float64)
    det_i = np.zeros((N, 4), np.int64)
    det_f[:, 0] = d[:, -1]
    det_f[:, 1:5] = np.hstack((d[:, 0:2], d[:, 2:4] - d[:, 0:2] + 1))
    chars = b""
    if segm and N:
        sizes = np.array(hw, dtype=object)
        if sizes.ndim != 2 or sizes.shape[1] != 2 or not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in sizes.flat):
            raise ValueError("results: RLE 'size' must be [h, w] integers")
        sizes = sizes.astype(np.int64)
        if np.any(sizes < 1) or np.any(sizes[:, 0] * sizes[:, 1] >= 2 ** 32):
            raise ValueError("results: RLE size outside [1, 2^32) pixels")
        lens = np.fromiter((len(s) for s in strs), np.int64, N)
        try:
            chars = b"".join(strs)
        except TypeError:
            raise ValueError("results: RLE 'counts' must be strings") from None
        _check_strings(chars, lens, "results")
        det_i[:, 0] = np.concatenate([[0], np.cumsum(lens)[:-1]])
        det_i[:, 1] = lens
        det_i[:, 2:4] = sizes
    order = np.argsort(key, kind='stable')
    if with_ids:
        return key[order], det_f[order], det_i[order], chars, order + 1
    return key[order], det_f[order], det_i[order], chars


def evaluate(gt, results, iou_type, all_segms=None, category_ids=None, keep_ious=False, keep_eval_imgs=False, params=None):
    """COCOeval(gt, loadRes(results file), iou_type).evaluate() + accumulate() on the device -> CocoEvalResult.
    results: detect_images() / batch_results() output (one tuple per image, images in sorted-id order), the notebooks' all_boxes
    [class][image] (with all_segms [class][image] for 'segm'), a DeviceResults (flattened on the device, on gt's device), or a
    LoadedResults (load_results(gt, results file): the evaluation is COCOeval(G, G.loadRes(file), iou_type)'s).  category_ids: json id of contiguous class j (1-based) at j - 1;
    default: the dataset's category order, as JsonDataset builds its classes.  keep_ious: also return COCOeval's .ious, {(image id,
    category id): [min(D, 100), G] array} for the pairs with detections and GTs.  keep_eval_imgs: also return COCOeval's per-image
    records, as .eval_imgs (columns, see _eval_imgs_columns) and .evalImgs (the list of dicts, built from the columns when first read);
    detection ids are the ones loadRes gives the results file's rows, 1 + the row's index.
    params: a Params (Params(gt, iou_type), then edited) whose imgIds, catIds and useCats are evaluated as COCOeval evaluates them:
    only the listed images' and categories' gts and detections take part (detections on other images are left out), and with useCats 0
    each image's detections and gts of all listed categories are matched together (one category, -1, as accumulate() makes it).  The
    other fields must keep their defaults.  Bad params raise ValueError before anything is launched; the result's .params is the
    one used, normalised as COCOeval.evaluate() normalises it.  None: the defaults."""
    if iou_type not in ('bbox', 'segm'):
        raise ValueError("iou_type must be 'bbox' or 'segm'")
    if not isinstance(gt, CocoGroundTruth):
        raise TypeError("gt must be a CocoGroundTruth")
    if iou_type == 'segm' and not gt.has_masks:
        raise ValueError("segm evaluation: some ground-truth annotations have no segmentation")
    if isinstance(results, LoadedResults):
        if all_segms is not None or category_ids is not None:
            raise ValueError("a LoadedResults carries its masks and json category ids; all_segms and category_ids are for all_boxes input")
        p = Params(gt, iou_type) if params is None else _normalised_params(gt, params, iou_type)
        return _evaluate_loaded(gt, results, iou_type, keep_ious, keep_eval_imgs, p)
    category_ids = list(gt.category_ids if category_ids is None else category_ids)
    if any(c not in set(gt.cat_ids) for c in category_ids):
        raise ValueError("category_ids names a category the ground truth does not have")
    p = Params(gt, iou_type) if params is None else _normalised_params(gt, params, iou_type)
    view = None if _is_default(gt, p) else _GtView(gt, p)
    ev = gt if view is None else view
    if isinstance(results, DeviceResults):
        if all_segms is not None:
            raise ValueError("a DeviceResults carries its masks; all_segms is for all_boxes input")
        f = _flatten_device(gt, results, iou_type, category_ids, keep_eval_imgs, view)
        imgs = (f['union'], f['det_ids']) if keep_eval_imgs else None
        return _evaluate_tables(ev, iou_type, None, f['pairs'], f['cat_kept'], f['order_off'], f['det_f'], f['det_i'], f['chars'],
                                f['num_chars'], f['num_kept'], f['num_ious'], f['num_order'], keep_ious, imgs, p)
    boxes, segms = _per_class(gt, results, all_segms, iou_type)
    key, det_f, det_i, chars, det_ids = _flatten_results(gt, boxes, segms, iou_type, category_ids, with_ids=True)
    if view is not None:
        rows, fine = view.select(key)
        key, det_f, det_i, det_ids = fine // view.per, det_f[rows], det_i[rows], det_ids[rows]
    pairs, cat_kept, order_off = _pair_tables(ev, key)
    kept, gn = np.minimum(pairs[:, 2], MAX_DETS[-1]), pairs[:, 4]
    n_kept, n_iou, n_order = int(kept.sum()), int((kept * gn).sum()), int(order_off[-1, -1])
    dev = gt.device
    up = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (pairs, cat_kept, order_off, det_f, det_i)]
    ch = torch.from_numpy(np.frombuffer(chars or b"\0", np.uint8).copy()).to(dev)
    imgs = None
    if keep_eval_imgs:
        # the pairs COCOeval keeps a record of: those with detections and those with gts
        imgs = tuple(torch.from_numpy(x).to(dev) for x in (np.union1d(pairs[:, 0], ev.keys).astype(np.int64), det_ids.astype(np.int64)))
    return _evaluate_tables(ev, iou_type, pairs, *up, ch, len(chars), n_kept, n_iou, n_order, keep_ious, imgs, p)


def _pair_tables(gt, key):
    """dt_coco_eval's tables of the (category, image) pairs with detections, for results sorted by key = k * I + i -> (pairs [P, 7]:
    key, first detection, D, first gt, G, first kept slot, first IoU; cat_kept [K + 1]; order_off [3, K + 1])."""
    I, K = gt.num_images, gt.num_cats
    pk, pstart, pcount = np.unique(key, return_index=True, return_counts=True)
    g0 = np.searchsorted(gt.keys, pk, 'left')
    gn = np.searchsorted(gt.keys, pk, 'right') - g0
    kept = np.minimum(pcount, MAX_DETS[-1])
    pairs = np.zeros((len(pk), 7), np.int64)
    pairs[:, 0], pairs[:, 1], pairs[:, 2], pairs[:, 3], pairs[:, 4] = pk, pstart, pcount, g0, gn
    pairs[:, 5] = np.concatenate([[0], np.cumsum(kept)[:-1]])
    pairs[:, 6] = np.concatenate([[0], np.cumsum(kept * gn)[:-1]])
    pcat = pk // max(I, 1)
    cat_kept = np.concatenate([[0], np.cumsum(np.bincount(pcat, weights=kept, minlength=K)[:K].astype(np.int64))])
    order_off = np.zeros((3, K + 1), np.int64)
    base = 0
    for m, cut in enumerate(MAX_DETS):
        c = np.bincount(pcat, weights=np.minimum(pcount, cut), minlength=K)[:K].astype(np.int64)
        order_off[m] = base + np.concatenate([[0], np.cumsum(c)])
        base = order_off[m, -1]
    return pairs, cat_kept, order_off


def _evaluate_tables(gt, iou_type, pairs, pairs_d, cat_kept_d, order_off_d, det_f_d, det_i_d, ch, num_chars, n_kept, n_iou, n_order, keep_ious,
                     imgs, params, det_area_d=None):
    """dt_coco_eval on the flattened results, already on gt's device (pairs: their host copy, or None to read it back for keep_ious).
    gt: the CocoGroundTruth, or its _GtView for params.  imgs: (union keys [Q], detection ids [N]) on the device to also run
    dt_coco_eval_imgs, None to leave it out.  det_area_d: each detection's area for the area ranges (a results file's loadRes area),
    None for w h of the box ('bbox') or the RLE area ('segm')."""
    I, K, N = gt.num_images, gt.num_cats, int(det_f_d.shape[0])
    dev = gt.device
    T, R, A, M = len(IOU_THRS), len(REC_THRS), len(AREA_RNG), len(MAX_DETS)
    prec = torch.empty((T, R, K, A, M), dtype=torch.float64, device=dev)
    rec = torch.empty((T, K, A, M), dtype=torch.float64, device=dev)
    scr = torch.empty((T, R, K, A, M), dtype=torch.float64, device=dev)
    L = _lib.lib()
    cat_gt_d, par_d = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (gt.cat_gt, _params()))
    if iou_type == 'segm' and N:
        # runs that do not cover h * w pixels would make rleIou's merge loop forever: decoded and summed on the device, refused here
        bad = torch.empty((N,), dtype=torch.uint8, device=dev)
        _lib.check(L.dt_coco_det_check(N, _p(det_i_d), _p(ch), _p(bad), _stream(dev)), "dt_coco_det_check")
        nb = torch.nonzero(bad).flatten()[:1].cpu().numpy()
        if len(nb):
            raise ValueError("results: RLE counts of result %d (in (category, image) order) do not sum to h * w" % nb[0])
    # the records read the IoU matrices dt_coco_eval keeps, rather than computing them again
    ious = torch.empty((max(n_iou, 1),), dtype=torch.float64, device=dev) if keep_ious or imgs is not None else None
    ws_bytes = L.dt_coco_eval_workspace_bytes(N, num_chars, n_kept, n_iou, gt.num_gts, n_order, K)
    if ws_bytes <= 0 and N:
        raise ValueError("evaluate: %d kept detections are more than the evaluation can rank" % n_kept)
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
    _lib.check(L.dt_coco_eval(1 if iou_type == 'segm' else 0, I, K, int(pairs_d.shape[0]), _p(pairs_d), _p(cat_gt_d), _p(cat_kept_d),
                              _p(order_off_d), N, _p(det_f_d), _p(det_i_d), _p(ch), num_chars, n_kept, n_iou, gt.num_gts, n_order, _p(gt.gt_f),
                              _p(gt.gt_i), _p(gt.gt_counts), _p(par_d), _p(prec), _p(rec), _p(scr), _p(ious), _p(ws), _stream(dev),
                              _p(det_area_d)), "dt_coco_eval")
    if imgs is not None:
        ukeys_d, det_ids_d = imgs
        Q, G = int(ukeys_d.shape[0]), gt.num_gts
        slot_det = torch.empty((max(n_kept, 1),), dtype=torch.int32, device=dev)
        dt_gt = torch.empty((max(n_kept, 1), A * T), dtype=torch.int32, device=dev)
        dt_ig = torch.empty((max(n_kept, 1), A * T), dtype=torch.uint8, device=dev)
        gt_dt = torch.empty((max(G, 1), A * T), dtype=torch.int32, device=dev)
        gt_pos = torch.empty((max(G, 1), A), dtype=torch.int32, device=dev)
        gt_ig = torch.empty((max(G, 1), A), dtype=torch.uint8, device=dev)
        _lib.check(L.dt_coco_eval_imgs(1 if iou_type == 'segm' else 0, Q, _p(ukeys_d), int(pairs_d.shape[0]), _p(pairs_d), N, _p(det_f_d),
                                       num_chars, n_kept, n_iou, G, n_order, _p(gt.keys_d), _p(gt.gt_f), _p(gt.gt_i), _p(par_d), _p(ious), _p(ws),
                                       _p(slot_det), _p(dt_gt), _p(dt_ig), _p(gt_dt), _p(gt_pos), _p(gt_ig), _stream(dev),
                                       _p(det_area_d)), "dt_coco_eval_imgs")
        # each kept slot's detection id and score, gathered on the device
        sd = slot_det[:n_kept].long()
        slot_id, slot_score = det_ids_d[sd], det_f_d[sd, 0]
        dev_out = dict(ukeys=ukeys_d, slot_id=slot_id, slot_score=slot_score, dt_gt=dt_gt[:n_kept], dt_ig=dt_ig[:n_kept], gt_dt=gt_dt[:G],
                       gt_pos=gt_pos[:G], gt_ig=gt_ig[:G])
    E = CocoEvalResult(params, prec.cpu().numpy(), rec.cpu().numpy(), scr.cpu().numpy())
    if (keep_ious or imgs is not None) and pairs is None:
        pairs = pairs_d.cpu().numpy()
    if imgs is not None:
        E.eval_imgs = _eval_imgs_columns(gt, pairs, {k: v.cpu().numpy() for k, v in dev_out.items()})
    if keep_ious:
        pk, kept, gn = pairs[:, 0], np.minimum(pairs[:, 2], MAX_DETS[-1]), pairs[:, 4]
        iv = ious.cpu().numpy()
        E.ious = {(gt.img_ids[k % I], gt.cat_ids[k // I]): iv[o:o + d * g].reshape(d, g)
                  for k, d, g, o in zip(pk, kept, gn, pairs[:, 6]) if g > 0}
    return E


def _eval_imgs_columns(gt, pairs, o):
    """dt_coco_eval_imgs' outputs (host copies, with each kept slot's detection id and score) -> COCOeval.evalImgs as flat columns.
    The records are evalImgs' non-None entries in its order (category, area range, image), one per area range of each pair with
    detections or gts; record r owns detection rows dt_off[r]:dt_off[r + 1] (score order, cut to 100) and gt rows gt_off[r]:gt_off[r + 1]
    (the area range's ignore-last order):
        index [R]                         the record's position in evalImgs (K * 4 * I entries)
        image_id, category_id, area [R]   its json ids and area range index
        dt_off, gt_off [R + 1]
        dtIds [n_dt] int64, dtScores [n_dt] float64, dtMatches [10, n_dt] float64 (matched gt's id, 0 for none), dtIgnore [10, n_dt] bool
        gtIds [n_gt] int64, gtIgnore [n_gt] int64, gtMatches [10, n_gt] float64 (id of the last detection that matched, 0 for none)"""
    I, A, T = gt.num_images, len(AREA_RNG), len(IOU_THRS)
    uk = o['ukeys']
    Q, P, n_kept = len(uk), len(pairs), len(o['slot_id'])
    pi = np.minimum(np.searchsorted(pairs[:, 0], uk), max(P - 1, 0))
    has = pairs[pi, 0] == uk if P else np.zeros(Q, bool)
    Dk = np.where(has, np.minimum(pairs[pi, 2], MAX_DETS[-1]), 0) if P else np.zeros(Q, np.int64)
    k0 = np.where(has, pairs[pi, 5], 0) if P else np.zeros(Q, np.int64)
    g0 = np.searchsorted(gt.keys, uk, 'left')
    Gq = np.searchsorted(gt.keys, uk, 'right') - g0
    # records (q, a) in evalImgs order
    pos = ((uk // max(I, 1))[:, None] * A + np.arange(A)) * I + (uk % max(I, 1))[:, None]
    order = np.argsort(pos, axis=None)
    rq, ra = order // A, order % A
    R = len(order)
    off = lambda c: np.concatenate([[0], np.cumsum(c)]).astype(np.int64)
    dt_off, gt_off = off(Dk[rq]), off(Gq[rq])
    ann = np.concatenate([np.asarray(gt.ann_ids, np.int64), [0]])          # index num_gts: "no gt"
    sid = np.concatenate([o['slot_id'].astype(np.int64), [0]])               # index n_kept: "no detection"
    # detection rows: the record's kept slots, in rank order
    rec = np.repeat(np.arange(R), Dk[rq])
    slot = k0[rq][rec] + np.arange(len(rec)) - dt_off[rec]
    a_dt = ra[rec]
    m = o['dt_gt'].reshape(-1, A, T)[slot, a_dt]
    dt_matches = ann[np.where(m >= 0, g0[rq][rec][:, None] + m, len(ann) - 1)].astype(np.float64).T.copy()
    dt_ignore = o['dt_ig'].reshape(-1, A, T)[slot, a_dt].astype(bool).T.copy()
    # gt rows: each gt of each area range at its place in that range's order
    Gt = len(gt.keys)
    rec_of = np.empty(Q * A, np.int64)
    rec_of[order] = np.arange(R)
    qg = np.searchsorted(uk, gt.keys)
    dest = (gt_off[rec_of[qg[:, None] * A + np.arange(A)]] + o['gt_pos']).reshape(-1)
    src_g, src_a = np.empty(Gt * A, np.int64), np.empty(Gt * A, np.int64)
    src_g[dest], src_a[dest] = np.repeat(np.arange(Gt), A), np.tile(np.arange(A), Gt)
    r = o['gt_dt'].reshape(-1, A, T)[src_g, src_a]
    gt_matches = sid[np.where(r >= 0, k0[qg][src_g][:, None] + r, n_kept)].astype(np.float64).T.copy()
    return dict(index=pos.reshape(-1)[order], image_id=np.asarray(gt.img_ids, np.int64)[uk[rq] % max(I, 1)],
                category_id=np.asarray(gt.cat_ids, np.int64)[uk[rq] // max(I, 1)], area=ra, dt_off=dt_off, gt_off=gt_off,
                dtIds=o['slot_id'].astype(np.int64)[slot], dtScores=o['slot_score'][slot], dtMatches=dt_matches, dtIgnore=dt_ignore,
                gtIds=ann[src_g], gtIgnore=o['gt_ig'][src_g, src_a].astype(np.int64), gtMatches=gt_matches)


def _eval_imgs_list(params, c):
    """The columns of _eval_imgs_columns -> COCOeval.evalImgs, a list of K * 4 * I dicts or None.  The arrays of a record are views of
    the columns."""
    out = [None] * ((len(params.catIds) if params.useCats else 1) * len(params.areaRng) * len(params.imgIds))
    dt_off, gt_off = c['dt_off'].tolist(), c['gt_off'].tolist()
    dt_ids, dt_scores, gt_ids = c['dtIds'].tolist(), c['dtScores'].tolist(), c['gtIds'].tolist()
    dm, di, gm, gi = c['dtMatches'], c['dtIgnore'], c['gtMatches'], c['gtIgnore']
    max_det = params.maxDets[-1]
    for r, (n, img, cat, a) in enumerate(zip(c['index'].tolist(), c['image_id'].tolist(), c['category_id'].tolist(), c['area'].tolist())):
        d0, d1, g0, g1 = dt_off[r], dt_off[r + 1], gt_off[r], gt_off[r + 1]
        out[n] = {'image_id': img, 'category_id': cat, 'aRng': params.areaRng[a], 'maxDet': max_det, 'dtIds': dt_ids[d0:d1],
                  'gtIds': gt_ids[g0:g1], 'dtMatches': dm[:, d0:d1], 'gtMatches': gm[:, g0:g1], 'dtScores': dt_scores[d0:d1],
                  'gtIgnore': gi[g0:g1] if g1 > g0 else np.array([]), 'dtIgnore': di[:, d0:d1]}   # COCOeval's np.array([]) of no gts
    return out


# ------------------------------------------------------------------------------------------------------------ device-resident results
_INT32_MAX = 2 ** 31 - 1


def _pinned_upload(a, dev):
    """A small host table -> device, copied from pinned memory without synchronising the host."""
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)


class _Pending:
    """One masked add (or its redo) whose outcome the host has not read yet: the batch's own copies of its inputs, the records it
    wrote, and the status the device copies to pinned memory, [runs needed, size flag, arena full, cursor after, chars needed]."""

    def __init__(self, inputs, n0, num_classes):
        self.inputs, self.n0, self.num_classes = inputs, n0, num_classes
        self.runs_cap = self.capacity = self.status = self.event = None


class DeviceResults:
    """detect() outputs accumulated on the device, for evaluate(gt, acc, 'bbox' | 'segm') without bringing any detection to the host:

        acc = DeviceResults()
        for ...:
            out = model.detect(blob, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
            acc.add(out, image_ids, original_sizes=orig)     # json image id of each image of the batch
        E = evaluate(gt, acc, 'segm')

    The evaluation equals evaluate(gt, per_image_results, ...) where image i holds what batch_results returned for it (images never
    added have no detections).  add() only enqueues work on the current stream and does not synchronise the host: detect()'s buffers
    may be overwritten by the next call straight away.  With masks it pastes and encodes them as batch_results does, appending the
    strings to a device char arena at a device-side cursor (ops.segm_rle_batch_append).  Whether a batch's run lengths or strings
    overflowed is learnt later: each masked batch keeps a copy of its inputs (masks, boxes, scores, classes, counts, sizes: 2.5 MB for
    8 x 100 slots of 28 x 28) in a ring of _RING batches until its status, copied to pinned memory, has arrived.  A later add() reads
    the statuses that have (event query, no wait); an overflowed batch is redone with the grown buffer and its records rewritten, in
    stream order.  Only an add() that finds the ring full waits, for its oldest batch; evaluate() waits for all of them.
    Each add keeps B * cap records of 76 bytes (+ the strings).  evaluate() takes K * I bins (K categories, I images of the ground truth)
    of 84 bytes each: an int32 counter and 5 int64 values with their scans, 34 MB for 80 x 5000.  Device-side problems (classes not
    grouped or out of range, non-finite values) are raised by evaluate().  The category ids given to evaluate() must be distinct, so
    that each (category, image) bin holds one class's slots."""
    _MIN_RECORDS = 1 << 12          # initial capacities; both buffers then grow geometrically
    _MIN_CHARS = 1 << 20
    _RING = 4                       # masked batches whose status may be outstanding before add() waits for the oldest
    _RUNS_CAP = 4096                # initial run-length capacity per slot; grows when a slot needs more

    def __init__(self, device=None):
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if dev.type != 'cuda':
            raise ValueError("DeviceResults lives on a CUDA device, got %s" % dev)
        self.device = torch.device('cuda', torch.cuda.current_device() if dev.index is None else dev.index)
        self.image_ids = []                 # json id of each image ordinal, in the order added
        self._ordinal = {}
        self._where = []                    # per ordinal: (position in its detect() batch, num_classes of its add)
        self._num_records = 0
        self._chars_used = 0                # the arena cursor as of the last status read
        self._num_classes = 1
        self._all_masks = True
        self._rec_f = self._rec_i = self._chars = None
        self._runs_cap = self._RUNS_CAP
        self._ring = collections.deque()
        with torch.cuda.device(self.device):
            self._err = _pinned_upload(np.array([0, _INT32_MAX], np.int32), self.device)
            self._cursor = torch.zeros((1,), dtype=torch.int64, device=self.device)

    def __len__(self):
        return len(self.image_ids)

    @property
    def _num_chars(self):
        """Bytes of the char arena in use: exact, as it waits for every outstanding masked batch."""
        self._drain()
        return self._chars_used

    def _reserve(self, records):
        dev, n = self.device, self._num_records
        if self._rec_f is None or records > self._rec_f.shape[0]:
            cap = max(records, 2 * (0 if self._rec_f is None else self._rec_f.shape[0]), self._MIN_RECORDS)
            f = torch.empty((cap, 5), dtype=torch.float32, device=dev)
            i = torch.empty((cap, 7), dtype=torch.int64, device=dev)
            if n:
                f[:n].copy_(self._rec_f[:n]); i[:n].copy_(self._rec_i[:n])
            self._rec_f, self._rec_i = f, i

    def _launch(self, p):
        """Paste + RLE of a retained batch appended at the device cursor, its records (re)written with the arena offsets, and its
        status sent to pinned memory; nothing is waited for."""
        masks, boxes, scores, classes, counts, sizes, img_d = p.inputs
        B, cap = int(boxes.size(0)), int(boxes.size(1))
        L = _lib.lib()
        from .. import ops
        p.runs_cap, p.capacity = self._runs_cap, self._chars.shape[0]
        offs, flags = ops.segm_rle_batch_append(masks, None, boxes, counts, sizes, self._chars, self._cursor, runs_cap=p.runs_cap)
        _lib.check(L.dt_coco_results_append(B, cap, p.num_classes, _p(boxes), _p(scores), _p(classes), _p(counts), _p(img_d), _p(offs), 0,
                                            _p(self._rec_f[p.n0:]), _p(self._rec_i[p.n0:]), _p(self._err), _stream(self.device)),
                   "dt_coco_results_append")
        status = torch.cat([flags.to(torch.int64), self._cursor, offs[-1:] - offs[:1]])
        p.status = torch.empty((5,), dtype=torch.int64, pin_memory=True)
        p.status.copy_(status, non_blocking=True)
        p.event = torch.cuda.Event()
        p.event.record()
        self._ring.append(p)

    def _settle(self, p):
        """A masked batch whose status has arrived: done if no flag is raised, else the overflowed capacity grows and the batch is
        redone (in stream order, after everything enqueued so far)."""
        runs, size, full, cursor, need = p.status.tolist()
        self._chars_used = cursor
        if not (runs or size or full):
            return
        if size:
            raise RuntimeError("DeviceResults: an image size beyond the mask encoder's tables reached the device")
        with torch.cuda.device(self.device):
            if runs:
                self._runs_cap = max(self._runs_cap, 2 * p.runs_cap, runs + 1)
            if full and self._chars.shape[0] == p.capacity:
                # the batches enqueued since wrote below the old capacity, so the redo finds the cursor there at most; a batch that
                # failed before an earlier growth is redone first, and grows the arena only if it fails again
                old = self._chars.shape[0]
                c = torch.empty((max(2 * old, old + need, self._MIN_CHARS),), dtype=torch.uint8, device=self.device)
                c[:old].copy_(self._chars)
                self._chars = c
            self._launch(p)

    def _poll(self):
        """Settles the masked batches whose status has arrived, oldest first, without waiting."""
        while self._ring and self._ring[0].event.query():
            self._settle(self._ring.popleft())

    def _drain(self, keep=0):
        """Waits for the oldest masked batches until at most `keep` are outstanding (redoing any that overflowed)."""
        while len(self._ring) > keep:
            p = self._ring.popleft()
            p.event.synchronize()
            self._settle(p)

    def add(self, out, image_ids, original_sizes=None, num_classes=81):
        """Append one detect() output (boxes [B,cap,4], scores, classes, counts and optionally masks [B,cap,M,M]) for the images
        image_ids (one json id each, never added before).  original_sizes [B,2] (host): each image's RLE canvas, int() of each value as
        in batch_results; required with masks, and at most ops.SEGM_APPEND_MAX_SIDE on either side.  num_classes: the model's, classes
        must lie in 1..num_classes-1."""
        from .. import ops
        if not isinstance(out, dict) or any(k not in out for k in ('boxes', 'scores', 'classes', 'counts')):
            raise ValueError("add: expected detect()'s output dict with 'boxes', 'scores', 'classes' and 'counts'")
        boxes, scores, classes, counts, masks = out['boxes'], out['scores'], out['classes'], out['counts'], out.get('masks')
        tensors = [boxes, scores, classes, counts] + ([masks] if masks is not None else [])
        if not all(torch.is_tensor(t) and t.device == self.device for t in tensors):
            raise ValueError("add: detect() output must be tensors on %s" % self.device)
        if boxes.dim() != 3 or boxes.size(2) != 4:
            raise ValueError("add: boxes must be [B, cap, 4], got %s" % (tuple(boxes.shape),))
        B, cap = int(boxes.size(0)), int(boxes.size(1))
        if tuple(scores.shape) != (B, cap) or tuple(classes.shape) != (B, cap) or tuple(counts.shape) != (B,):
            raise ValueError("add: scores / classes must be [%d, %d] and counts [%d]" % (B, cap, B))
        if masks is not None and (masks.dim() != 4 or tuple(masks.shape[:2]) != (B, cap)):
            raise ValueError("add: masks must be [%d, %d, M, M] (the detected class's mask)" % (B, cap))
        num_classes = _int(num_classes, "num_classes")
        if num_classes < 1:
            raise ValueError("add: num_classes must be at least 1")
        if isinstance(image_ids, (str, bytes)) or torch.is_tensor(image_ids):
            raise ValueError("add: image_ids must be a sequence of integer json ids")
        ids = [_int(v, "image id") for v in image_ids]
        if len(ids) != B:
            raise ValueError("add: %d image ids for %d images" % (len(ids), B))
        if len(set(ids)) != B:
            raise ValueError("add: an image id is repeated in this batch")
        again = [v for v in ids if v in self._ordinal]
        if again:
            raise ValueError("add: image id %d was already added" % again[0])
        if masks is not None and original_sizes is None:
            raise ValueError("add: masks need original_sizes, each image's (height, width) RLE canvas")
        sizes = ops.segm_image_sizes(original_sizes, B) if original_sizes is not None else np.zeros((B, 2), np.int64)
        if masks is not None and B and sizes.max() > ops.SEGM_APPEND_MAX_SIDE:
            raise ValueError("add: an image of %d x %d is beyond the %d x %d the masks are encoded for" %
                             (tuple(sizes[int(np.argmax(sizes.max(1)))]) + (ops.SEGM_APPEND_MAX_SIDE,) * 2))
        o0, n0 = len(self.image_ids), self._num_records
        L = _lib.lib()
        with torch.cuda.device(self.device):
            self._poll()
            self._reserve(n0 + B * cap)
            table = np.concatenate([np.arange(o0, o0 + B, dtype=np.int64)[:, None], sizes.astype(np.int64)], 1)
            img_d = _pinned_upload(table, self.device)
            if masks is not None:
                self._drain(keep=self._RING - 1)
                if self._chars is None:
                    self._chars = torch.empty((max(self._MIN_CHARS, 1),), dtype=torch.uint8, device=self.device)
                own = lambda t, dt: t.to(dtype=dt, memory_format=torch.contiguous_format, copy=True)
                p = _Pending((own(masks, torch.float32), own(boxes, torch.float32), own(scores, torch.float32), own(classes, torch.int32),
                              own(counts, torch.int32), img_d[:, 1:].to(torch.int32).contiguous(), img_d), n0, num_classes)
                self._launch(p)
            else:
                bx, sc = boxes.contiguous().float(), scores.contiguous().float()
                cl, ct = classes.contiguous().to(torch.int32), counts.contiguous().to(torch.int32)
                _lib.check(L.dt_coco_results_append(B, cap, num_classes, _p(bx), _p(sc), _p(cl), _p(ct), _p(img_d), _p(None), 0,
                                                    _p(self._rec_f[n0:]), _p(self._rec_i[n0:]), _p(self._err), _stream(self.device)),
                           "dt_coco_results_append")
        for b, v in enumerate(ids):
            self._ordinal[v] = o0 + b
            self._where.append((b, num_classes))
        self.image_ids += ids
        self._num_records += B * cap
        self._num_classes = max(self._num_classes, num_classes)
        self._all_masks = self._all_masks and masks is not None


def _flatten_device(gt, acc, iou_type, category_ids, keep_eval_imgs=False, view=None):
    """_flatten_results + _pair_tables for a DeviceResults, on the device: -> dict of device tensors key [N], det_f [N, 5], det_i [N, 4]
    (char offsets into acc's buffer `chars`), pairs [P, 7], cat_kept [K + 1], order_off [3, K + 1], and the sizes dt_coco_eval takes.
    Host checks raise ValueError before anything is launched; the device's error flags come back with the sizes, in one copy.
    keep_eval_imgs adds det_ids [N] (loadRes ids, as with_ids of _flatten_results) and union [Q], the sorted keys of the pairs with
    detections or gts.  view: the _GtView of a Params (None: the default), whose images, categories and pairs the tables are over."""
    b = _bins_device(gt, acc, iou_type, category_ids, keep_eval_imgs, view)
    ev = gt if view is None else view
    per = 1 if view is None else view.per
    I, K, nb, dev = ev.num_images, ev.num_cats, ev.num_images * ev.num_cats, gt.device
    n, nc, rec_f, rec_i, cls_d, ord_d, scan = b['n'], b['nc'], b['rec_f'], b['rec_i'], b['cls_d'], b['ord_d'], b['scan']
    L = _lib.lib()
    with torch.cuda.device(dev):
        tail = b['tail'].cpu().numpy()
        if tail[5]:
            bo, ncls = acc._where[int(tail[6])]
            raise RuntimeError("batch_results: the detections of image %d are not grouped by class in 1..%d" % (bo, ncls - 1))
        if tail[7]:
            raise ValueError("non-finite box or score in the results")
        N, P, c10, n_kept, n_iou = (int(v) for v in tail[:5])
        key = torch.empty((max(N, 1),), dtype=torch.int64, device=dev)
        det_f = torch.empty((max(N, 1), 5), dtype=torch.float64, device=dev)
        det_i = torch.empty((max(N, 1), 4), dtype=torch.int64, device=dev)
        pairs = torch.empty((max(P, 1), 7), dtype=torch.int64, device=dev)
        cat_kept = torch.empty((K + 1,), dtype=torch.int64, device=dev)
        order_off = torch.empty((3, K + 1), dtype=torch.int64, device=dev)
        _lib.check(L.dt_coco_results_write(n, _p(rec_f), _p(rec_i), nc, _p(cls_d), _p(ord_d), I, K, per, _p(b['cnt']), _p(scan), _p(ev.keys_d),
                                           ev.num_gts, _p(key), _p(det_f), _p(det_i), _p(pairs), _p(cat_kept), _p(order_off), _stream(dev)),
                   "dt_coco_results_write")
        extra = {}
        if keep_eval_imgs:
            # row n of key k is file row file_start[k] + (n - first row of k); the union's keys are compacted by their scan
            Q = int(tail[8])
            if nb:
                k = key[:N]
                if view is None:
                    first = scan[0] - b['vals'][0]
                else:                           # rows are in fine bin order; key holds each row's fine bin
                    cnt = b['cnt'].to(torch.int64)
                    first = torch.cumsum(cnt, 0) - cnt
                extra['det_ids'] = torch.arange(N, device=dev) - first[k] + b['file_start'][k] + 1
                dst = torch.where(b['has'], b['union_scan'] - 1, nb)
                union = torch.empty((nb + 1,), dtype=torch.int64, device=dev)         # slot nb takes the bins left out
                extra['union'] = union.scatter_(0, dst, torch.arange(nb, device=dev))[:Q]
            else:
                extra['det_ids'] = extra['union'] = torch.zeros((0,), dtype=torch.int64, device=dev)
    chars = acc._chars if acc._chars is not None else torch.zeros((1,), dtype=torch.uint8, device=dev)
    return dict(key=key[:N], det_f=det_f[:N], det_i=det_i[:N], pairs=pairs[:P], cat_kept=cat_kept, order_off=order_off, chars=chars,
                num_chars=acc._num_chars, num_kept=n_kept, num_ious=n_iou, num_order=P + c10 + n_kept, **extra)


def _bins_device(gt, acc, iou_type, category_ids, keep_eval_imgs=False, view=None):
    """_flatten_device up to its one read-back, without a host synchronisation: the host checks, the counting pass and the bin scans;
    -> dict of the tables the write pass takes and `tail`, the device vector of sizes and flags to read back.  keep_eval_imgs adds
    each bin's first row in the results file (file_start: class-major, images in sorted-id order, the scan of the bins' counts in
    that order), the bins that have detections or gts (has) and their inclusive scan, whose total ends `tail`.  With a view, the bins
    are its fine bins (cnt), the scans over its pairs, and file_start is per fine bin, counted over every record of the results file."""
    if acc.device != gt.device:
        raise ValueError("the results are on %s, the ground truth on %s" % (acc.device, gt.device))
    if iou_type == 'segm' and not acc._all_masks:
        raise ValueError("segm evaluation of results without masks")
    if len(set(category_ids)) != len(category_ids):
        raise ValueError("category_ids must be distinct to evaluate a DeviceResults")
    img_index = {v: n for n, v in enumerate(gt.img_ids)}
    unknown = [v for v in acc.image_ids if v not in img_index]
    if unknown:
        raise ValueError("image id %d was added to the results but is not an image of the ground truth" % unknown[0])
    ord_i = np.array([img_index[v] for v in acc.image_ids] or [0], np.int32)
    cat_index = {v: n for n, v in enumerate(gt.cat_ids)}
    nc = acc._num_classes
    cls_k = np.full(nc, -1, np.int32)
    for j in range(1, min(len(category_ids) + 1, nc)):        # classes past category_ids are dropped, as the host loop's break drops them
        cls_k[j] = cat_index[category_ids[j - 1]]
    ev, per = (gt, 1) if view is None else (view, view.per)
    if view is not None:                # the maps of the view: category slot of each class, image index of each ordinal (-1: left out)
        cls_v = np.where(cls_k >= 0, view.cat_slot[np.maximum(cls_k, 0)], -1).astype(np.int32)
        ord_v = view.img_slot[ord_i].astype(np.int32) if acc.image_ids else ord_i
    I, K = ev.num_images, ev.num_cats
    nb, n, dev = I * K, acc._num_records, gt.device
    acc._drain()                        # every masked batch settled (and redone if it overflowed) before its records are read
    L = _lib.lib()
    rec_f, rec_i = (acc._rec_f, acc._rec_i) if n else (None, None)
    out = dict(n=n, nc=nc, rec_f=rec_f, rec_i=rec_i)
    with torch.cuda.device(dev):
        cls_d, ord_d = _pinned_upload(cls_k, dev), _pinned_upload(ord_i, dev)
        nonfinite = torch.zeros((1,), dtype=torch.int32, device=dev)
        if view is not None:
            full = (cls_d, ord_d)
            cls_d, ord_d = _pinned_upload(cls_v, dev), _pinned_upload(ord_v, dev)
        cnt = torch.zeros((nb * per,), dtype=torch.int32, device=dev) if nb else None
        vals = torch.empty((5, nb), dtype=torch.int64, device=dev) if nb else None
        _lib.check(L.dt_coco_results_count(n, _p(rec_f), _p(rec_i), nc, _p(cls_d), _p(ord_d), I, K, per, _p(ev.keys_d), ev.num_gts, _p(cnt),
                                           _p(vals), _p(nonfinite), _stream(dev)), "dt_coco_results_count")
        scan = torch.cumsum(vals, 1) if nb else None
        totals = scan[:, -1] if nb else torch.zeros((5,), dtype=torch.int64, device=dev)
        parts = [totals, acc._err.to(torch.int64), nonfinite.to(torch.int64)]
        if keep_eval_imgs and nb:
            # the results file's order of the bins: class j = 1, 2, .. (its category's bins, images in sorted-id order)
            K0, I0 = gt.num_cats, gt.num_images
            cats = cls_k[1:][cls_k[1:] >= 0].astype(np.int64)
            cats_d = _pinned_upload(cats, dev)
            if view is None:
                counts = vals[0].view(K, I).index_select(0, cats_d)
            else:                   # the file holds every record: its bins are counted over all of gt's images and categories
                cnt0 = torch.zeros((K0 * I0,), dtype=torch.int32, device=dev)
                vals0 = torch.empty((5, K0 * I0), dtype=torch.int64, device=dev)
                _lib.check(L.dt_coco_results_count(n, _p(rec_f), _p(rec_i), nc, _p(full[0]), _p(full[1]), I0, K0, 1, _p(gt.keys_d), gt.num_gts,
                                                   _p(cnt0), _p(vals0), _p(torch.zeros_like(nonfinite)), _stream(dev)), "dt_coco_results_count")
                counts = cnt0.to(torch.int64).view(K0, I0).index_select(0, cats_d)
            in_file = torch.cumsum(counts.reshape(-1), 0).view(len(cats), I0) - counts
            file_start = torch.zeros((K0, I0), dtype=torch.int64, device=dev).index_copy_(0, cats_d, in_file).view(-1)
            if view is not None:    # each fine bin's (category, image) of gt
                ks, ims = np.flatnonzero(view.cat_slot >= 0), np.flatnonzero(view.img_slot >= 0)
                kk, ii = np.meshgrid(ks, ims, indexing='ij')
                fine = view.fine_key(view.cat_slot[kk], view.img_slot[ii]).reshape(-1)
                src = np.empty(nb * per, np.int64)
                src[fine] = (kk * I0 + ii).reshape(-1)
                file_start = file_start.index_select(0, _pinned_upload(src, dev))
            has = vals[1] > 0
            if ev.num_gts:
                has.index_fill_(0, ev.keys_d, True)
            union_scan = torch.cumsum(has, 0)
            out.update(vals=vals, file_start=file_start, has=has, union_scan=union_scan)
            parts.append(union_scan[-1:])
        elif keep_eval_imgs:
            parts.append(torch.zeros((1,), dtype=torch.int64, device=dev))
        out.update(cls_d=cls_d, ord_d=ord_d, scan=scan, cnt=cnt, tail=torch.cat(parts))
    return out


# ------------------------------------------------------------------------------------------------------------ results json
_JSON_CHUNK = 64 << 20          # bytes per pinned staging buffer (two of them) between the device text and the file


def _counts_first(all_segms, all_boxes, category_ids, num_images):
    """The RLE dicts in file order (the loop of _flatten_results) -> uint8 [rows], 1 where 'counts' comes before 'size'.  A dict with
    a key other than these two, or 'counts' that is not a str (json.dump writes no bytes), is refused."""
    flags = []
    for j in range(1, len(category_ids) + 1):
        if j >= len(all_boxes):
            break
        for i in range(num_images):
            d = all_boxes[j][i]
            if isinstance(d, list) and len(d) == 0:
                continue
            for r in all_segms[j][i][:np.asarray(d).shape[0]]:
                if set(r) != {'size', 'counts'}:
                    raise ValueError("class %d image %d: an RLE dict must have exactly the keys 'size' and 'counts'" % (j, i))
                if not isinstance(r['counts'], str):
                    raise ValueError("class %d image %d: RLE 'counts' must be a str to be written to json" % (j, i))
                flags.append(next(iter(r)) == 'counts')
    return np.array(flags, np.uint8)


def write_results(gt, results, iou_type, path, all_segms=None, category_ids=None):
    """The COCO results json of `results` ('bbox' or 'segm') written to `path` -> bytes written.  The file holds the bytes the
    reference's _write_coco_bbox_results_file / _write_coco_segms_results_file + json.dump write: records class-major (j = 1, 2, ..),
    images in sorted-id order, each (class, image)'s detections in their order; bbox [x1, y1, x2 - x1 + 1, y2 - y1 + 1] and the score
    as float64, printed as float.__repr__ prints them; an RLE dict in its own key order.
    results, all_segms and category_ids as for evaluate(): per-image tuples, all_boxes [class][image] (+ all_segms), or a
    DeviceResults.  gt only supplies the sorted image ids and the categories: one without annotations (a test-dev image-info file)
    will do, for either iou_type.
    Unlike the reference, a non-finite box or score raises ValueError (json.dump would write NaN / Infinity, which is not json).
    Input evaluate() refuses is refused here, before anything is written: no file is created and an existing one is left as it
    was (the text goes to a temporary file in the same directory, renamed over `path` once complete).
    The records are formatted on the device (csrc/coco_json.cuh): a length pass, a scan, a write pass; the text reaches the file
    through two pinned buffers of 64 MB."""
    if iou_type not in ('bbox', 'segm'):
        raise ValueError("iou_type must be 'bbox' or 'segm'")
    if not isinstance(gt, CocoGroundTruth):
        raise TypeError("gt must be a CocoGroundTruth")
    category_ids = list(gt.category_ids if category_ids is None else category_ids)
    if any(c not in set(gt.cat_ids) for c in category_ids):
        raise ValueError("category_ids names a category the ground truth does not have")
    segm, dev, first = iou_type == 'segm', gt.device, None
    if isinstance(results, DeviceResults):
        if all_segms is not None:
            raise ValueError("a DeviceResults carries its masks; all_segms is for all_boxes input")
        f = _flatten_device(gt, results, iou_type, category_ids, keep_eval_imgs=True)
        key, det_f, det_i, chars, pos = f['key'], f['det_f'], f['det_i'], f['chars'], f['det_ids'] - 1
    else:
        boxes, segms = _per_class(gt, results, all_segms, iou_type)
        key, det_f, det_i, chars, det_ids = _flatten_results(gt, boxes, segms, iou_type, category_ids, with_ids=True)
        if segm and len(key):
            first = _counts_first(segms, boxes, category_ids, gt.num_images)
        key, det_f, det_i, pos = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (key, det_f, det_i, det_ids - 1))
        chars = torch.from_numpy(np.frombuffer(chars or b"\0", np.uint8).copy()).to(dev)
        first = torch.from_numpy(first).to(dev) if first is not None and first.any() else None
    N = int(key.shape[0])
    text = np.frombuffer(b"[]", np.uint8)
    L = _lib.lib()
    with torch.cuda.device(dev):
        if N:
            ids = [torch.tensor(v, dtype=torch.int64, device=dev) for v in (gt.img_ids, gt.cat_ids)]
            args = (1 if segm else 0, N, _p(det_f), _p(key), _p(pos), gt.num_images, _p(ids[0]), _p(ids[1]), _p(det_i), _p(chars), _p(first))
            lens = torch.empty((N,), dtype=torch.int64, device=dev)
            _lib.check(L.dt_coco_json(*args, None, _p(lens), None, _stream(dev)), "dt_coco_json")
            lens.cumsum_(0)
            tail = [lens[-1:]]
            if segm:
                # as evaluate() refuses them: runs that do not cover h * w pixels
                bad = torch.empty((N,), dtype=torch.uint8, device=dev)
                _lib.check(L.dt_coco_det_check(N, _p(det_i), _p(chars), _p(bad), _stream(dev)), "dt_coco_det_check")
                tail.append(bad.any().view(1).to(torch.int64))
            tail = torch.cat(tail).cpu().numpy()            # the one read-back: the file's size, and the RLE check
            if segm and tail[1]:
                raise ValueError("results: RLE counts of a result do not sum to h * w")
            text = torch.empty((int(tail[0]),), dtype=torch.uint8, device=dev)
            _lib.check(L.dt_coco_json(*args, _p(lens), None, _p(text), _stream(dev)), "dt_coco_json")
        return _write_text(text, path)


def _write_text(text, path):
    """Device bytes (or a host array) -> path, through a temporary file renamed over it; the device text in chunks through two
    pinned buffers, the copy of the next chunk under the write of this one."""
    import os
    import tempfile
    total = int(text.shape[0])
    fd, tmp = tempfile.mkstemp(prefix=".%s." % os.path.basename(path), suffix=".tmp", dir=os.path.dirname(os.path.abspath(path)))
    try:
        with os.fdopen(fd, "wb") as fh:
            if isinstance(text, np.ndarray):
                fh.write(text.tobytes())
            else:
                stage = [torch.empty((min(total, _JSON_CHUNK),), dtype=torch.uint8, pin_memory=True) for _ in range(1 + (total > _JSON_CHUNK))]
                spans = [(o, min(o + _JSON_CHUNK, total)) for o in range(0, total, _JSON_CHUNK)]
                events = []

                def copy(c):
                    a, b = spans[c]
                    stage[c % 2][:b - a].copy_(text[a:b], non_blocking=True)
                    events.append(torch.cuda.Event())
                    events[-1].record()
                copy(0)
                for c, (a, b) in enumerate(spans):
                    if c + 1 < len(spans):
                        copy(c + 1)             # its buffer's previous chunk is already in the file
                    events[c].synchronize()
                    fh.write(memoryview(stage[c % 2].numpy())[:b - a])
        os.chmod(tmp, 0o666 & ~_umask())
        os.replace(tmp, path)
    except BaseException:
        os.unlink(tmp)
        raise
    return total


def _umask():
    import os
    m = os.umask(0)
    os.umask(m)
    return m


# ------------------------------------------------------------------------------------------------------------ reading a results file
# error bits of csrc/coco_results_file.cuh, in the order they are reported
_FILE_ERRORS = [(1 << 1, "a byte >= 0x80 (a json.dump file is ASCII)"), (1 << 0, "not valid JSON"),
                (1 << 2, "the top level is not one JSON array"), (1 << 3, "an element of the array is not an object"),
                (1 << 4, "values nested deeper than 64 levels"), (1 << 5, "a score or bbox number that is not finite as a double"),
                (1 << 6, "'image_id' missing or not an integer literal in int64"),
                (1 << 7, "an image_id that is not an image of the ground truth (loadRes asserts)"),
                (1 << 8, "'category_id' missing or not an integer literal in int64"), (1 << 9, "'score' missing or not a number"),
                (1 << 10, "a segmentation dict that is not a compressed RLE (string 'counts', 'size' [h, w] integers, 1 <= h w < 2^32)"),
                (1 << 11, "RLE counts with a character outside '0'..'o', a value longer than 6 characters, or ending inside a value"),
                (1 << 12, "RLE counts that do not sum to h * w")]
_NO_BBOX, _BAD_BBOX, _NO_RLE = 1, 2, 4
_HAS_BBOX, _BBOX_EMPTY, _HAS_CAPTION = 1, 4, 16
_INFO = 8


class LoadedResults:
    """A COCO results file as pycocotools' COCO.loadRes(file) hands it to COCOeval, held on the device (load_results).
        branch          'bbox' or 'segm': loadRes's branch, decided by the first record ('bbox' when it has a bbox that is not [])
        num_records     records in the file;  num_dropped: those of categories the ground truth does not have (COCOeval never
                        selects them)
    The detections of the other records are kept in dt_coco_eval's layout, sorted by (category, image), file order inside a pair;
    their loadRes ids are 1 + their index in the file and their 'area' is loadRes's (bbox branch: w h; segm branch: the RLE area).
    evaluate(gt, loaded, 'bbox' | 'segm', ...) takes it any number of times, for either iou type."""

    def __init__(self, gt, branch, num_records, num_dropped, key, det_f, det_i, det_area, det_ids, chars, num_chars, summary):
        self.gt, self.branch, self.num_records, self.num_dropped = gt, branch, num_records, num_dropped
        self._key, self._det_f, self._det_i, self._det_area, self._det_ids = key, det_f, det_i, det_area, det_ids
        self._chars, self._num_chars, self._summary = chars, num_chars, summary

    def __len__(self):
        return len(self._key)


def _read_text(source, dev):
    """A path or a bytes-like object -> its bytes on the device, read into two pinned buffers of 64 MB and copied in chunks (the
    read of the next chunk under the copy of this one)."""
    import os
    if isinstance(source, (str, os.PathLike)):
        fh = open(source, "rb")
        total = os.fstat(fh.fileno()).st_size
    else:
        try:
            view = memoryview(source).cast("B")
        except TypeError:
            raise ValueError("load_results: source must be a path or a bytes-like object") from None
        fh, total = None, view.nbytes
    try:
        text = torch.empty((max(total, 1),), dtype=torch.uint8, device=dev)
        if total:
            stage = [torch.empty((min(total, _JSON_CHUNK),), dtype=torch.uint8, pin_memory=True) for _ in range(1 + (total > _JSON_CHUNK))]
            events = [None, None]
            for c, a in enumerate(range(0, total, _JSON_CHUNK)):
                b = min(a + _JSON_CHUNK, total)
                if events[c % 2] is not None:
                    events[c % 2].synchronize()         # the buffer's previous chunk has reached the device
                buf = stage[c % 2].numpy()[:b - a]
                if fh is None:
                    buf[:] = np.frombuffer(view[a:b], np.uint8)
                elif fh.readinto(memoryview(buf)) != b - a:
                    raise ValueError("load_results: the file changed size while it was read")
                text[a:b].copy_(stage[c % 2][:b - a], non_blocking=True)
                events[c % 2] = torch.cuda.Event()
                events[c % 2].record()
            for e in events:
                if e is not None:
                    e.synchronize()
    finally:
        if fh is not None:
            fh.close()
    return text, total


def _file_error(info, what):
    err = int(info[1])
    for bit, msg in _FILE_ERRORS:
        if err & bit:
            at = "" if info[4] == np.iinfo(np.int64).max else " (record %d)" % info[4]
            raise ValueError("%s: %s%s" % (what, msg, at))


def load_results(gt, source):
    """COCO.loadRes(source) on the device -> LoadedResults for evaluate(gt, loaded, 'bbox' | 'segm').  source: the path of a COCO
    results json (a list of {"image_id", "category_id", "score", "bbox" and / or "segmentation"} records, as the reference's results
    writers, detectron2 or mmdetection write them) or a bytes-like object holding one.  The file is copied to the device once and
    parsed there (csrc/coco_results_file.cuh): numbers become the doubles json.loads gives, the last occurrence of a key wins, keys
    loadRes does not read are skipped.  Records of categories gt does not have are kept out (COCOeval never selects them).
    Raises ValueError, before anything is evaluated, for text json.loads rejects and for NaN / Infinity and non-ASCII bytes (json.dump
    writes neither), a top level that is not an array of objects, an image_id or category_id that is not an integer literal in int64
    or an image_id that is not an image of gt (loadRes asserts), a missing or non-numeric score, a number that is not finite as a
    double, a bbox that is not 4 numbers in the bbox branch, a record without a compressed RLE in the segm branch, a segmentation dict
    that is not a valid compressed RLE (its counts are checked as list input's are), nesting deeper than 64 levels, and a first record
    with a 'caption' (loadRes's caption branch).
    Unlike loadRes, which raises IndexError on it, an empty array [] gives results with no detections."""
    if not isinstance(gt, CocoGroundTruth):
        raise TypeError("gt must be a CocoGroundTruth")
    dev, what = gt.device, "results file"
    L = _lib.lib()
    with torch.cuda.device(dev):
        text, n = _read_text(source, dev)
        if n == 0:
            raise ValueError("%s: empty (not valid JSON)" % what)
        st = _stream(dev)
        info = torch.zeros((_INFO,), dtype=torch.int64, device=dev)
        info[4] = np.iinfo(np.int64).max
        ws = torch.empty((L.dt_coco_file_struct_workspace_bytes(n),), dtype=torch.uint8, device=dev)
        _lib.check(L.dt_coco_file_struct(n, _p(text), _p(ws), _p(info), st), "dt_coco_file_struct")
        h = info.cpu().numpy()
        _file_error(h, what)
        if h[5] != 1 or h[0] < 2:
            raise ValueError("%s: the top level is not one JSON array" % what)
        sep = torch.empty((int(h[0]),), dtype=torch.int64, device=dev)
        _lib.check(L.dt_coco_file_separators(n, _p(ws), _p(sep), st), "dt_coco_file_separators")
        R = int(h[0]) - 1
        img_d = torch.tensor(gt.img_ids or [0], dtype=torch.int64, device=dev)
        cat_d = torch.tensor(gt.cat_ids or [0], dtype=torch.int64, device=dev)
        rec_f = torch.empty((R, 5), dtype=torch.float64, device=dev)
        rec_open = torch.empty((R, 5), dtype=torch.int64, device=dev)
        rec_i = torch.empty((R, 6), dtype=torch.int64, device=dev)
        rec_n = torch.empty((R,), dtype=torch.int64, device=dev)
        rec_b = torch.empty((R,), dtype=torch.uint8, device=dev)
        _lib.check(L.dt_coco_file_records(R, n, _p(text), _p(sep), gt.num_images, _p(img_d), gt.num_cats, _p(cat_d), _p(rec_f), _p(rec_open),
                                          _p(rec_i), _p(rec_n), _p(rec_b), _p(info), st), "dt_coco_file_records")
        del ws
        offs = torch.cumsum(rec_n, 0)
        h = torch.cat([info, offs[-1:], rec_b[:1].to(torch.int64)]).cpu().numpy()
        _file_error(h, what)
        empty = bool(h[6])
        num_chars, first = int(h[_INFO]), int(h[_INFO + 1])
        if empty:
            z = torch.zeros
            return LoadedResults(gt, 'bbox', 0, 0, np.zeros(0, np.int64), z((0, 5), dtype=torch.float64, device=dev),
                                 z((0, 4), dtype=torch.int64, device=dev), z((0,), dtype=torch.float64, device=dev),
                                 z((0,), dtype=torch.int64, device=dev), z((1,), dtype=torch.uint8, device=dev), 0, 0)
        if first & _HAS_CAPTION:
            raise ValueError("%s: the first record has a 'caption' (loadRes's caption branch is not evaluated here)" % what)
        branch = 'bbox' if (first & _HAS_BBOX) and not (first & _BBOX_EMPTY) else 'segm'
        summary = int(h[2])
        if branch == 'bbox' and summary & _NO_BBOX:
            raise ValueError("%s: a record without a bbox of 4 numbers (the first record's bbox makes every record's bbox read)" % what)
        if branch == 'segm' and summary & _NO_RLE:
            raise ValueError("%s: a record without a compressed RLE segmentation (the first record has no bbox: loadRes reads every "
                             "record's RLE)" % what)
        N = R - int(h[3])
        chars = torch.empty((num_chars + 1,), dtype=torch.uint8, device=dev)
        ws = torch.empty((L.dt_coco_file_finish_workspace_bytes(R, num_chars, int(branch == 'segm')),), dtype=torch.uint8, device=dev)
        det_key = torch.empty((R,), dtype=torch.int64, device=dev)
        det_f = torch.empty((N, 5), dtype=torch.float64, device=dev)
        det_i = torch.empty((N, 4), dtype=torch.int64, device=dev)
        det_area = torch.empty((N,), dtype=torch.float64, device=dev)
        det_ids = torch.empty((N,), dtype=torch.int64, device=dev)
        _lib.check(L.dt_coco_file_finish(R, int(branch == 'segm'), _p(text), _p(rec_i), _p(rec_n), _p(offs), _p(rec_b), _p(rec_f), gt.num_images,
                                         gt.num_cats, num_chars, _p(chars), _p(ws), N, _p(det_key), _p(det_f), _p(det_i), _p(det_area),
                                         _p(det_ids), _p(info), st), "dt_coco_file_finish")
        _file_error(info.cpu().numpy(), what)
        key = det_key[:N].cpu().numpy()
    return LoadedResults(gt, branch, R, R - N, key, det_f, det_i, det_area, det_ids, chars, num_chars, summary)


def _evaluate_loaded(gt, res, iou_type, keep_ious, keep_eval_imgs, p):
    """evaluate() of a LoadedResults: its tables, re-keyed for a Params view, with loadRes's areas."""
    if res.gt is not gt:
        raise ValueError("the results were loaded for another ground truth")
    if iou_type == 'segm' and res._summary & _NO_RLE:
        raise ValueError("segm evaluation of a results file with records without a compressed RLE (loadRes would make a polygon "
                         "of their box; not supported)")
    if iou_type == 'bbox' and res._summary & _BAD_BBOX:
        raise ValueError("bbox evaluation of a results file with a bbox that is not 4 numbers")
    view = None if _is_default(gt, p) else _GtView(gt, p)
    ev = gt if view is None else view
    key, det_f, det_i, det_area, det_ids = res._key, res._det_f, res._det_i, res._det_area, res._det_ids
    dev = gt.device
    if view is not None:
        rows, fine = view.select(key)
        rows_d = torch.from_numpy(rows).to(dev)
        key = fine // view.per
        det_f, det_i, det_area, det_ids = (x.index_select(0, rows_d) for x in (det_f, det_i, det_area, det_ids))
    pairs, cat_kept, order_off = _pair_tables(ev, key)
    kept, gn = np.minimum(pairs[:, 2], MAX_DETS[-1]), pairs[:, 4]
    n_kept, n_iou, n_order = int(kept.sum()), int((kept * gn).sum()), int(order_off[-1, -1])
    up = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (pairs, cat_kept, order_off)]
    imgs = None
    if keep_eval_imgs:
        imgs = (torch.from_numpy(np.union1d(pairs[:, 0], ev.keys).astype(np.int64)).to(dev), det_ids)
    return _evaluate_tables(ev, iou_type, pairs, *up, det_f.contiguous(), det_i.contiguous(), res._chars, res._num_chars, n_kept, n_iou,
                            n_order, keep_ious, imgs, p, det_area.contiguous())


# ------------------------------------------------------------------------------------------------------------ proposal recall
# evaluate_box_proposals' area ranges (json_dataset_evaluator.py:247-264), both bounds inclusive
PROPOSAL_AREAS = {'all': [0 ** 2, 1e5 ** 2], 'small': [0 ** 2, 32 ** 2], 'medium': [32 ** 2, 96 ** 2], 'large': [96 ** 2, 1e5 ** 2],
                  '96-128': [96 ** 2, 128 ** 2], '128-256': [128 ** 2, 256 ** 2], '256-512': [256 ** 2, 512 ** 2], '512-inf': [512 ** 2, 1e5 ** 2]}
_BOX_COORD_MAX = 1e15            # |coordinate| bound that keeps every float32 area and union of bbox_overlaps finite
_AREA_DTYPES = (np.float32, np.float64, np.int32, np.int64)


def _entry_arrays(n, e):
    what = "roidb entry %d" % n
    if not isinstance(e, dict) or any(k not in e for k in ('boxes', 'gt_classes', 'is_crowd', 'seg_areas')):
        raise ValueError("%s: needs 'boxes', 'gt_classes', 'is_crowd' and 'seg_areas'" % what)
    boxes, cls, crowd, areas = (np.asarray(e[k]) for k in ('boxes', 'gt_classes', 'is_crowd', 'seg_areas'))
    if boxes.ndim != 2 or boxes.shape[1] != 4 or not (np.issubdtype(boxes.dtype, np.floating) or np.issubdtype(boxes.dtype, np.integer)):
        raise ValueError("%s: boxes must be a numeric [n, 4] array" % what)
    r = boxes.shape[0]
    if cls.shape != (r,) or not np.issubdtype(cls.dtype, np.integer):
        raise ValueError("%s: gt_classes must be an integer array of one value per box" % what)
    if crowd.shape != (r,) or not (crowd.dtype == np.bool_ or np.issubdtype(crowd.dtype, np.integer)):
        raise ValueError("%s: is_crowd must be a bool or integer array of one value per box" % what)
    if areas.shape != (r,) or areas.dtype.type not in _AREA_DTYPES:
        raise ValueError("%s: seg_areas must be a float32 / float64 / int32 / int64 array of one value per box" % what)
    return boxes, cls, crowd, areas


def _proposal_tables(roidb):
    """roidb -> (prop_off, props, gt_off, gts, gt_area): per image its proposals (gt_classes == 0 rows, in order) and its ground truth
    (gt_classes > 0, not crowd), boxes as float32 as bbox_overlaps is given them.  Malformed entries raise ValueError."""
    props, gts, areas = [], [], []
    np_i, ng_i = np.zeros(len(roidb), np.int64), np.zeros(len(roidb), np.int64)
    for n, e in enumerate(roidb):
        boxes, cls, crowd, area = _entry_arrays(n, e)
        g = (cls > 0) & (crowd == 0)
        p = cls == 0
        b = boxes.astype(np.float32, copy=False)
        props.append(b[p]); gts.append(b[g]); areas.append(area[g].astype(np.float64))
        np_i[n], ng_i[n] = props[-1].shape[0], gts[-1].shape[0]
    props = np.ascontiguousarray(np.concatenate(props) if props else np.zeros((0, 4), np.float32), np.float32)
    gts = np.ascontiguousarray(np.concatenate(gts) if gts else np.zeros((0, 4), np.float32), np.float32)
    gt_area = np.concatenate(areas) if areas else np.zeros(0)
    for what, b in (("proposal", props), ("ground-truth", gts)):
        if b.size and not (np.all(np.isfinite(b)) and np.abs(b).max() <= _BOX_COORD_MAX):
            raise ValueError("roidb: a %s box is not finite or has a coordinate beyond %g" % (what, _BOX_COORD_MAX))
    off = lambda c: np.concatenate([[0], np.cumsum(c)]).astype(np.int64)
    return off(np_i), props, off(ng_i), gts, gt_area


def _limit(v):
    if v is None:
        return -1
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < 0:
        raise ValueError("proposal limit must be None or a non-negative integer, got %r" % (v,))
    return int(v)


def box_proposal_recall(roidb, areas=('all', 'small', 'medium', 'large'), limits=(100, 1000), thresholds=None, device=None):
    """Detectron's evaluate_box_proposals(json_dataset, roidb, thresholds, area, limit) for every (area, limit) combination at once
    -> {(area, limit): {'ar', 'recalls', 'thresholds', 'gt_overlaps', 'num_pos'}}, each dict equal to what the reference returns.
    roidb: entries with 'boxes' (ground truth then proposals), 'gt_classes' (0 for a proposal), 'is_crowd' and 'seg_areas', as
    JsonDataset.get_roidb(gt=True, proposal_file=...) builds them.  The greedy matching of every (image, combination) runs in one
    CUDA launch; the host sorts the overlaps and counts them against the thresholds as the reference does."""
    areas, limits = list(areas), list(limits)
    for a in areas:
        if a not in PROPOSAL_AREAS:
            raise ValueError("Unknown area range: {}".format(a))
    combos = [(a, l) for a in areas for l in limits]
    lims = np.array([_limit(l) for _, l in combos], np.int64)
    rng = np.array([PROPOSAL_AREAS[a] for a, _ in combos], np.float64).reshape(-1, 2)
    prop_off, props, gt_off, gts, gt_area = _proposal_tables(roidb)
    I, C = len(prop_off) - 1, len(combos)
    np_i, ng_i = np.diff(prop_off), np.diff(gt_off)
    img_of_gt = np.repeat(np.arange(I), ng_i)
    # GTs inside each range per image (the kernel selects the same ones), outputs only for images with proposals
    sel = np.zeros((C, I), np.int64)
    for c in range(C):
        m = (gt_area >= rng[c, 0]) & (gt_area <= rng[c, 1])
        sel[c] = np.bincount(img_of_gt[m], minlength=I)
    outlen = np.where(np_i[None, :] > 0, sel, 0)
    out_off = np.concatenate([[0], np.cumsum(outlen.reshape(-1))]).astype(np.int64)
    total = int(out_off[-1])
    max_gts = int(ng_i.max()) if I else 0
    max_props = int(np_i.max()) if I else 0
    L = _lib.lib()
    smem = L.dt_proposal_recall_smem_bytes(max_gts, max_props)
    if smem == 0 or smem > 227 * 1024:
        raise ValueError("box_proposal_recall: %d ground-truth boxes and %d proposals in one image do not fit one CTA's shared memory" %
                         (max_gts, max_props))
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    ov = np.zeros(0)
    if total and I:
        up = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (prop_off, props.reshape(-1) if props.size else np.zeros(4, np.float32),
                                                                           gt_off, gts.reshape(-1), gt_area, rng.reshape(-1), lims, out_off[:-1])]
        out = torch.empty((total,), dtype=torch.float64, device=dev)
        flag = torch.zeros((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.dt_proposal_recall(I, C, _p(up[0]), _p(up[1]), _p(up[2]), _p(up[3]), _p(up[4]), _p(up[5]), _p(up[6]), _p(up[7]),
                                            max_gts, max_props, _p(out), _p(flag), _stream(dev)), "dt_proposal_recall")
        f = int(flag.item())
        if f & 2:
            raise ValueError("roidb: a proposal and a ground-truth box whose union is 0 (bbox_overlaps divides by zero)")
        if f & 1:
            raise ValueError("roidb: a recorded overlap below 0 (the reference asserts gt_ovr >= 0)")
        ov = out.cpu().numpy()
    res = {}
    for c, key in enumerate(combos):
        gt_overlaps = np.sort(ov[out_off[c * I]:out_off[(c + 1) * I]])
        res[key] = _recall_summary(gt_overlaps, int(sel[c].sum()), thresholds)
    return res


def _recall_summary(gt_overlaps, num_pos, thresholds):
    """json_dataset_evaluator.py:308-319 on the sorted overlaps."""
    if thresholds is None:
        step = 0.05
        thresholds = np.arange(0.5, 0.95 + 1e-5, step)
    recalls = np.zeros_like(thresholds)
    # compute recall for each iou threshold
    for i, t in enumerate(thresholds):
        recalls[i] = (gt_overlaps >= t).sum() / float(num_pos)
    ar = recalls.mean()
    return {'ar': ar, 'recalls': recalls, 'thresholds': thresholds, 'gt_overlaps': gt_overlaps, 'num_pos': num_pos}

"""Synthetic COCO ground truth and detection results for the device evaluation (detectorch_b200.utils.coco_eval), and the oracle
run on them: the notebooks' results-file conversion (lib/utils/json_dataset_evaluator.py) + the reference's own pycocotools
COCOeval, built by oracle/build_cocoapi.sh.

The case covers what COCOeval treats specially: multi-part, concave, sub-pixel and border-touching polygons with .5 coordinates, a
polygon with a repeated vertex, crowd GTs as uncompressed RLE, a compressed-RLE GT, images without GT or without detections, absent categories,
a pair with more than 100 detections, equal scores across images, GT areas of exactly 32^2 and 96^2, and boxes whose IoU with a GT
is exactly 0.5 or 0.75."""
import contextlib
import copy
import io
import json

import numpy as np


def _poly_rect(x, y, w, h):
    return [x, y, x + w, y, x + w, y + h, x, y + h]


def make_case(seed=0, num_images=12, with_masks=True, encode=None):
    """-> (annotation dict, all_boxes [class][image], all_segms [class][image] or None).  encode(mask uint8 [h, w]) -> RLE string
    (pycocotools mask.encode); needed for the detection masks when with_masks."""
    rng = np.random.RandomState(seed)
    cat_ids = [3, 7, 1, 12, 9, 20]            # dataset order != sorted order; 20 is absent (no GT, no detections)
    images = []
    for i in range(num_images):
        h, w = int(rng.randint(40, 120)), int(rng.randint(40, 140))
        images.append(dict(id=int(100 + 7 * ((i * 5) % num_images)), height=h, width=w))   # ids not in list order
    img_ids = sorted(im['id'] for im in images)
    hw = {im['id']: (im['height'], im['width']) for im in images}
    anns = []
    aid = [1]

    def add(img, cat, seg, bbox, area, crowd=0):
        anns.append(dict(id=aid[0], image_id=img, category_id=cat, segmentation=seg, bbox=[float(v) for v in bbox], area=area, iscrowd=crowd))
        aid[0] += 1

    for n, img in enumerate(img_ids):
        h, w = hw[img]
        if n == 1:
            continue                          # an image without GT
        for g in range(int(rng.randint(2, 8))):
            cat = int(rng.choice([3, 7, 1, 12]))
            x, y = rng.uniform(-3, w - 10), rng.uniform(-3, h - 10)
            bw, bh = rng.uniform(2, w / 2), rng.uniform(2, h / 2)
            kind = g % 5
            if kind == 0:                     # concave L, half-pixel coordinates, may cross the border
                x, y = np.floor(x) + .5, np.floor(y) + .5
                seg = [[x, y, x + bw, y, x + bw, y + bh / 2, x + bw / 2, y + bh / 2, x + bw / 2, y + bh, x, y + bh]]
            elif kind == 1:                   # two parts
                seg = [_poly_rect(x, y, bw / 2, bh / 2), _poly_rect(x + bw / 3, y + bh / 3, bw / 2, bh / 2)]
            elif kind == 2:                   # sub-pixel triangle
                seg = [[x, y, x + .3, y + .1, x + .1, y + .4]]
            elif kind == 3:                   # touching the right / bottom border, star-shaped
                cx, cy = w - bw / 4, h - bh / 4
                t = np.linspace(0, 2 * np.pi, 11)[:-1]
                r = np.where(np.arange(10) % 2, bw / 4, bw / 2)
                seg = [list(np.stack([cx + r * np.cos(t), cy + r * np.sin(t)], 1).reshape(-1))]
            else:                             # a repeated vertex (a zero-length edge)
                seg = [[x, y, x + bw, y, x + bw, y, x + bw / 2, y + bh]]
            seg = [[float(v) for v in p] for p in seg]
            area = [1024, 9216, float(bw * bh), 32.0 ** 2, float(rng.uniform(0, 2e4))][g % 5]
            add(img, cat, seg, [x, y, bw, bh], area)
        if n % 3 == 0:                        # crowd region as uncompressed RLE
            m = np.zeros((h, w), np.uint8)
            m[h // 4:h // 2, w // 3:w - 2] = 1
            flat = m.flatten(order='F')
            change = np.flatnonzero(np.diff(np.concatenate([[0], flat, [2]])) != 0)
            counts = np.diff(np.concatenate([[0], change])).tolist()
            add(img, 7, dict(size=[h, w], counts=[int(c) for c in counts]), [w // 3, h // 4, w - 2 - w // 3, h // 2 - h // 4],
                float(flat.sum()), crowd=1)
        if n % 4 == 2 and encode is not None:   # compressed RLE GT
            m = np.zeros((h, w), np.uint8)
            m[2:h // 3, 3:w // 2] = 1
            add(img, 1, dict(size=[h, w], counts=encode(m)), [3, 2, w // 2 - 3, h // 3 - 2], float(m.sum()))
    # exact-threshold boxes on the last image: GT 10 x 10 at (4, 4); detections cover 50 and 75 of its 100 pixels
    last = img_ids[-1]
    add(last, 12, [_poly_rect(4, 4, 10, 10)], [4, 4, 10, 10], 100.0)
    dataset = dict(images=images, annotations=anns, categories=[dict(id=c, name="c%d" % c) for c in cat_ids])

    # detections: all_boxes[j][i] for contiguous class j (dataset category order), image i in sorted-id order
    J = len(cat_ids) + 1
    all_boxes = [[[] for _ in img_ids] for _ in range(J)]
    all_segms = [[[] for _ in img_ids] for _ in range(J)] if with_masks else None
    for i, img in enumerate(img_ids):
        h, w = hw[img]
        if i == 2:
            continue                          # an image without detections
        for j in range(1, J):
            if cat_ids[j - 1] == 20:
                continue
            n = 130 if (i == 3 and j == 1) else int(rng.randint(0, 9))
            if n == 0:
                continue
            x1, y1 = rng.uniform(-2, w - 5, n), rng.uniform(-2, h - 5, n)
            x2, y2 = x1 + rng.uniform(1, w / 2, n), y1 + rng.uniform(1, h / 2, n)
            sc = np.round(rng.uniform(0.05, 1, n) * 8) / 8     # few distinct scores: ties within and across images
            d = np.stack([x1, y1, x2, y2, sc], 1).astype(np.float32)
            # jittered copies of the GT boxes of this image and class: detections that match at some thresholds
            near = [a['bbox'] for a in anns if a['image_id'] == img and a['category_id'] == cat_ids[j - 1] and rng.rand() < .8]
            if near:
                b = np.array(near) + rng.uniform(-2, 2, (len(near), 4))
                nd = np.stack([b[:, 0], b[:, 1], b[:, 0] + b[:, 2] - 1, b[:, 1] + b[:, 3] - 1, rng.randint(1, 9, len(near)) / 8.], 1)
                d = np.concatenate([d, nd.astype(np.float32)])
            if img == last and cat_ids[j - 1] == 12:
                d = np.concatenate([d, np.array([[4, 4, 13, 8, .9], [4, 4, 13, 10.5, .8]], np.float32)])
            all_boxes[j][i] = d
            if with_masks:
                segs = []
                for r in d:
                    m = np.zeros((h, w), np.uint8)
                    a, b = int(max(r[1], 0)), int(max(r[0], 0))
                    m[a:max(int(r[3]), a + 1), b:max(int(r[2]), b + 1)] = 1
                    if rng.rand() < .3:
                        m[a:a + 2, :] = 0             # split into more runs
                    segs.append(dict(size=[h, w], counts=encode(m)))
                all_segms[j][i] = segs
    return dataset, all_boxes, all_segms


def results_file(dataset, all_boxes, all_segms, iou_type):
    """_write_coco_bbox_results_file / _write_coco_segms_results_file, then json.dump + json.load (what loadRes reads)."""
    cats = [c['id'] for c in dataset['categories']]
    img_ids = sorted(im['id'] for im in dataset['images'])
    res = []
    for j, cat in enumerate(cats, 1):
        if j >= len(all_boxes):
            break
        for i, img in enumerate(img_ids):
            dets = all_boxes[j][i]
            if isinstance(dets, list) and len(dets) == 0:
                continue
            dets = dets.astype(np.float64)
            scores = dets[:, -1]
            if iou_type == 'bbox':
                xywh = np.hstack((dets[:, 0:2], dets[:, 2:4] - dets[:, 0:2] + 1))
                res.extend([{'image_id': img, 'category_id': cat, 'bbox': [xywh[k, 0], xywh[k, 1], xywh[k, 2], xywh[k, 3]],
                             'score': scores[k]} for k in range(dets.shape[0])])
            else:
                res.extend([{'image_id': img, 'category_id': cat, 'segmentation': all_segms[j][i][k], 'score': scores[k]}
                            for k in range(dets.shape[0])])
    return json.loads(json.dumps(res))


def oracle_eval(mods, dataset, all_boxes, all_segms, iou_type):
    """-> the COCOeval object after evaluate() + accumulate() + summarize() (output silenced)."""
    COCO, COCOeval, _ = mods
    with contextlib.redirect_stdout(io.StringIO()):
        gt = COCO()
        gt.dataset = copy.deepcopy(dataset)
        gt.createIndex()
        dt = gt.loadRes(results_file(dataset, all_boxes, all_segms, iou_type))
        E = COCOeval(gt, dt, iou_type)
        E.evaluate()
        E.accumulate()
        E.summarize()
    return E

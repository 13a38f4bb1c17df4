"""The reference's results writers (lib/utils/json_dataset_evaluator.py _write_coco_bbox_results_file /
_write_coco_segms_results_file + json.dump) restated, and a JsonDataset-like object to run the reference's own writers on."""
import json

import numpy as np


def reference_text(image_ids, category_ids, all_boxes, all_segms, iou_type):
    """The bytes json.dump writes for the reference's results list (classes j = 1.. over category_ids, break at len(all_boxes))."""
    res = []
    img_ids = sorted(int(v) for v in image_ids)
    for j, cat in enumerate(category_ids, 1):
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
                res.extend([{'image_id': img, 'category_id': int(cat), 'bbox': [xywh[k, 0], xywh[k, 1], xywh[k, 2], xywh[k, 3]],
                             'score': scores[k]} for k in range(dets.shape[0])])
            else:
                res.extend([{'image_id': img, 'category_id': int(cat), 'segmentation': all_segms[j][i][k], 'score': scores[k]}
                            for k in range(dets.shape[0])])
    return json.dumps(res).encode()


class FakeCOCO:
    def __init__(self, image_ids):
        self._ids = list(image_ids)

    def getImgIds(self):
        return list(self._ids)


class FakeJsonDataset:
    """What the results writers read of a JsonDataset: classes, category_to_id_map, COCO.getImgIds() (and name)."""

    def __init__(self, image_ids, category_ids, name='coco_2017_test-dev'):
        self.name = name
        self.classes = ['__background__'] + ['c%d' % c for c in category_ids]
        self.category_to_id_map = {'c%d' % c: int(c) for c in category_ids}
        self.COCO = FakeCOCO(image_ids)


def per_class(results, num_images):
    """detect_images / batch_results per-image tuples -> (all_boxes, all_segms) [class][image], as extend_results files them."""
    nc = max(len(r[2]) for r in results)
    boxes = [[[] for _ in range(num_images)] for _ in range(nc)]
    segms = [[[] for _ in range(num_images)] for _ in range(nc)]
    for i, r in enumerate(results):
        for j in range(1, len(r[2])):
            boxes[j][i] = r[2][j]
            if r[3] is not None:
                segms[j][i] = r[3][j]
    return boxes, segms

"""Host side of the per-image records (evaluate(..., keep_eval_imgs=True)), without a GPU: the detection-id column of the results
conversion is the id COCO.loadRes gives each result, 1 + its index in the notebooks' results file, whatever the category order."""
import json
import os

import numpy as np
import pytest

import coco_eval_cases as cc

GOLD = os.path.join(os.path.dirname(__file__), "golden", "coco_eval_golden.npz")


def _golden_case():
    case = json.loads(np.load(GOLD)['case'].tobytes().decode())
    boxes = [[np.array(b, np.float32).reshape(-1, 5) if len(b) else [] for b in c] for c in case['all_boxes']]
    return case['dataset'], boxes, case['all_segms']


@pytest.mark.parametrize("order", ["dataset", "permuted", "shortened"])
def test_detection_ids_follow_results_file(order):
    from detectorch_b200.utils import coco_eval
    ds, boxes, segms = _golden_case()
    gt = coco_eval.CocoGroundTruth(dict(ds, annotations=[{k: v for k, v in a.items() if k != 'segmentation'} for a in ds['annotations']]),
                                   device='cpu')
    cids = {"dataset": gt.category_ids, "permuted": gt.category_ids[::-1], "shortened": gt.category_ids[:-1]}[order]
    for t in ('bbox', 'segm'):
        res = cc.results_file(dict(ds, categories=[dict(id=c) for c in cids]), boxes, segms, t)
        key, f, i, chars, ids = coco_eval._flatten_results(gt, boxes, segms, t, cids, with_ids=True)
        assert ids.dtype.kind == 'i' and np.array_equal(np.sort(ids), np.arange(1, len(res) + 1))
        rows = [res[n - 1] for n in ids]
        assert np.array_equal(key, [gt.cat_ids.index(r['category_id']) * gt.num_images + gt.img_ids.index(r['image_id']) for r in rows])
        assert np.array_equal(f[:, 0], [r['score'] for r in rows])
        if t == 'bbox':
            assert np.array_equal(f[:, 1:], [r['bbox'] for r in rows])
        else:
            assert [chars[a:a + b] for a, b in i[:, :2]] == [r['segmentation']['counts'].encode() for r in rows]
        if order == "permuted":
            assert not np.array_equal(ids, np.arange(1, len(ids) + 1))       # the file order is not the (category, image) order
        # without with_ids the conversion is what it was
        assert all(np.array_equal(a, b) for a, b in zip(coco_eval._flatten_results(gt, boxes, segms, t, cids)[:3], (key, f, i)))

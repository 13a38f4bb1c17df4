"""Host side of the device COCO evaluation, without a GPU: the results conversion equals the notebooks' results file, malformed
annotations and results raise before anything is launched, and (where oracle/build_cocoapi.sh has built it) the reference's own
pycocotools pins the project's RLE encoder restatement and reproduces the committed golden arrays."""
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


def _bbox_gt(ds):
    """The golden ground truth without masks: nothing is built on a device."""
    from detectorch_b200.utils import coco_eval
    d = dict(ds, annotations=[{k: v for k, v in a.items() if k != 'segmentation'} for a in ds['annotations']])
    return coco_eval.CocoGroundTruth(d, device='cpu')


def test_results_conversion_equals_results_file():
    """_flatten_results == _write_coco_*_results_file + json round trip, grouped by (category, image) in file order."""
    from detectorch_b200.utils import coco_eval
    ds, boxes, segms = _golden_case()
    gt = _bbox_gt(ds)
    assert not gt.has_masks
    for t in ('bbox', 'segm'):
        res = cc.results_file(ds, boxes, segms, t)
        key = np.array([gt.cat_ids.index(r['category_id']) * gt.num_images + gt.img_ids.index(r['image_id']) for r in res])
        order = np.argsort(key, kind='stable')
        k, f, i, chars = coco_eval._flatten_results(gt, boxes, segms, t, gt.category_ids)
        assert np.array_equal(k, key[order])
        assert np.array_equal(f[:, 0], np.array([res[n]['score'] for n in order]))
        if t == 'bbox':
            assert np.array_equal(f[:, 1:], np.array([res[n]['bbox'] for n in order]))
        else:
            assert [chars[a:a + b] for a, b in i[:, :2]] == [res[n]['segmentation']['counts'].encode() for n in order]
            assert np.array_equal(i[:, 2:], np.array([res[n]['segmentation']['size'] for n in order]))


def test_ground_truth_tables():
    ds, _, _ = _golden_case()
    gt = _bbox_gt(ds)
    assert gt.img_ids == sorted(im['id'] for im in ds['images']) and gt.cat_ids == sorted(c['id'] for c in ds['categories'])
    assert gt.num_gts == len(ds['annotations']) and np.all(np.diff(gt.keys) >= 0)
    byid = {a['id']: a for a in ds['annotations']}
    for n, aid in enumerate(gt.ann_ids):
        a = byid[aid]
        assert gt.keys[n] == gt.cat_ids.index(a['category_id']) * gt.num_images + gt.img_ids.index(a['image_id'])
        assert list(gt._gt_f[n, :5]) == a['bbox'] + [a['area']] and gt._gt_i[n, 4] == a['iscrowd']


def _ds(**ann):
    a = dict(id=1, image_id=1, category_id=1, bbox=[0., 0., 4., 4.], area=16., iscrowd=0, segmentation=[[0., 0., 4., 0., 4., 4.]])
    a.update(ann)
    return dict(images=[dict(id=1, height=10, width=10)], categories=[dict(id=1)], annotations=[a])


@pytest.mark.parametrize("bad", [
    dict(bbox=[0, 0, 4]), dict(bbox=[0, 0, float('nan'), 4]), dict(area=None), dict(iscrowd=2), dict(iscrowd=None),
    dict(segmentation=[]), dict(segmentation=[[0., 0., 4., 4.]]), dict(segmentation=[[0., 0., 4., 0., 4.]]),
    dict(segmentation=[[0., 0., 4., 0., 4., float('inf')]]), dict(segmentation=[[0., 0., 4., 0., 4., 1e12]]),
    dict(segmentation=dict(size=[10, 10], counts=[3, -1])), dict(segmentation=dict(size=[10], counts=[3])),
    dict(segmentation=dict(size=[10, 10], counts="0p")), dict(segmentation=dict(size=[10, 10], counts="0\x7f1")),
    dict(segmentation=dict(size=[10, 10], counts="0" + "P" * 6 + "1")), dict(segmentation="x"), dict(id=1.5),
    # runs that do not cover the mask: rleIou's merge of two such masks never ends
    dict(segmentation=dict(size=[10, 10], counts=[3, 5])), dict(segmentation=dict(size=[10, 10], counts="35")),
    dict(segmentation=dict(size=[10, 10], counts=[])), dict(segmentation=dict(size=[10, 10], counts=[90, 20])),
    # a count difference of 2^29: 7 chars in pycocotools' string form
    dict(segmentation=dict(size=[30000, 30000], counts=[0, 900000000])),
])
def test_malformed_annotations_raise(bad):
    from detectorch_b200.utils import coco_eval
    with pytest.raises(ValueError):
        coco_eval.CocoGroundTruth(_ds(**bad), device='cpu')


def test_malformed_datasets_raise():
    from detectorch_b200.utils import coco_eval
    ds = _ds()
    for bad in (dict(ds, images=ds['images'] * 2), dict(ds, categories=ds['categories'] * 2), dict(ds, annotations=ds['annotations'] * 2),
                dict(ds, images=[dict(id=1, height=0, width=10)]),
                dict(ds, images=[dict(id=1, height=23171, width=23171)])):      # a polygon on 2^29 pixels: its RLE may need 7-char values
        with pytest.raises(ValueError):
            coco_eval.CocoGroundTruth(bad, device='cpu')
    with pytest.raises(ValueError):
        coco_eval.CocoGroundTruth([ds], device='cpu')


def test_malformed_results_raise():
    """Everything is checked before the first launch: these run without a GPU."""
    from detectorch_b200.utils import coco_eval
    ds, boxes, segms = _golden_case()
    gt = _bbox_gt(ds)
    J, I = len(boxes), gt.num_images
    ok = np.array([[1, 1, 5, 5, .5]], np.float32)

    def one(d, s=None):
        b = [[[] for _ in range(I)] for _ in range(J)]
        b[1][0] = d
        sg = None if s is None else [[[] for _ in range(I)] for _ in range(J)]
        if s is not None:
            sg[1][0] = s
        return b, sg
    cases = [(one(np.array([[1, 1, 5, 5, np.nan]], np.float32)), 'bbox'), (one(np.zeros((1, 4), np.float32)), 'bbox'),
             (([[[]] * (I - 1)] * J, None), 'bbox'), (one(ok), 'segm'),
             (one(ok, [dict(size=[10, 10], counts="0p")]), 'segm'), (one(ok, [dict(size=[10, 10], counts=[1, 2])]), 'segm'),
             (one(ok, [dict(size=[0, 10], counts="0")]), 'segm'), (one(ok, []), 'segm')]
    for (b, s), t in cases:
        with pytest.raises(ValueError):
            gt_t = gt if t == 'bbox' else _masked_gt_stub(gt)
            coco_eval.evaluate(gt_t, b, t, s)
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, boxes, 'segm', segms)          # the ground truth has no masks
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, boxes, 'keypoints')
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, boxes, 'bbox', category_ids=[999])


def _masked_gt_stub(gt):
    import copy
    g = copy.copy(gt)
    g.has_masks = True
    return g


def test_oracle_pins_rle_encoder():
    """oracle/ref.py's rleEncode + rleToString restatement (used for the segm golden strings) against pycocotools' mask.encode."""
    from oracle import cocoapi, ref
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh)")
    mask = cocoapi.load()[2]
    rng = np.random.RandomState(3)
    for n in range(200):
        h, w = rng.randint(1, 40, 2)
        m = (rng.rand(h, w) < rng.choice([0.02, 0.5, 0.98])).astype(np.uint8)
        if n % 7 == 0:
            m[:] = n % 2
        want = mask.encode(np.asfortranarray(m[:, :, None]))[0]['counts']
        assert ref.rle_to_string(ref.rle_encode(m)) == want, n


def test_oracle_reproduces_golden():
    """The committed golden arrays are what the reference's COCOeval computes on the committed case."""
    from oracle import cocoapi
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh)")
    mods = cocoapi.load()
    z = np.load(GOLD)
    ds, boxes, segms = _golden_case()
    for t in ('bbox', 'segm'):
        E = cc.oracle_eval(mods, ds, boxes, segms, t)
        for k in ('precision', 'recall', 'scores'):
            assert np.array_equal(E.eval[k], z[t + '_' + k]), (t, k)
        assert np.array_equal(np.array(E.stats), z[t + '_stats'])

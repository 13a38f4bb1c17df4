"""Host side of evaluate(..., params=) without a GPU: every rejected Params raises ValueError before anything is launched, the
normalisation follows COCOeval.evaluate(), and the re-indexed gt rows and detection rows of each pair come in the order in which the
reference COCOeval's _prepare / computeIoU concatenate them (checked against the live reference where it is built)."""
import contextlib
import copy
import io

import numpy as np
import pytest
import torch

import coco_eval_cases as cc
import coco_eval_fuzz_cases as fz


def _gt(ds):
    """A box-only CocoGroundTruth on the CPU: no mask is built, so nothing is launched."""
    from detectorch_b200.utils import coco_eval
    ds = dict(ds, annotations=[{k: v for k, v in a.items() if k != 'segmentation'} for a in ds['annotations']])
    return coco_eval.CocoGroundTruth(ds, device='cpu')


def _case():
    ds, boxes, _ = fz.make_case("wide", 0)
    return ds, boxes


def _p(gt, **kw):
    from detectorch_b200.utils import coco_eval
    p = coco_eval.Params(gt, kw.pop('iou_type', 'bbox'))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_rejections_raise_before_any_launch():
    from detectorch_b200.utils import coco_eval
    ds, boxes = _case()
    gt = _gt(ds)
    bad = [dict(imgIds=[]), dict(catIds=[]), dict(imgIds=[gt.img_ids[0], 123456789]), dict(catIds=[gt.cat_ids[0], 999]),
           dict(imgIds="1"), dict(imgIds=[1.5]), dict(iouThrs=np.linspace(.5, .9, 9)), dict(iouThrs=coco_eval.IOU_THRS + 1e-12),
           dict(recThrs=np.linspace(0, 1, 11)), dict(maxDets=[1, 10, 300]), dict(maxDets=[100]),
           dict(areaRng=[[0, 1e10]] * 4), dict(areaRngLbl=['all', 'a', 'b', 'c']), dict(useCats=2), dict(useCats=0.0),
           dict(useCats=0, catIds=[gt.cat_ids[0], gt.cat_ids[0]]), dict(iou_type='segm')]
    for kw in bad:
        with pytest.raises(ValueError):
            coco_eval.evaluate(gt, boxes, 'bbox', params=_p(gt, **kw))
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, boxes, 'bbox', params=dict(imgIds=gt.img_ids))


def test_normalised_as_cocoeval():
    from detectorch_b200.utils import coco_eval
    ds, _ = _case()
    gt = _gt(ds)
    imgs, cats = gt.img_ids[::-1][:5] + gt.img_ids[:2], gt.cat_ids[::-1][:4] + gt.cat_ids[-1:]
    p = coco_eval._normalised_params(gt, _p(gt, imgIds=imgs, catIds=cats, maxDets=[100, 1, 10]), 'bbox')
    assert p.imgIds == sorted(set(imgs)) and p.catIds == sorted(set(cats)) and p.maxDets == [1, 10, 100] and p.useCats == 1
    p = coco_eval._normalised_params(gt, _p(gt, catIds=cats[:4], useCats=0), 'bbox')
    assert p.catIds == cats[:4] and p.useCats == 0
    assert coco_eval._is_default(gt, coco_eval._normalised_params(gt, _p(gt), 'bbox'))


def _prepared(ds, res, imgs, cats, use_cats):
    from oracle import cocoapi
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh)")
    COCO, COCOeval, _ = cocoapi.load()
    with contextlib.redirect_stdout(io.StringIO()):
        g = COCO()
        g.dataset = copy.deepcopy(ds)
        g.createIndex()
        E = COCOeval(g, g.loadRes(res), 'bbox')
        E.params.imgIds, E.params.catIds, E.params.useCats = list(imgs), list(cats), use_cats
        E.params.imgIds = list(np.unique(E.params.imgIds))
        if use_cats:
            E.params.catIds = list(np.unique(E.params.catIds))
        E._prepare()
    return E


@pytest.mark.parametrize("use_cats", [1, 0])
def test_pair_rows_in_cocoeval_order(use_cats):
    """Per pair, the gt ids and detection ids (loadRes ids) in the order COCOeval concatenates them per (image, category list)."""
    from detectorch_b200.utils import coco_eval
    ds, boxes = _case()
    gt = _gt(ds)
    rng = np.random.RandomState(use_cats)
    imgs = [gt.img_ids[i] for i in rng.permutation(len(gt.img_ids))[:30]]
    cats = [gt.cat_ids[i] for i in rng.permutation(len(gt.cat_ids))[:25]]
    p = coco_eval._normalised_params(gt, _p(gt, imgIds=imgs, catIds=cats, useCats=use_cats), 'bbox')
    view = coco_eval._GtView(gt, p)
    key, _, _, _, ids = coco_eval._flatten_results(gt, boxes, None, 'bbox', list(gt.category_ids), with_ids=True)
    rows, fine = view.select(key)
    dkey, dids = fine // view.per, ids[rows]
    E = _prepared(ds, cc.results_file(ds, boxes, None, 'bbox'), imgs, cats, use_cats)
    I = view.num_images
    n_pairs = 0
    for ki, cat in enumerate(view.cat_ids):
        for ii, img in enumerate(view.img_ids):
            k = ki * I + ii
            cs = [cat] if use_cats else p.catIds
            want_g = [a['id'] for c in cs for a in E._gts[img, c]]
            want_d = [d['id'] for c in cs for d in E._dts[img, c]]
            got_g = [view.ann_ids[r] for r in np.flatnonzero(view.keys == k)]
            assert got_g == want_g, (img, cat)
            assert dids[dkey == k].tolist() == want_d, (img, cat)
            n_pairs += bool(want_d or want_g)
    assert n_pairs > 10
    assert np.array_equal(view.gt_f.numpy(), gt.gt_f.numpy()[view.rows])

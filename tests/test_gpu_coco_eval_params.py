"""Evaluation with COCOeval's imgIds, catIds and useCats (evaluate(..., params=)) against the reference's own pycocotools COCOeval
(built by oracle/build_cocoapi.sh into oracle/_ref) run with the same Params on the results file: precision, recall, scores, stats and
every IoU matrix np.array_equal, evalImgs record by record.  Cases: the golden case and every family of tests/coco_eval_fuzz_cases.py
with image subsets (half, one, out of order with repeats), category subsets (one, a few shuffled), useCats 0 alone and with an image
subset; cross-category matches (a crowd gt among them) and score ties across categories; DeviceResults input; the sort-based rank."""
import contextlib
import copy
import io

import numpy as np
import pytest
import torch

import coco_eval_cases as cc
import coco_eval_fuzz_cases as fz
from test_gpu_device_results import _accumulate, _case
from test_gpu_eval_imgs import _golden_case, _results, _same_records

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def oracle(dev):
    from oracle import cocoapi
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh)")
    mods = cocoapi.load()
    mask = mods[2]
    return mods, lambda m: mask.encode(np.asfortranarray(m[:, :, None]))[0]['counts'].decode()


def _variants(gt, seed):
    """(name, imgIds, catIds, useCats) of the params the tests evaluate with."""
    rng = np.random.RandomState(seed)
    imgs, cats = list(gt.img_ids), list(gt.cat_ids)
    half = [imgs[i] for i in sorted(rng.permutation(len(imgs))[:max(1, len(imgs) // 2)])]
    messy = [imgs[i] for i in rng.randint(0, len(imgs), max(2, len(imgs) // 3))]
    messy = messy[::-1] + messy[:2]
    shuffled = [cats[i] for i in rng.permutation(len(cats))[:min(3, len(cats))]]
    return [("half", half, cats, 1), ("one image", [imgs[int(rng.randint(len(imgs)))]], cats, 1), ("repeats", messy, cats, 1),
            ("one category", imgs, [cats[int(rng.randint(len(cats)))]], 1), ("few categories", imgs, shuffled, 1),
            ("agnostic", imgs, [cats[i] for i in rng.permutation(len(cats))], 0), ("agnostic half", half, cats[::-1], 0)]


def _params(gt, t, imgs, cats, use_cats):
    from detectorch_b200.utils import coco_eval
    p = coco_eval.Params(gt, t)
    p.imgIds, p.catIds, p.useCats = list(imgs), list(cats), use_cats
    return p


def _cocoeval(mods, ds, res, t, imgs, cats, use_cats):
    COCO, COCOeval, _ = mods
    with contextlib.redirect_stdout(io.StringIO()):
        g = COCO()
        g.dataset = copy.deepcopy(ds)
        g.createIndex()
        E = COCOeval(g, g.loadRes(copy.deepcopy(res)), t)         # loadRes edits the results in place
        E.params.imgIds, E.params.catIds, E.params.useCats = list(imgs), list(cats), use_cats
        E.evaluate()
        E.accumulate()
        E.summarize()
    return E


def _same(got, E, what):
    for k in ('precision', 'recall', 'scores'):
        a, b = got.eval[k], E.eval[k]
        assert a.shape == b.shape and np.array_equal(a, b), (what, k)
    assert np.array_equal(got.stats, np.array(E.stats)), (what, got.stats, E.stats)
    want = {(int(i), int(c)): np.asarray(v, np.float64) for (i, c), v in E.ious.items() if len(v)}
    assert set(got.ious) == set(want), (what, sorted(set(got.ious) ^ set(want))[:5])
    for key, v in want.items():
        assert got.ious[key].shape == v.shape and np.array_equal(got.ious[key], v), (what, key)
    return _same_records(got.evalImgs, E.evalImgs, what)


def _check(mods, case, name, seed=0, variants=None):
    from detectorch_b200.utils import coco_eval
    ds, boxes, segms = case
    gt = coco_eval.CocoGroundTruth(ds)
    n = 0
    for t in ('bbox', 'segm'):
        res = _results(ds, boxes, segms, t, None)
        for vname, imgs, cats, uc in (variants or _variants(gt, seed)):
            got = coco_eval.evaluate(gt, boxes, t, segms if t == 'segm' else None, keep_ious=True, keep_eval_imgs=True,
                                     params=_params(gt, t, imgs, cats, uc))
            assert got.params.imgIds == sorted(set(imgs)) and got.params.useCats == uc
            assert got.params.catIds == (sorted(set(cats)) if uc else list(cats))
            n += _same(got, _cocoeval(mods, ds, res, t, imgs, cats, uc), (name, t, vname))
    return n


def test_golden_with_params(oracle):
    mods, _ = oracle
    assert _check(mods, _golden_case(), "golden") > 0


@pytest.mark.parametrize("family", list(fz.FAMILIES))
def test_family_with_params(oracle, family):
    mods, enc = oracle
    assert _check(mods, fz.make_case(family, 0, enc), family, seed=list(fz.FAMILIES).index(family)) > 0


def _cross_case(enc):
    """Two categories on each image: a detection of category A sits on a gt of category B (a crowd one on image 2), another
    detection of B on A's gt; scores tie across categories, so the concatenation order over catIds decides their order."""
    c = fz.Case(np.random.RandomState(7), [3, 1, 2], enc)
    for n in range(4):
        img = c.image(60, 80)
        c.poly_gt(img, 1, [[5, 5, 30, 5, 30, 30, 5, 30]], area=625.)
        c.poly_gt(img, 2, [[40, 10, 70, 10, 70, 50, 40, 50]], area=1200., crowd=int(n == 2))
        c.poly_gt(img, 3, [[10, 35, 25, 35, 25, 55, 10, 55]], area=300.)
        c.det(img, 2, [5, 5, 30, 30], 0.75)                  # category 2 on category 1's gt
        c.det(img, 1, [41, 11, 69, 49], 0.75)                # category 1 on category 2's gt (crowd on image 2)
        c.det(img, 3, [6, 6, 29, 29], 0.75)                  # a third category, same score
        c.det(img, 3, [10, 35, 25, 55], 0.5)
        c.det(img, 1, [42, 12, 60, 40], 0.5)
    return c.build()


def test_cross_category_matches_and_ties(oracle):
    from detectorch_b200.utils import coco_eval
    mods, enc = oracle
    ds, boxes, segms = _cross_case(enc)
    gt = coco_eval.CocoGroundTruth(ds)
    cat_of = {a['id']: a['category_id'] for a in ds['annotations']}
    crowd = {a['id'] for a in ds['annotations'] if a['iscrowd']}
    for order in ([1, 2, 3], [3, 1, 2], [2, 3, 1]):
        _check(mods, (ds, boxes, segms), "cross %s" % order, variants=[("agnostic", gt.img_ids, order, 0)])
    for t in ('bbox', 'segm'):
        got = coco_eval.evaluate(gt, boxes, t, segms if t == 'segm' else None, keep_eval_imgs=True,
                                 params=_params(gt, t, gt.img_ids, [1, 2, 3], 0))
        res = _results(ds, boxes, segms, t, None)
        det_cat = {n + 1: r['category_id'] for n, r in enumerate(res)}
        c = got.eval_imgs
        m = c['dtMatches'][0]
        ids = c['dtIds']
        other = [(int(d), int(g)) for d, g in zip(ids, m) if g > 0 and cat_of[int(g)] != det_cat[int(d)]]
        assert other, t
        assert any(g in crowd for _, g in other), t


@pytest.mark.parametrize("seed", [1, 2])
def test_device_results_with_params(dev, oracle, seed):
    """DeviceResults (batches added out of id order) == list input for every params variant, and == COCOeval's records."""
    from detectorch_b200.utils import coco_eval
    mods, _ = oracle
    gt, ds, batches, results = _case(dev, seed=seed)
    acc = _accumulate(batches, dev)
    for t in ('bbox', 'segm'):
        boxes, segms = coco_eval._per_class(gt, results, None, t)
        res = _results(ds, boxes, segms, t, None)
        for vname, imgs, cats, uc in _variants(gt, seed):
            p = _params(gt, t, imgs, cats, uc)
            want = coco_eval.evaluate(gt, results, t, keep_eval_imgs=True, keep_ious=True, params=p)
            got = coco_eval.evaluate(gt, acc, t, keep_eval_imgs=True, keep_ious=True, params=p)
            for k in ('precision', 'recall', 'scores'):
                assert np.array_equal(got.eval[k], want.eval[k]), (t, vname, k)
            for k, v in want.eval_imgs.items():
                assert v.dtype == got.eval_imgs[k].dtype and np.array_equal(v, got.eval_imgs[k]), (t, vname, k)
            assert got.ious.keys() == want.ious.keys() and all(np.array_equal(got.ious[k], want.ious[k]) for k in want.ious)
            _same(got, _cocoeval(mods, ds, res, t, imgs, cats, uc), ("DeviceResults", t, vname))


def test_device_flattening_with_params_does_not_synchronise(dev):
    from detectorch_b200.utils import coco_eval
    gt, _, batches, results = _case(dev, seed=3)
    acc = _accumulate(batches, dev)
    cids = list(gt.category_ids)
    for vname, imgs, cats, uc in _variants(gt, 3):
        view = coco_eval._GtView(gt, coco_eval._normalised_params(gt, _params(gt, 'segm', imgs, cats, uc), 'segm'))
        acc._drain()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            b = coco_eval._bins_device(gt, acc, 'segm', cids, keep_eval_imgs=True, view=view)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert b['tail'].shape == (9,), vname


def test_default_params_change_nothing(oracle):
    from detectorch_b200.utils import coco_eval
    _, enc = oracle
    ds, boxes, segms = fz.make_case("matching", 0, enc)
    gt = coco_eval.CocoGroundTruth(ds)
    for t in ('bbox', 'segm'):
        s = segms if t == 'segm' else None
        a = coco_eval.evaluate(gt, boxes, t, s, keep_ious=True, keep_eval_imgs=True)
        b = coco_eval.evaluate(gt, boxes, t, s, keep_ious=True, keep_eval_imgs=True, params=coco_eval.Params(gt, t))
        for k in ('precision', 'recall', 'scores'):
            assert np.array_equal(a.eval[k], b.eval[k])
        for k, v in a.eval_imgs.items():
            assert np.array_equal(v, b.eval_imgs[k]), k
        assert a.ious.keys() == b.ious.keys() and np.array_equal(a.stats, b.stats)


def test_agnostic_rank_of_1e5_detections(oracle):
    """useCats 0 over 1000 images of 100 detections: one category holding 100,000 kept detections, scores on 9 levels (ties within and
    across images and categories); accumulate()'s order comes from the sort over all of them."""
    from detectorch_b200.utils import coco_eval
    mods, _ = oracle
    rng = np.random.RandomState(11)
    c = fz.Case(rng, [4, 2, 7])
    for n in range(1000):
        img = c.image(100, 100)
        for g in range(3):
            x, y, w, h = rng.uniform(0, 60), rng.uniform(0, 60), rng.uniform(5, 40), rng.uniform(5, 40)
            c.gt(img, int(rng.choice(c.cat_ids)), None, [x, y, w, h], w * h, crowd=int(rng.rand() < .05))
            for _ in range(20):
                j = rng.uniform(-4, 4, 4)
                c.det(img, int(rng.choice(c.cat_ids)), [x + j[0], y + j[1], x + w + j[2], y + h + j[3]], float(rng.randint(0, 9)) / 8)
        for _ in range(40):
            x, y = rng.uniform(0, 90), rng.uniform(0, 90)
            c.det(img, int(rng.choice(c.cat_ids)), [x, y, x + rng.uniform(1, 30), y + rng.uniform(1, 30)], float(rng.randint(0, 9)) / 8)
    ds, boxes, _ = c.build()
    ds = dict(ds, annotations=[{k: v for k, v in a.items() if k != 'segmentation'} for a in ds['annotations']])
    gt = coco_eval.CocoGroundTruth(ds)
    res = _results(ds, boxes, None, 'bbox', None)
    assert len(res) == 100000
    for vname, imgs, cats, uc in (("agnostic", gt.img_ids, [7, 2, 4], 0), ("per category", gt.img_ids, gt.cat_ids, 1)):
        got = coco_eval.evaluate(gt, boxes, 'bbox', params=_params(gt, 'bbox', imgs, cats, uc))
        E = _cocoeval(mods, ds, res, 'bbox', imgs, cats, uc)
        for k in ('precision', 'recall', 'scores'):
            assert got.eval[k].shape == E.eval[k].shape and np.array_equal(got.eval[k], E.eval[k]), (vname, k)
        assert np.array_equal(got.stats, np.array(E.stats)), vname

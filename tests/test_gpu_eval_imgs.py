"""Per-image records of the device COCO evaluation (evaluate(..., keep_eval_imgs=True)) against the reference's own pycocotools
COCOeval.evalImgs (built by oracle/build_cocoapi.sh into oracle/_ref), record by record: the same length and None positions, the same
keys, equal ids / area range / maxDet / score lists, and matches / ignore flags np.array_equal with COCOeval's dtype and shape.  Cases:
the golden case, every family of tests/coco_eval_fuzz_cases.py and its 40 mixed seeds, permuted and shortened category ids, and a
DeviceResults (synthetic batches added out of id order, and two detect() batches of the synthetic Mask R-CNN).  Keeping the records
leaves precision / recall / scores / stats / ious as they are; the DeviceResults flattening adds no host synchronisation."""
import contextlib
import copy
import io
import json
import os
import warnings

import numpy as np
import pytest
import torch

import coco_eval_cases as cc
import coco_eval_fuzz_cases as fz
from test_gpu_device_results import CANVAS, _accumulate, _case, _model, _model_case

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "coco_eval_golden.npz")
COUNTS = dict(evaluations=0, records=0, empty=0)


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def oracle(dev):
    """(COCO, COCOeval, mask) of the reference pycocotools and its mask.encode as a string encoder."""
    from oracle import cocoapi
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh)")
    mods = cocoapi.load()
    mask = mods[2]
    return mods, lambda m: mask.encode(np.asfortranarray(m[:, :, None]))[0]['counts'].decode()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nevalImgs compared: %(evaluations)d evaluations, %(records)d records (+ %(empty)d None positions)" % COUNTS)


def _cocoeval(mods, ds, res, iou_type):
    """COCOeval.evaluate() + accumulate() of the results list res (output silenced)."""
    COCO, COCOeval, _ = mods
    with contextlib.redirect_stdout(io.StringIO()):
        gt = COCO()
        gt.dataset = copy.deepcopy(ds)
        gt.createIndex()
        E = COCOeval(gt, gt.loadRes(res), iou_type)
        E.evaluate()
        E.accumulate()
    return E


def _results(ds, boxes, segms, iou_type, category_ids):
    """The results file evaluate(..., category_ids) stands for: contiguous class j is category_ids[j - 1]."""
    cats = [c['id'] for c in ds['categories']] if category_ids is None else list(category_ids)
    return cc.results_file(dict(ds, categories=[dict(id=c) for c in cats]), boxes, segms, iou_type)


def _same_records(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    n = 0
    for i, (a, b) in enumerate(zip(got, want)):
        assert (a is None) == (b is None), (what, i)
        if a is None:
            COUNTS['empty'] += 1
            continue
        assert a.keys() == b.keys(), (what, i)
        for k in ('image_id', 'category_id', 'aRng', 'maxDet', 'dtIds', 'gtIds', 'dtScores'):
            assert a[k] == b[k], (what, i, k, a[k], b[k])
        for k in ('dtMatches', 'gtMatches', 'gtIgnore', 'dtIgnore'):
            x, y = a[k], b[k]
            assert isinstance(x, np.ndarray) and x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), \
                (what, i, k, x, y)
        n += 1
    COUNTS['records'] += n
    COUNTS['evaluations'] += 1
    return n


def _columns_agree(E):
    """The columns of .eval_imgs and the materialised list hold the same records."""
    c, L = E.eval_imgs, E.evalImgs
    assert [i for i, r in enumerate(L) if r is not None] == c['index'].tolist()
    for r, n in enumerate(c['index']):
        rec = L[n]
        d0, d1, g0, g1 = c['dt_off'][r], c['dt_off'][r + 1], c['gt_off'][r], c['gt_off'][r + 1]
        assert rec['image_id'] == c['image_id'][r] and rec['category_id'] == c['category_id'][r]
        assert rec['aRng'] == E.params.areaRng[c['area'][r]]
        assert rec['dtIds'] == c['dtIds'][d0:d1].tolist() and rec['gtIds'] == c['gtIds'][g0:g1].tolist()
        assert np.array_equal(rec['dtMatches'], c['dtMatches'][:, d0:d1]) and np.array_equal(rec['gtMatches'], c['gtMatches'][:, g0:g1])
        assert np.array_equal(rec['dtIgnore'], c['dtIgnore'][:, d0:d1]) and np.array_equal(rec['gtIgnore'], c['gtIgnore'][g0:g1])


def _check(mods, case, name, category_ids=None, gt=None):
    from detectorch_b200.utils import coco_eval
    ds, boxes, segms = case
    gt = coco_eval.CocoGroundTruth(ds) if gt is None else gt
    for t in ('bbox', 'segm'):
        E = _cocoeval(mods, ds, _results(ds, boxes, segms, t, category_ids), t)
        got = coco_eval.evaluate(gt, boxes, t, segms if t == 'segm' else None, category_ids=category_ids, keep_eval_imgs=True)
        for k in ('precision', 'recall', 'scores'):
            assert np.array_equal(got.eval[k], E.eval[k]), (name, t, k)
        _same_records(got.evalImgs, E.evalImgs, (name, t))
    return gt


def _golden_case():
    case = json.loads(np.load(GOLD)['case'].tobytes().decode())
    boxes = [[np.array(b, np.float32).reshape(-1, 5) if len(b) else [] for b in c] for c in case['all_boxes']]
    return case['dataset'], boxes, case['all_segms']


def test_golden_equals_cocoeval(oracle):
    mods, _ = oracle
    _check(mods, _golden_case(), "golden")


@pytest.mark.parametrize("family", list(fz.FAMILIES))
def test_family_equals_cocoeval(oracle, family):
    mods, enc = oracle
    _check(mods, fz.make_case(family, 0, enc), family)


@pytest.mark.parametrize("seed", range(40))
def test_mixed_seed_equals_cocoeval(oracle, seed):
    mods, enc = oracle
    _check(mods, fz.make_mixed_case(seed, enc), "mixed %d" % seed)


@pytest.mark.parametrize("category_ids", [fz.CAT_IDS[::-1], fz.CAT_IDS[:5]], ids=["permuted", "shortened"])
def test_category_ids_equal_cocoeval(oracle, category_ids):
    """Detection ids follow the results file (class-major in category_ids' order), not the (category, image) key order."""
    from detectorch_b200.utils import coco_eval
    mods, enc = oracle
    case = fz.make_case("matching", 0, enc)
    gt = _check(mods, case, "matching %s" % category_ids, category_ids=category_ids)
    ds, boxes, segms = case
    _, _, _, _, ids = coco_eval._flatten_results(gt, boxes, None, 'bbox', category_ids, with_ids=True)
    assert not np.array_equal(ids, np.arange(1, len(ids) + 1))


def test_keeping_records_changes_nothing_else(dev, oracle):
    from detectorch_b200.utils import coco_eval
    _, enc = oracle
    ds, boxes, segms = fz.make_case("matching", 0, enc)
    gt = coco_eval.CocoGroundTruth(ds)
    for t in ('bbox', 'segm'):
        s = segms if t == 'segm' else None
        a = coco_eval.evaluate(gt, boxes, t, s, keep_ious=True)
        b = coco_eval.evaluate(gt, boxes, t, s, keep_ious=True, keep_eval_imgs=True)
        c = coco_eval.evaluate(gt, boxes, t, s, keep_eval_imgs=True)
        for k in ('precision', 'recall', 'scores'):
            assert np.array_equal(a.eval[k], b.eval[k]) and np.array_equal(a.eval[k], c.eval[k]), (t, k)
        assert np.array_equal(a.stats, b.stats) and np.array_equal(a.stats, c.stats)
        assert a.ious.keys() == b.ious.keys() and all(np.array_equal(a.ious[k], b.ious[k]) for k in a.ious)
        assert not hasattr(a, 'evalImgs') and not hasattr(c, 'ious')
        _columns_agree(b)


def test_device_results_equal_list_input_and_cocoeval(dev, oracle):
    """Synthetic batches added out of id order (two images never added), dataset / permuted / shortened category ids."""
    from detectorch_b200.utils import coco_eval
    mods, _ = oracle
    gt, ds, batches, results = _case(dev, seed=1)
    acc = _accumulate(batches, dev)
    cats = [c['id'] for c in ds['categories']]
    for category_ids in (None, cats[::-1], cats[:9]):
        for t in ('bbox', 'segm'):
            want = coco_eval.evaluate(gt, results, t, category_ids=category_ids, keep_eval_imgs=True)
            got = coco_eval.evaluate(gt, acc, t, category_ids=category_ids, keep_eval_imgs=True)
            for k, v in want.eval_imgs.items():
                assert v.dtype == got.eval_imgs[k].dtype and np.array_equal(v, got.eval_imgs[k]), (category_ids, t, k)
            boxes, segms = coco_eval._per_class(gt, results, None, t)
            E = _cocoeval(mods, ds, _results(ds, boxes, segms, t, category_ids), t)
            _same_records(got.evalImgs, E.evalImgs, ("DeviceResults", category_ids, t))
            _columns_agree(got)


def test_detect_batches_equal_cocoeval(dev, oracle):
    """Two detect() batches of the synthetic-weight Mask R-CNN on ragged images, added out of order, one image never added."""
    from detectorch_b200.utils import blob, coco_eval
    from oracle import network as net
    mods, _ = oracle
    model = _model(net.synthetic_params("resnet50"))
    ims, results, ds, gt = _model_case(model)
    acc = coco_eval.DeviceResults()
    for part in ([5, 2, 0], [6, 3, 1]):
        data, sizes, scales, orig = blob.images_to_batch([ims[p] for p in part], 128, 200, canvas=CANVAS)
        out = model.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
        acc.add(out, [10 * (p + 1) for p in part], original_sizes=orig)
    all_boxes = [[[] for _ in ims]] + [[r[2][j] for r in results] for j in range(1, 81)]
    all_segms = [[[] for _ in ims]] + [[r[3][j] for r in results] for j in range(1, 81)]
    for t in ('bbox', 'segm'):
        got = coco_eval.evaluate(gt, acc, t, keep_eval_imgs=True)
        want = coco_eval.evaluate(gt, results, t, keep_eval_imgs=True)
        for k, v in want.eval_imgs.items():
            assert np.array_equal(v, got.eval_imgs[k]), (t, k)
        E = _cocoeval(mods, ds, cc.results_file(ds, all_boxes, all_segms, t), t)
        assert _same_records(got.evalImgs, E.evalImgs, ("detect", t)) > 0
        assert got.eval_imgs['dtIds'].size > 0 and np.any(got.eval_imgs['dtMatches'] > 0), t


def test_device_flattening_does_not_synchronise(dev, oracle):
    """With the records kept, the DeviceResults flattening enqueues its extra scans without a host synchronisation: everything up to
    the read-back of the sizes runs under sync debug mode "error", and the whole flattening synchronises once."""
    from detectorch_b200.utils import coco_eval
    gt, _, batches, results = _case(dev, seed=3)
    acc = _accumulate(batches, dev)
    cids = list(gt.category_ids)[::-1]
    acc._drain()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = coco_eval._bins_device(gt, acc, 'segm', cids, keep_eval_imgs=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert b['tail'].shape == (9,)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            f = coco_eval._flatten_device(gt, acc, 'segm', cids, keep_eval_imgs=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    assert len(syncs) == 1, [str(x.message) for x in syncs]
    boxes, segms = coco_eval._per_class(gt, results, None, 'segm')
    key, _, _, _, ids = coco_eval._flatten_results(gt, boxes, segms, 'segm', cids, with_ids=True)
    assert np.array_equal(f['det_ids'].cpu().numpy(), ids)
    assert np.array_equal(f['union'].cpu().numpy(), np.union1d(np.unique(key), gt.keys))

"""Differential tests of the device COCO evaluation (detectorch_b200.utils.coco_eval) against the reference's own pycocotools
COCOeval (built by oracle/build_cocoapi.sh into oracle/_ref), on the generated cases of tests/coco_eval_fuzz_cases.py: every family
and 40 mixed seeds, 'bbox' and 'segm'.  precision, recall, scores, stats and every pair's IoU matrix are np.array_equal (float64, no
tolerance); every GT mask equals COCO.annToRLE byte for byte; a GT build split into many chunks equals the unchunked one."""
import numpy as np
import pytest
import torch

import coco_eval_cases as cc
import coco_eval_fuzz_cases as fz

pytestmark = pytest.mark.gpu
SEEDS = range(40)
COUNTS = dict(cases=0, evaluations=0, pairs=0, gt_masks=0)


@pytest.fixture(scope="module")
def oracle(built):
    """(COCO, COCOeval, mask) of the reference pycocotools and its mask.encode as a string encoder."""
    from oracle import cocoapi
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh)")
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    mods = cocoapi.load()
    mask = mods[2]
    return mods, lambda m: mask.encode(np.asfortranarray(m[:, :, None]))[0]['counts'].decode()


def _where(a, b):
    d = np.argwhere(~((a == b) | (np.isnan(a) & np.isnan(b))))
    return "first difference at %s: %r vs %r" % (tuple(d[0]), a[tuple(d[0])], b[tuple(d[0])]) if len(d) else "shapes %s %s" % (a.shape, b.shape)


def _compare(mods, case, name, gt=None):
    """Device evaluation == COCOeval for both types; -> the device ground truth."""
    from detectorch_b200.utils import coco_eval
    from oracle import ref
    ds, boxes, segms = case
    gt = coco_eval.CocoGroundTruth(ds) if gt is None else gt
    for t in ('bbox', 'segm'):
        E = cc.oracle_eval(mods, ds, boxes, segms, t)
        got = coco_eval.evaluate(gt, boxes, t, segms if t == 'segm' else None, keep_ious=True)
        for k in ('precision', 'recall', 'scores'):
            a, b = got.eval[k], E.eval[k]
            assert a.dtype == np.float64 and a.shape == b.shape and np.array_equal(a, b), (name, t, k, _where(a, b))
        assert np.array_equal(got.stats, np.array(E.stats)), (name, t, got.stats, E.stats)
        want = {(int(i), int(c)): np.asarray(v, np.float64) for (i, c), v in E.ious.items() if len(v)}
        assert set(got.ious) == set(want), (name, t, sorted(set(got.ious) ^ set(want))[:5])
        for key, v in want.items():
            assert got.ious[key].shape == v.shape and np.array_equal(got.ious[key], v), (name, t, key, _where(got.ious[key], v))
        COUNTS['evaluations'] += 1
        COUNTS['pairs'] += len(want)
        if t == 'segm':
            # _prepare has replaced every GT segmentation by COCO.annToRLE's result
            anns = E.cocoGt.anns
            for aid, counts in zip(gt.ann_ids, gt.rles()):
                want_s = E.cocoGt.annToRLE(anns[aid])['counts']
                want_s = want_s.encode() if isinstance(want_s, str) else want_s
                assert ref.rle_to_string(counts) == want_s, (name, aid)
            COUNTS['gt_masks'] += len(gt.ann_ids)
    COUNTS['cases'] += 1
    return gt


@pytest.mark.parametrize("family", list(fz.FAMILIES))
def test_family_equals_cocoeval(oracle, family):
    mods, enc = oracle
    _compare(mods, fz.make_case(family, 0, enc), family)


@pytest.mark.parametrize("seed", SEEDS)
def test_mixed_seed_equals_cocoeval(oracle, seed):
    mods, enc = oracle
    _compare(mods, fz.make_mixed_case(seed, enc), "mixed %d" % seed)


class _CountingLib:
    """The loaded library with dt_coco_gt_build calls recorded (annotations per chunk)."""

    def __init__(self, L):
        self.L, self.chunks = L, []

    def __getattr__(self, name):
        return getattr(self.L, name)

    def dt_coco_gt_build(self, n, *args):
        self.chunks.append(n)
        return self.L.dt_coco_gt_build(n, *args)


@pytest.mark.parametrize("family,budget,packs", [("poly", 1000, False), ("poly", 20000, True), ("rle_gt", 200, True)])
def test_chunked_gt_build(oracle, monkeypatch, family, budget, packs):
    """A GT build split by a small budget into many chunks gives the same masks, boxes and evaluation as the unchunked build, and as
    COCOeval.  Every chunk of several annotations fits the budget, some annotations larger than the budget get a chunk of their own,
    and with packs, chunks hold several polygons (per-annotation workspace and part offsets inside a chunk)."""
    from detectorch_b200.utils import coco_eval
    mods, enc = oracle
    case = fz.make_case(family, 1, enc)
    whole = coco_eval.CocoGroundTruth(case[0])
    lib = _CountingLib(coco_eval._lib.lib())
    with monkeypatch.context() as m:
        m.setattr(coco_eval, "_GT_BUDGET_INTS", budget)
        m.setattr(coco_eval._lib, "lib", lambda: lib)
        chunked = coco_eval.CocoGroundTruth(case[0])
    sizes, cost = lib.chunks, chunked._mask_cost
    first = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    assert len(sizes) > 5 and sum(sizes) == whole.num_gts, sizes
    assert all(cost[f:f + n].sum() <= budget for f, n in zip(first, sizes) if n > 1), sizes
    assert any(cost[f] > budget for f, n in zip(first, sizes) if n == 1), sizes
    if packs:
        kinds = [isinstance(a['segmentation'], list) for a in case[0]['annotations']]
        assert max(sizes) >= 3 and (family != "poly" or all(kinds)), sizes
    assert all(np.array_equal(a, b) for a, b in zip(chunked.rles(), whole.rles()))
    assert np.array_equal(chunked._gt_f, whole._gt_f) and np.array_equal(chunked._gt_i, whole._gt_i)
    _compare(mods, case, "chunked %s %d" % (family, budget), gt=chunked)


def test_results_runs_not_covering_mask_raise(oracle):
    """Detection strings whose runs do not sum to h * w (rleIou would never end on them) are refused before the evaluation launches.
    Their boxes miss the GT, so no run merge would start even without the check."""
    from detectorch_b200.utils import coco_eval
    from oracle import ref
    ds = dict(images=[dict(id=1, height=10, width=10)], categories=[dict(id=1)],
              annotations=[dict(id=1, image_id=1, category_id=1, bbox=[5., 5., 4., 4.], area=16., iscrowd=0,
                                segmentation=[[5., 5., 9., 5., 9., 9., 5., 9.]])])
    gt = coco_eval.CocoGroundTruth(ds)
    m = np.zeros((10, 10), np.uint8)
    m[5:9, 5:9] = 1
    good = dict(size=[10, 10], counts=ref.rle_to_string(ref.rle_encode(m)).decode())
    boxes = [[[]], [np.array([[5, 5, 8, 8, .9], [0, 3, 0, 7, .5]], np.float32)]]
    for bad in ("35", "", ref.rle_to_string([3, 5, 0, 2]).decode()):
        with pytest.raises(ValueError, match="sum to h"):
            coco_eval.evaluate(gt, boxes, 'segm', [[[]], [[good, dict(size=[10, 10], counts=bad)]]])
    E = coco_eval.evaluate(gt, boxes, 'segm', [[[]], [[good, good]]])
    assert E.stats[0] > 0


def test_report_counts(oracle):
    """What the tests above compared (run with -rP to see it)."""
    print("compared %(cases)d cases, %(evaluations)d evaluations, %(pairs)d IoU matrices, %(gt_masks)d GT masks" % COUNTS)

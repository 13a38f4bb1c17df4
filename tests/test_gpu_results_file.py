"""COCO results files read on the device (coco_eval.load_results) and evaluated: evaluate(gt, load_results(gt, file), t) against the
reference's own pycocotools (oracle/_ref) running COCOeval(G, G.loadRes(file), t).evaluate() + accumulate() on the same file --
precision, recall, scores, stats, every IoU matrix and evalImgs record np.array_equal -- and against evaluate() of the same results
held in memory.  Files: the writers' output for the golden case, every fuzz family and mixed seeds, write_results of detect_images()
and of a DeviceResults; re-serialisations and edited records; 10^6 numbers against json.loads bit for bit; refusals."""
import contextlib
import copy
import io
import json
import random
import types

import numpy as np
import pytest
import torch

import coco_eval_cases as cc
import coco_eval_fuzz_cases as fz
import results_file_cases as rc
from test_gpu_coco_eval_params import _same
from test_gpu_eval_imgs import _golden_case

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


def _file(tmp_path, data, name="res.json"):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def _cocoeval(mods, ds, path, t, params=None):
    COCO, COCOeval, _ = mods
    with contextlib.redirect_stdout(io.StringIO()):
        g = COCO()
        g.dataset = copy.deepcopy(ds)
        g.createIndex()
        E = COCOeval(g, g.loadRes(path), t)
        if params is not None:
            E.params.imgIds, E.params.catIds, E.params.useCats = params
        E.evaluate()
        E.accumulate()
        E.summarize()
    return E


def _params(gt, t, p):
    from detectorch_b200.utils import coco_eval
    if p is None:
        return None
    q = coco_eval.Params(gt, t)
    q.imgIds, q.catIds, q.useCats = list(p[0]), list(p[1]), p[2]
    return q


def _check_file(mods, tmp_path, ds, gt, data, t, params=None, what=""):
    """evaluate(load_results(file)) == COCOeval(loadRes(file)); -> the evaluation."""
    from detectorch_b200.utils import coco_eval
    path = _file(tmp_path, data)
    loaded = coco_eval.load_results(gt, path if len(data) % 2 else data)       # a path or the bytes
    got = coco_eval.evaluate(gt, loaded, t, keep_ious=True, keep_eval_imgs=True, params=_params(gt, t, params))
    _same(got, _cocoeval(mods, ds, path, t, params), (what, t, params))
    return got


def _same_eval(a, b, what):
    for k in ('precision', 'recall', 'scores'):
        assert np.array_equal(a.eval[k], b.eval[k]), (what, k)
    assert np.array_equal(a.stats, b.stats), what


def _agree(mods, tmp_path, case, what, param_sets=False):
    from detectorch_b200.utils import coco_eval
    ds, boxes, segms = case
    gt = coco_eval.CocoGroundTruth(ds)
    rng = np.random.RandomState(len(what))
    imgs, cats = list(gt.img_ids), list(gt.cat_ids)
    half = sorted(rng.permutation(imgs)[:max(1, len(imgs) // 2)].tolist())
    for t in ('bbox', 'segm'):
        recs = cc.results_file(ds, boxes, segms, t)
        data = json.dumps(recs).encode()
        got = _check_file(mods, tmp_path, ds, gt, data, t, what=what)
        mem = coco_eval.evaluate(gt, boxes, t, segms if t == 'segm' else None, keep_ious=True)
        _same_eval(got, mem, (what, t))
        if param_sets:
            for p in ((half, cats, 1), (imgs, [cats[int(rng.randint(len(cats)))]], 1), (imgs, cats, 0), (half, cats[::-1], 0)):
                _check_file(mods, tmp_path, ds, gt, data, t, p, what)


def test_golden_file(oracle, tmp_path):
    _agree(oracle[0], tmp_path, _golden_case(), "golden", param_sets=True)


@pytest.mark.parametrize("family", list(fz.FAMILIES))
def test_family_file(oracle, tmp_path, family):
    mods, enc = oracle
    _agree(mods, tmp_path, fz.make_case(family, 0, enc), family, param_sets=family in ('matching', 'rank'))


@pytest.mark.parametrize("seed", range(12))
def test_mixed_file(oracle, tmp_path, seed):
    mods, enc = oracle
    _agree(mods, tmp_path, fz.make_mixed_case(100 + seed, enc), "mixed %d" % seed)


def test_written_files(oracle, tmp_path):
    """write_results of detect_images() (synthetic-weight Mask R-CNN) and of a DeviceResults of the same detections, read back."""
    import test_gpu_device_results as tdr
    from detectorch_b200.utils import blob, coco_eval
    from oracle import network as net
    mods, _ = oracle
    model = tdr._model(net.synthetic_params("resnet50"))
    ims, results, ds, gt = tdr._model_case(model)
    acc = coco_eval.DeviceResults(gt.device)
    for idx in ([6, 2, 0], [5, 1, 3, 4]):
        data, sizes, scales, orig = blob.images_to_batch([ims[i] for i in idx], 128, 200, canvas=tdr.CANVAS)
        out = model.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
        acc.add(out, [10 * (i + 1) for i in idx], original_sizes=orig)
    for src in (results, acc):
        for t in ('bbox', 'segm'):
            path = str(tmp_path / ("w_%s.json" % t))
            coco_eval.write_results(gt, src, t, path)
            with open(path, "rb") as f:
                data = f.read()
            got = _check_file(mods, tmp_path, ds, gt, data, t, what="written")
            _same_eval(got, coco_eval.evaluate(gt, src, t), ("written", t))


def _dump(recs, fmt):
    """The json text of recs with each float written by fmt."""
    def enc(v):
        if isinstance(v, float):
            return fmt(v)
        if isinstance(v, list):
            return "[" + ", ".join(enc(x) for x in v) + "]"
        if isinstance(v, dict):
            return "{" + ", ".join(json.dumps(k) + ": " + enc(x) for k, x in v.items()) + "}"
        return json.dumps(v)
    text = enc(recs)
    assert json.loads(text) == recs
    return text.encode()


def test_format_variants(oracle, tmp_path):
    from detectorch_b200.utils import coco_eval
    mods, enc = oracle
    ds, boxes, segms = fz.make_case('matching', 1, enc)
    gt = coco_eval.CocoGroundTruth(ds)
    rng = random.Random(5)
    brecs, srecs = cc.results_file(ds, boxes, segms, 'bbox'), cc.results_file(ds, boxes, segms, 'segm')
    both = [dict(b, segmentation=s['segmentation']) for b, s in zip(brecs, srecs)]        # detectron2 / mmdetection
    for t, recs in (('bbox', brecs), ('segm', srecs), ('bbox', both), ('segm', both)):
        shuffled = recs[:]
        rng.shuffle(shuffled)
        files = rc.variants(recs, 0) + [("shuffled", json.dumps(shuffled).encode()), ("duplicates", rc.duplicate_keys(recs)),
                                        ("escaped counts", rc.escaped_counts(recs)),
                                        ("exponents", _dump(recs, lambda v: "%.17e" % v)),
                                        ("E forms", _dump(recs, lambda v: ("%.20E" % v).replace("E+", "E")))]
        ints = [dict(r, bbox=[float(round(x)) for x in r['bbox']] if 'bbox' in r else None, score=float(round(r['score'] * 4)))
                for r in recs]
        ints = [{k: v for k, v in r.items() if v is not None} for r in ints]
        files.append(("integers", json.dumps(ints).replace(".0,", ",").replace(".0]", "]").replace(".0}", "}").encode()))
        for name, data in files:
            want = ints if name == "integers" else shuffled if name == "shuffled" else recs
            strip = [{k: v for k, v in r.items() if k not in ('note', 'zz')} for r in json.loads(data)]
            assert strip == want, name
            _check_file(mods, tmp_path, ds, gt, data, t, what=name)
    # segm-only records evaluated as 'bbox': toBbox and the RLE area; with boxes on every other record (not the first)
    some = [dict(s, bbox=b['bbox']) if n % 2 else s for n, (b, s) in enumerate(zip(brecs, srecs))]
    for recs in (srecs, some):
        _check_file(mods, tmp_path, ds, gt, json.dumps(recs).encode(), 'bbox', what="segm as bbox")
    # categories the ground truth does not have: dropped, their ids still counted
    extra = brecs[:]
    for n in range(5):
        extra.insert(rng.randrange(len(extra) + 1), dict(brecs[0], category_id=999 + n))
    loaded = coco_eval.load_results(gt, json.dumps(extra).encode())
    assert loaded.num_dropped == 5 and loaded.num_records == len(extra) and loaded.branch == 'bbox'
    _check_file(mods, tmp_path, ds, gt, json.dumps(extra).encode(), 'bbox', what="unknown categories")
    _check_file(mods, tmp_path, ds, gt, json.dumps(extra).encode(), 'bbox', (list(gt.img_ids), list(gt.cat_ids), 0), "unknown, agnostic")
    # [] evaluates as no detections (loadRes raises IndexError there)
    for t in ('bbox', 'segm'):
        empty = [[[] for _ in gt.img_ids] for _ in range(len(gt.cat_ids) + 1)]
        for text in (b"[]", b" [ \r\n ] "):
            got = coco_eval.evaluate(gt, coco_eval.load_results(gt, text), t, keep_ious=True, keep_eval_imgs=True)
            _same_eval(got, coco_eval.evaluate(gt, empty, t, empty if t == 'segm' else None), "empty")


def test_numbers_bit_for_bit(dev):
    """10^6 numbers in score and bbox fields read as json.loads reads them (bits compared: -0.0 counts)."""
    from detectorch_b200.utils import coco_eval
    gt = coco_eval.CocoGroundTruth(dict(images=[dict(id=1, height=10, width=10)], categories=[dict(id=1)]))
    nums = rc.numbers(0, 10 ** 6)
    recs = ['{"image_id": 1, "category_id": 1, "bbox": [%s, %s, %s, %s], "score": %s}' % tuple(nums[i:i + 5])
            for i in range(0, len(nums), 5)]
    text = ("[" + ", ".join(recs) + "]").encode()
    want = np.array([float(v) for r in json.loads(text) for v in [r['score']] + r['bbox']], np.float64)
    loaded = coco_eval.load_results(gt, text)
    assert loaded.num_records == len(recs) and np.array_equal(loaded._det_ids.cpu().numpy(), np.arange(1, len(recs) + 1))
    got = loaded._det_f.cpu().numpy().reshape(-1)
    bad = np.flatnonzero(got.view(np.int64) != want.view(np.int64))
    assert len(bad) == 0, [(nums[i], got[i], want[i]) for i in bad[:5]]


def _gt_small():
    from detectorch_b200.utils import coco_eval
    ds = dict(images=[dict(id=1, height=4, width=5), dict(id=7, height=4, width=5)], categories=[dict(id=1), dict(id=3)],
              annotations=[dict(id=1, image_id=1, category_id=1, bbox=[0, 0, 2, 2], area=4, iscrowd=0,
                                segmentation=[[0, 0, 2, 0, 2, 2, 0, 2]])])
    return ds, coco_eval.CocoGroundTruth(ds)


def _r(**kw):
    d = {"image_id": "1", "category_id": "1", "bbox": "[1, 2, 3, 4]", "score": "0.5"}
    d.update(kw)
    return "{" + ", ".join('"%s": %s' % (k, v) for k, v in d.items() if v is not None) + "}"


def test_refusals(oracle):
    from detectorch_b200.utils import coco_eval
    _, gt = _gt_small()
    mask = oracle[0][2]
    rle = mask.encode(np.asfortranarray(np.pad(np.ones((2, 2), np.uint8), ((0, 2), (0, 3)))[:, :, None]))[0]
    good_rle = json.dumps({"size": [4, 5], "counts": rle['counts'].decode()})
    for ok in ("[" + _r() + ", " + _r(segmentation=good_rle) + "]", "[" + _r(bbox=None, segmentation=good_rle) + ", " + _r(segmentation=good_rle) + "]"):
        coco_eval.load_results(gt, ok.encode())
    texts = [rc.encode(t) for t in rc.MALFORMED + rc.NOT_ARRAY + rc.EXTRA]
    for bad in (_r(image_id="1.0"), _r(image_id='"1"'), _r(image_id="99999999999999999999"), _r(image_id="2"), _r(image_id=None),
                _r(score=None), _r(score="true"), _r(score="null"), _r(score='"0.5"'), _r(score="1e400"), _r(category_id=None),
                _r(category_id="1e0"), _r(bbox="[1, 2, 3]"), _r(bbox="[1, 2, 3, true]"), _r(bbox="[1, 2, 3, 4, 5]"), _r(bbox="null"),
                _r(bbox="[1, 2, 3, -1e400]"), _r(extra="[" * 70 + "]" * 70),
                _r(segmentation='{"size": [4, 5], "counts": [20]}'), _r(segmentation='{"size": [0, 5], "counts": "0"}'),
                _r(segmentation='{"size": [4.0, 5], "counts": "04"}'), _r(segmentation='{"size": [4, 5], "counts": "0 4"}'),
                _r(segmentation='{"size": [4, 5], "counts": "05"}'), _r(segmentation='{"size": [4, 5]}'),
                _r(segmentation='{"size": [4, 5], "counts": "0\\u00e9"}')):
        texts.append(("[" + _r() + ", " + bad + "]").encode())
    texts.append(("[" + _r(bbox=None, segmentation=good_rle) + ", " + _r(bbox=None) + "]").encode())      # segm branch, no RLE
    texts.append(("[" + _r(caption='"a cat"') + "]").encode())
    for data in texts:
        with pytest.raises(ValueError):
            coco_eval.load_results(gt, data)
    # refused by evaluate: a 'segm' evaluation of box-only records, a 'bbox' one of a segm-branch bad bbox, other inputs
    boxes_only = coco_eval.load_results(gt, ("[" + _r() + "]").encode())
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, boxes_only, 'segm')
    bad_box = coco_eval.load_results(gt, ("[" + _r(bbox=None, segmentation=good_rle) + ", " + _r(bbox="[1]", segmentation=good_rle) +
                                          "]").encode())
    coco_eval.evaluate(gt, bad_box, 'segm')
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, bad_box, 'bbox')
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, boxes_only, 'bbox', all_segms=[])
    with pytest.raises(ValueError):
        coco_eval.evaluate(gt, boxes_only, 'bbox', category_ids=[1, 3])
    with pytest.raises(ValueError):
        coco_eval.evaluate(_gt_small()[1], boxes_only, 'bbox')


def test_reference_named_functions(oracle, tmp_path):
    from detectorch_b200.utils import json_dataset_evaluator as jde
    mods, enc = oracle
    ds, boxes, segms = fz.make_case('segm_dets', 0, enc)
    jd = types.SimpleNamespace(name='coco_2014_minival', COCO=types.SimpleNamespace(dataset=ds))
    for t, fn in (('bbox', jde._do_detection_eval), ('segm', jde._do_segmentation_eval)):
        path = _file(tmp_path, json.dumps(cc.results_file(ds, boxes, segms, t)).encode(), "%s.json" % t)
        with contextlib.redirect_stdout(io.StringIO()):
            got = fn(jd, path, str(tmp_path))
        E = _cocoeval(mods, ds, path, t)
        _same_eval(got, types.SimpleNamespace(eval=E.eval, stats=np.array(E.stats)), t)

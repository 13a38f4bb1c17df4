"""The COCO results json written on the device (coco_eval.write_results, json_dataset_evaluator._write_coco_*_results_file): byte for
byte the file of the reference's results writers + json.dump, against a restatement of them (results_json_cases) always and the
reference's own writers (oracle/_ref/reflib.zip) when they are staged; float64 values printed as float.__repr__ prints them;
refused input leaves no file behind."""
import json
import os

import numpy as np
import pytest
import torch

import coco_eval_fuzz_cases as fz
import results_json_cases as rj

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "coco_eval_golden.npz")


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ref_writers():
    """The reference's _write_coco_*_results_file, or None when oracle/_ref is not staged."""
    from oracle import cython_bbox
    if not cython_bbox.available():
        return None
    return cython_bbox.load()[0]


def _write(tmp_path, gt, results, t, segms=None, cats=None, name="r.json"):
    from detectorch_b200.utils import coco_eval
    p = str(tmp_path / name)
    n = coco_eval.write_results(gt, results, t, p, segms, category_ids=cats)
    with open(p, "rb") as f:
        data = f.read()
    assert n == len(data)
    return data


def _check(tmp_path, ref_writers, ds, boxes, segms, t, cats=None):
    """write_results and _write_coco_*_results_file against the restatement and the reference's writers (all_boxes input)."""
    from detectorch_b200.utils import coco_eval, json_dataset_evaluator as jde
    gt = coco_eval.CocoGroundTruth(ds)
    cats = list(gt.category_ids if cats is None else cats)
    want = rj.reference_text(gt.img_ids, cats, boxes, segms, t)
    assert _write(tmp_path, gt, boxes, t, segms if t == 'segm' else None, cats) == want
    jd = rj.FakeJsonDataset([im['id'] for im in ds['images']], cats)
    mine, theirs = str(tmp_path / "mine.json"), str(tmp_path / "theirs.json")
    if t == 'bbox':
        jde._write_coco_bbox_results_file(jd, boxes, mine)
    else:
        jde._write_coco_segms_results_file(jd, boxes, segms, mine)
    with open(mine, "rb") as f:
        assert f.read() == want
    if ref_writers is not None:
        if t == 'bbox':
            ref_writers._write_coco_bbox_results_file(jd, boxes, theirs)
        else:
            ref_writers._write_coco_segms_results_file(jd, boxes, segms, theirs)
        with open(theirs, "rb") as f:
            assert f.read() == want


def _golden():
    z = np.load(GOLD)
    case = json.loads(z['case'].tobytes().decode())
    boxes = [[np.array(b, np.float32).reshape(-1, 5) if len(b) else [] for b in c] for c in case['all_boxes']]
    return case['dataset'], boxes, case['all_segms']


def _enc(m):
    from oracle import ref
    return ref.rle_to_string(ref.rle_encode(m)).decode()


@pytest.mark.parametrize("t", ['bbox', 'segm'])
def test_golden(dev, tmp_path, ref_writers, t):
    ds, boxes, segms = _golden()
    _check(tmp_path, ref_writers, ds, boxes, segms, t)
    # more classes in all_boxes than categories: the reference's break; a permuted, shortened category list
    cats = [c['id'] for c in ds['categories']]
    _check(tmp_path, ref_writers, ds, boxes + [boxes[1]], (segms + [segms[1]]) if t == 'segm' else None, t)
    _check(tmp_path, ref_writers, ds, boxes, segms, t, cats=cats[::-1][:max(len(cats) - 1, 1)])


@pytest.mark.parametrize("family", list(fz.FAMILIES))
def test_fuzz_families(dev, tmp_path, ref_writers, family):
    ds, boxes, segms = fz.make_case(family, 0, _enc)
    for t in ('bbox', 'segm'):
        _check(tmp_path, ref_writers, ds, boxes, segms, t)


@pytest.mark.parametrize("seed", range(12))
def test_fuzz_mixed(dev, tmp_path, ref_writers, seed):
    ds, boxes, segms = fz.make_mixed_case(seed, _enc)
    for t in ('bbox', 'segm'):
        _check(tmp_path, ref_writers, ds, boxes, segms, t)


def _float_boxes(vals):
    """One class, one image: rows (x1, y1, x1, y1, score) so that x, y and the score carry the values and w = h = 1."""
    v = np.asarray(vals, np.float64)
    n = (len(v) + 2) // 3
    v = np.concatenate([v, np.zeros(3 * n - len(v))]).reshape(n, 3)
    return np.stack([v[:, 0], v[:, 1], v[:, 0], v[:, 1], v[:, 2]], 1)


def _edge_values():
    e = [0.0, -0.0, 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, 1e-05, 0.0001, 9.999999999999999e-05, 1e-05 * (1 + 2 ** -52),
         9999999999999998.0, 1e16, 1.0000000000000002e16, 2.0 ** 53, 2.0 ** 53 + 2, 1234567890123456.8, 258.1499938964844, 0.1 + 0.2,
         1 / 3, 2 / 3, 123456789012345678.0, 4.35, 0.3]
    e += [2.0 ** p for p in range(-1074, 1024)]
    for k in range(-30, 31):
        x = float("1e%d" % k)
        e += [x, float(np.nextafter(x, 0)), float(np.nextafter(x, np.inf))]
    return np.array(e + [-x for x in e])


def test_float_repr(dev, tmp_path):
    """>= 10^6 float64 values printed as float.__repr__ (json.dumps) prints them: random bit patterns over the finite doubles,
    widened float32 values, (x2 - x1) + 1 of float32 pairs, and the edge list."""
    from detectorch_b200.utils import coco_eval
    rng = np.random.RandomState(0)
    bits = rng.randint(0, 2 ** 63, 900000, dtype=np.int64).view(np.uint64) | (rng.randint(0, 2, 900000).astype(np.uint64) << np.uint64(63))
    v = bits.view(np.float64)
    f32 = rng.randint(0, 2 ** 32, 300000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    vals = np.concatenate([v[np.isfinite(v)], f32[np.isfinite(f32)].astype(np.float64), _edge_values()])
    a = (rng.rand(200000) * 2000 - 500).astype(np.float32)
    pairs = np.stack([a, a * 0 + 1, a + (rng.rand(200000) * 700).astype(np.float32), a * 0 + 1, a], 1)
    gt = coco_eval.CocoGroundTruth({'images': [{'id': 1, 'height': 1, 'width': 1}], 'categories': [{'id': 3}]})
    for boxes in (_float_boxes(vals), pairs):
        all_boxes = [[[]], [boxes]]
        assert _write(tmp_path, gt, all_boxes, 'bbox') == rj.reference_text([1], [3], all_boxes, None, 'bbox')
    assert len(vals) + 2 * len(a) >= 10 ** 6


def test_device_results(dev, tmp_path):
    """A DeviceResults of three batches added out of id order, two dataset images never added: the bytes of the per-image results'
    file, for the dataset's, a permuted and a shortened category list; an evaluation after writing equals one before."""
    import test_gpu_device_results as tdr
    from detectorch_b200.utils import coco_eval
    gt, ds, batches, results = tdr._case(dev, seed=3)
    acc = tdr._accumulate(batches, dev)
    boxes, segms = rj.per_class(results, gt.num_images)
    before = coco_eval.evaluate(gt, acc, 'segm')
    cats = list(gt.category_ids)
    for cl in (None, cats[::-1], cats[3:11]):
        for t in ('bbox', 'segm'):
            want = rj.reference_text(gt.img_ids, cats if cl is None else cl, boxes, segms, t)
            assert _write(tmp_path, gt, acc, t, cats=cl) == want, (t, cl)
            assert _write(tmp_path, gt, results, t, cats=cl) == want, (t, cl)
            assert _write(tmp_path, gt, acc, t, cats=cl) == want, (t, cl)          # twice: the same bytes
    tdr._same_eval(coco_eval.evaluate(gt, acc, 'segm'), before)
    # an image-info gt (no annotations) will do for both types
    info = coco_eval.CocoGroundTruth(dict(images=ds['images'], categories=ds['categories']))
    assert _write(tmp_path, info, acc, 'segm') == rj.reference_text(gt.img_ids, cats, boxes, segms, 'segm')


def test_detect_images(dev, tmp_path, ref_writers):
    """detect_images output of the synthetic-weight Mask R-CNN, and the same detections as a DeviceResults."""
    import test_gpu_device_results as tdr
    from detectorch_b200.utils import blob, coco_eval
    from oracle import network as net
    model = tdr._model(net.synthetic_params("resnet50"))
    ims, results, ds, gt = tdr._model_case(model)
    boxes, segms = rj.per_class(results, gt.num_images)
    for t in ('bbox', 'segm'):
        _check(tmp_path, ref_writers, ds, boxes, segms, t)
        assert _write(tmp_path, gt, results, t) == rj.reference_text(gt.img_ids, gt.category_ids, boxes, segms, t)
    acc = coco_eval.DeviceResults()
    for idx in ([6, 2, 0], [5, 1, 3]):                  # image 4 never added
        data, sizes, scales, orig = blob.images_to_batch([ims[i] for i in idx], 128, 200, canvas=tdr.CANVAS)
        out = model.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
        acc.add(out, [10 * (i + 1) for i in idx], original_sizes=orig)
    for t in ('bbox', 'segm'):
        assert _write(tmp_path, gt, acc, t) == rj.reference_text(gt.img_ids, gt.category_ids, boxes, segms, t)


def test_rle_key_order_and_backslash(dev, tmp_path, ref_writers):
    """counts before size is written in that order; '\\' (a valid RLE char) is escaped; no detections at all is '[]'."""
    from detectorch_b200.utils import coco_eval
    from oracle import ref
    rng = np.random.RandomState(1)
    ds = dict(images=[dict(id=i, height=40, width=60) for i in (7, 3)], categories=[dict(id=c) for c in (4, 2)])
    boxes = [[[], []], [np.array([[1, 2, 30, 20, .5], [3, 4, 10, 11, .25]], np.float32), []],
             [np.array([[0, 0, 59, 39, .75]], np.float32), np.zeros((0, 5), np.float32)]]
    segms = [[[], []], [[], []], [[], []]]
    n_bs = 0
    for j, i in ((1, 0), (2, 0)):
        out = []
        for k in range(len(boxes[j][i])):
            m = np.zeros((40, 60), np.uint8)
            while True:       # a mask whose string holds a backslash (92)
                m[:] = rng.rand(40, 60) < rng.rand()
                s = ref.rle_to_string(ref.rle_encode(m)).decode()
                if '\\' in s:
                    break
            n_bs += s.count('\\')
            out.append({'counts': s, 'size': [40, 60]} if k == 0 else {'size': [40, 60], 'counts': s})
        segms[j][i] = out
    assert n_bs
    for t in ('bbox', 'segm'):
        _check(tmp_path, ref_writers, ds, boxes, segms, t)
    gt = coco_eval.CocoGroundTruth(ds)
    assert _write(tmp_path, gt, [[[], []], [[], []]], 'bbox') == b"[]"
    assert _write(tmp_path, gt, [[[], []], [[], []]], 'segm', [[[], []], [[], []]]) == b"[]"


def test_refusals_leave_no_file(dev, tmp_path):
    from detectorch_b200.utils import coco_eval
    import test_gpu_device_results as tdr
    ds = dict(images=[dict(id=1, height=10, width=10)], categories=[dict(id=5)])
    gt = coco_eval.CocoGroundTruth(ds)
    good = np.array([[1, 1, 5, 5, .5]], np.float32)
    seg = {'size': [10, 10], 'counts': '0:'}            # 0 then 10: 10 of 100 pixels
    old = tmp_path / "old.json"
    for results, t, segms in (([[[]], [np.array([[1, 1, np.nan, 5, .5]])]], 'bbox', None),
                              ([[[]], [np.array([[1, 1, 5, 5, np.inf]])]], 'bbox', None),
                              ([[[]], [good[:, :4]]], 'bbox', None),
                              ([[[]], [good]], 'segm', [[[]], [[seg]]]),                         # counts do not cover h * w
                              ([[[]], [good]], 'segm', [[[]], [[{'size': [10, 10], 'counts': 'L9', 'x': 1}]]]),
                              ([[[]], [good]], 'segm', [[[]], [[{'size': [10, 10], 'counts': b'L9'}]]]),
                              ([[[]], [good]], 'segm', [[[]], [[{'size': [10, True], 'counts': 'L9'}]]])):
        for p in (tmp_path / "new.json", old):
            old.write_bytes(b"keep")
            with pytest.raises(ValueError):
                coco_eval.write_results(gt, results, t, str(p), segms)
        assert not (tmp_path / "new.json").exists() and old.read_bytes() == b"keep"
    # a DeviceResults image that is not an image of gt
    g2, _, batches, _ = tdr._case(dev, seed=4)
    acc = tdr._accumulate(batches, dev)
    with pytest.raises(ValueError):
        coco_eval.write_results(gt, acc, 'bbox', str(old))
    assert old.read_bytes() == b"keep" and sorted(os.listdir(tmp_path)) == ["old.json"]

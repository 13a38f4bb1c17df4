"""Device-resident COCO results (utils.coco_eval.DeviceResults): detect() batches accumulated on the device and evaluated without a
host-side conversion.  The device tables must equal _flatten_results + _pair_tables of the same data through batch_results, and every
evaluation must equal evaluate() on the per-image results, np.array_equal throughout."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NC = 25                                        # contiguous classes 0..24 of the synthetic detections
CATS = [7, 3, 11, 5, 2, 9, 13, 1, 4, 6, 8, 10, 12, 14, 15, 16, 17, 18, 19, 20]     # json category ids, in dataset order


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _sizes(rng, n):
    return [(int(rng.randint(40, 90)), int(rng.randint(40, 100))) for _ in range(n)]


def _batch(rng, hw, cap, counts, dev, with_masks=True):
    """A detect()-shaped output: boxes [B,cap,4] inside each image, scores on a coarse grid (ties across images), int32 classes in
    1..NC-1 grouped by class, counts as given, masks [B,cap,28,28]; dead slots hold garbage, as the engine's buffers may."""
    B = len(hw)
    boxes = np.zeros((B, cap, 4), np.float32)
    for b, (h, w) in enumerate(hw):
        x1, y1 = rng.uniform(0, w - 8, cap), rng.uniform(0, h - 8, cap)
        boxes[b] = np.stack([x1, y1, np.minimum(x1 + rng.uniform(2, 40, cap), w - 1), np.minimum(y1 + rng.uniform(2, 40, cap), h - 1)], 1)
    scores = (rng.randint(1, 9, (B, cap)) / 8.0).astype(np.float32)
    classes = np.sort(rng.randint(1, NC, (B, cap)), 1).astype(np.int32)
    out = {"boxes": torch.from_numpy(boxes).to(dev), "scores": torch.from_numpy(scores).to(dev), "classes": torch.from_numpy(classes).to(dev),
           "counts": torch.tensor(counts, dtype=torch.int32, device=dev)}
    if with_masks:
        out["masks"] = torch.from_numpy(rng.rand(B, cap, 28, 28).astype(np.float32)).to(dev)
    return out


def _ground_truth(rng, ids, hw, with_masks=True, near=()):
    """Random annotations per image, plus one jittered copy of each (image id, category id, x1, y1, x2, y2) in `near`."""
    from detectorch_b200.utils import coco_eval
    images = [dict(id=i, height=h, width=w) for i, (h, w) in zip(ids, hw)]
    boxes = []
    for i, (h, w) in zip(ids, hw):
        for _ in range(rng.randint(0, 9)):
            x, y = rng.uniform(0, w - 10), rng.uniform(0, h - 10)
            boxes.append((i, int(rng.choice(CATS[:12])), x, y, rng.uniform(3, 40), rng.uniform(3, 40)))
    for i, c, x1, y1, x2, y2 in near:
        boxes.append((i, c, x1 + rng.uniform(-2, 2), y1 + rng.uniform(-2, 2), x2 - x1 + rng.uniform(-2, 2), y2 - y1 + rng.uniform(-2, 2)))
    anns = []
    for i, c, x, y, bw, bh in boxes:
        a = dict(id=len(anns) + 1, image_id=i, category_id=c, bbox=[x, y, bw, bh], area=max(bw * bh, 0.), iscrowd=int(rng.rand() < .1))
        if with_masks:
            a["segmentation"] = [[x, y, x + bw, y, x + bw, y + bh, x, y + bh]]
        anns.append(a)
    ds = dict(images=images, annotations=anns, categories=[dict(id=c, name="c%d" % c) for c in CATS])
    return ds, coco_eval.CocoGroundTruth(ds)


def _empty(nc=NC):
    return (np.zeros(0, np.float32), np.zeros((0, 4), np.float32), [[]] + [np.zeros((0, 5), np.float32) for _ in range(1, nc)],
            [[] for _ in range(nc)])


def _case(dev, seed=0, with_masks=True):
    """Three batches over 14 of 16 images (two never added), added out of id order; -> (gt, ds, batches, per-image results)."""
    from detectorch_b200.utils import result_utils
    rng = np.random.RandomState(seed)
    ids = [int(v) for v in rng.permutation(np.arange(100, 116)) * 3]
    hw = _sizes(rng, 16)
    order = rng.permutation(16)[:14]
    cap = 12
    batches, near = [], []
    for part, counts in ((order[:5], [0, 12, 5, 9, 1]), (order[5:9], [12, 3, 7, 12]), (order[9:], [4, 0, 12, 6, 11])):
        sz = [hw[p] for p in part]
        out = _batch(rng, sz, cap, counts, dev, with_masks)
        orig = np.array([[h + .75, w + .5] for h, w in sz])          # int() of each value is the RLE canvas
        batches.append((out, [ids[p] for p in part], orig))
        bx, cl = out["boxes"].cpu().numpy(), out["classes"].cpu().numpy()
        for b, p in enumerate(part):
            for d in range(0, counts[b], 2):
                if cl[b, d] <= len(CATS):
                    near.append((ids[p], CATS[cl[b, d] - 1]) + tuple(float(v) for v in bx[b, d]))
    ds, gt = _ground_truth(rng, ids, hw, with_masks, near)
    results = [None] * 16
    idx = {v: n for n, v in enumerate(gt.img_ids)}
    for out, bids, orig in batches:
        for r, v in zip(result_utils.batch_results(out, orig, num_classes=NC), bids):
            results[idx[v]] = r if with_masks else (r[0], r[1], r[2], [[] for _ in range(NC)])
    results = [r if r is not None else _empty() for r in results]
    return gt, ds, batches, results


def _accumulate(batches, dev, **kw):
    from detectorch_b200.utils import coco_eval
    acc = coco_eval.DeviceResults(dev)
    for k, v in kw.items():
        setattr(acc, k, v)
    for out, ids, orig in batches:
        acc.add(out, ids, original_sizes=orig, num_classes=NC)
    return acc


def _same_eval(a, b):
    for k in ('precision', 'recall', 'scores'):
        assert np.array_equal(a.eval[k], b.eval[k]), k
    assert np.array_equal(a.stats, b.stats)


@pytest.mark.parametrize("category_ids", [None, CATS[::-1], CATS[:9]], ids=["dataset", "permuted", "shortened"])
def test_tables_equal_host_flattening(dev, category_ids):
    from detectorch_b200.utils import coco_eval
    gt, _, batches, results = _case(dev)
    acc = _accumulate(batches, dev)
    cids = list(gt.category_ids if category_ids is None else category_ids)
    for t in ('bbox', 'segm'):
        boxes, segms = coco_eval._per_class(gt, results, None, t)
        key, det_f, det_i, chars = coco_eval._flatten_results(gt, boxes, segms, t, cids)
        pairs, cat_kept, order_off = coco_eval._pair_tables(gt, key)
        f = coco_eval._flatten_device(gt, acc, t, cids)
        assert len(key) > 30 and len(pairs) > 10
        assert np.array_equal(f['key'].cpu().numpy(), key), t
        assert np.array_equal(f['det_f'].cpu().numpy(), det_f), t
        assert np.array_equal(f['pairs'].cpu().numpy(), pairs), t
        assert np.array_equal(f['cat_kept'].cpu().numpy(), cat_kept), t
        assert np.array_equal(f['order_off'].cpu().numpy(), order_off), t
        assert f['num_order'] == order_off[-1, -1] and f['num_kept'] == cat_kept[-1]
        if t == 'segm':
            di = f['det_i'].cpu().numpy()
            assert np.array_equal(di[:, 1:], det_i[:, 1:])
            buf = f['chars'][:f['num_chars']].cpu().numpy().tobytes()
            for (o, n, _, _), (oh, _, _, _) in zip(di, det_i):
                assert buf[o:o + n] == chars[oh:oh + n]
    # score ties across images within one category are present, so the stable order is exercised
    s = det_f[:, 0]
    cat = key // gt.num_images
    assert any(len(np.unique(s[cat == c])) < np.sum(cat == c) and len(np.unique(key[cat == c])) > 1 for c in np.unique(cat))


@pytest.mark.parametrize("category_ids", [None, CATS[::-1], CATS[:9]], ids=["dataset", "permuted", "shortened"])
def test_evaluation_equals_per_image_results(dev, category_ids):
    from detectorch_b200.utils import coco_eval
    gt, _, batches, results = _case(dev, seed=1)
    acc = _accumulate(batches, dev)
    for t in ('bbox', 'segm', 'bbox'):                     # evaluated several times, for either type
        want = coco_eval.evaluate(gt, results, t, category_ids=category_ids, keep_ious=True)
        got = coco_eval.evaluate(gt, acc, t, category_ids=category_ids, keep_ious=True)
        _same_eval(got, want)
        assert got.ious.keys() == want.ious.keys() and (category_ids is not None or want.stats[0] > 0)
        for k in want.ious:
            assert np.array_equal(got.ious[k], want.ious[k]), (t, k)


def test_add_after_evaluate_and_growth(dev):
    """Many one-image adds with tiny initial buffers equal one add per batch; adding after an evaluation is allowed."""
    from detectorch_b200.utils import coco_eval
    gt, _, batches, results = _case(dev, seed=2)
    big = _accumulate(batches, dev)
    small = coco_eval.DeviceResults(dev)
    small._MIN_RECORDS, small._MIN_CHARS = 1, 1
    first = True
    for out, ids, orig in batches:
        for b in range(len(ids)):
            one = {k: v[b:b + 1] for k, v in out.items()}
            small.add(one, [ids[b]], original_sizes=orig[b:b + 1], num_classes=NC)
            if first:
                coco_eval.evaluate(gt, small, 'segm')
                first = False
    assert small._rec_f.shape[0] < 2 * small._num_records and small._chars.shape[0] < 2 * small._num_chars
    for t in ('bbox', 'segm'):
        _same_eval(coco_eval.evaluate(gt, small, t), coco_eval.evaluate(gt, big, t))
        _same_eval(coco_eval.evaluate(gt, small, t), coco_eval.evaluate(gt, results, t))


def test_bbox_add_does_not_synchronise(dev):
    from detectorch_b200.utils import coco_eval
    gt, _, batches, results = _case(dev, seed=3, with_masks=False)
    acc = coco_eval.DeviceResults(dev)
    acc._MIN_RECORDS = 8                                    # the buffers grow inside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for out, ids, orig in batches:
            acc.add(out, ids, original_sizes=orig, num_classes=NC)
        acc2 = coco_eval.DeviceResults(dev)
        for out, ids, _ in batches:
            acc2.add(out, ids, num_classes=NC)              # original_sizes is optional without masks
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _same_eval(coco_eval.evaluate(gt, acc, 'bbox'), coco_eval.evaluate(gt, results, 'bbox'))
    _same_eval(coco_eval.evaluate(gt, acc2, 'bbox'), coco_eval.evaluate(gt, results, 'bbox'))


class _Spy:
    """Records the C-ABI entry points called through _lib.lib()."""

    def __init__(self, L):
        self.L, self.calls = L, []

    def __getattr__(self, name):
        f = getattr(self.L, name)
        if not name.startswith("dt_") or name.endswith("_bytes"):
            return f

        def call(*a):
            self.calls.append(name)
            return f(*a)
        return call


def test_errors(dev, monkeypatch):
    from detectorch_b200 import _lib
    from detectorch_b200.utils import coco_eval
    gt, ds, batches, _ = _case(dev, seed=4)
    out, ids, orig = batches[1]
    spy = _Spy(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: spy)
    acc = coco_eval.DeviceResults(dev)
    with pytest.raises(ValueError, match="repeated"):
        acc.add(out, [ids[0]] * len(ids), original_sizes=orig, num_classes=NC)
    acc.add(out, ids, original_sizes=orig, num_classes=NC)
    with pytest.raises(ValueError, match="already added"):
        acc.add(batches[2][0], [batches[2][1][0]] + ids[:1] + batches[2][1][2:], original_sizes=batches[2][2], num_classes=NC)
    with pytest.raises(ValueError, match="original_sizes"):
        acc.add(batches[2][0], batches[2][1], num_classes=NC)
    with pytest.raises(ValueError, match="image id"):
        acc.add(batches[2][0], [1.5] * len(batches[2][1]), original_sizes=batches[2][2], num_classes=NC)
    with pytest.raises(ValueError, match="tensors on"):
        acc.add({k: v.cpu() for k, v in batches[2][0].items()}, batches[2][1], original_sizes=batches[2][2], num_classes=NC)
    assert acc.image_ids == ids                            # failed adds leave the accumulator as it was
    spy.calls.clear()

    def refused(exc, match, *a, **kw):
        n = len(spy.calls)
        with pytest.raises(exc, match=match):
            coco_eval.evaluate(*a, **kw)
        return spy.calls[n:]

    # host-side checks: nothing is launched
    bad = coco_eval.DeviceResults(dev)
    bad.add(out, [10 ** 6] + ids[1:], original_sizes=orig, num_classes=NC)
    assert refused(ValueError, "not an image", gt, bad, 'bbox') == []
    bbox_only = coco_eval.DeviceResults(dev)
    bbox_only.add({k: v for k, v in out.items() if k != "masks"}, ids, num_classes=NC)
    assert refused(ValueError, "without masks", gt, bbox_only, 'segm') == []
    assert refused(ValueError, "all_segms", gt, acc, 'segm', all_segms=[[]]) == []
    gt_cpu = coco_eval.CocoGroundTruth(dict(ds, annotations=[{k: v for k, v in a.items() if k != "segmentation"} for a in ds["annotations"]]),
                                       device="cpu")
    assert refused(ValueError, "ground truth on", gt_cpu, acc, 'bbox') == []
    # device-side flags: read back with the sizes; nothing is flattened or evaluated
    def nan_score(o):
        o["classes"][1, 0] = 1                          # a class with a category: its record is evaluated
        o["scores"][1, 0] = float("nan")

    for mutate, exc, match in ((nan_score, ValueError, "non-finite"),
                               (lambda o: o["classes"][1, :3].copy_(torch.tensor([5, 3, 5], dtype=torch.int32)), RuntimeError, "not grouped"),
                               (lambda o: o["classes"][1, 0].fill_(NC), RuntimeError, "not grouped")):
        o = {k: v.clone() for k, v in out.items()}
        o["counts"][1] = 12
        mutate(o)
        a = coco_eval.DeviceResults(dev)
        a.add(o, ids, original_sizes=orig, num_classes=NC)
        for t in ('bbox', 'segm'):
            calls = refused(exc, match, gt, a, t)
            assert calls == ["dt_coco_results_count"], calls


def test_json_dataset_evaluator_wrappers(dev):
    from detectorch_b200.utils import coco_eval
    from detectorch_b200.utils import json_dataset_evaluator as jde
    gt, ds, batches, results = _case(dev, seed=5)
    acc = _accumulate(batches, dev)

    class _Coco:
        dataset = ds

    class _JsonDataset:
        name = 'coco_2014_minival'
        COCO = _Coco()
        classes = ['__background__'] + [c['name'] for c in ds['categories']]
        category_to_id_map = {c['name']: c['id'] for c in ds['categories']}

    jd = _JsonDataset()
    _same_eval(jde.evaluate_boxes(jd, acc, "/nonexistent-output-dir"), coco_eval.evaluate(gt, results, 'bbox'))
    _same_eval(jde.evaluate_masks(jd, acc, None, "/nonexistent-output-dir"), coco_eval.evaluate(gt, results, 'segm'))


def _model(params):
    from detectorch_b200.model.detector import detector
    model = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                     conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                     roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                     use_rpn_head=True, use_mask_head=True, mask_head_type='1up4convs')
    sd = model.state_dict()
    for k, v in params.items():
        if k in sd:
            sd[k].copy_(v)
    return model.cuda()


@pytest.fixture(scope="module")
def mask_rcnn(dev):
    from oracle import network as net
    return _model(net.synthetic_params("resnet50"))


CANVAS = (224, 224)


def _model_case(model, n=7, seed=5):
    """Ragged images, their detect_images results (never-added image 4 emptied), a GT built around the detections, json ids 10 (i + 1)."""
    from detectorch_b200.utils import coco_eval
    rng = np.random.RandomState(seed)
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(60, 80), (90, 50), (64, 64), (41, 97), (77, 70), (58, 66), (70, 90)][:n]]
    results = model.detect_images(ims, target_size=128, max_size=200, canvas=CANVAS)
    assert sum(len(r[0]) for r in results) > 0
    results[4] = _empty(81)
    anns = []
    for i, r in enumerate(results):
        for j in range(1, 81):
            for b in np.asarray(r[2][j]).reshape(-1, 5)[:3]:
                x, y = float(b[0]) + rng.uniform(-3, 3), float(b[1]) + rng.uniform(-3, 3)
                w, h = float(b[2] - b[0]) + rng.uniform(-3, 3), float(b[3] - b[1]) + rng.uniform(-3, 3)
                anns.append(dict(id=len(anns) + 1, image_id=10 * (i + 1), category_id=81 - j, bbox=[x, y, w, h], area=max(w * h, 0.),
                                 iscrowd=int(rng.rand() < .1), segmentation=[[x, y, x + w, y, x + w / 2, y + h, x, y + h]]))
    images = [dict(id=10 * (i + 1), height=im.shape[0], width=im.shape[1]) for i, im in enumerate(ims)]
    ds = dict(images=images, annotations=anns, categories=[dict(id=c, name="c%d" % c) for c in range(80, 0, -1)])
    return ims, results, ds, coco_eval.CocoGroundTruth(ds)


def test_detect_equals_cocoeval(dev, mask_rcnn):
    """Two detect() batches of the synthetic-weight Mask R-CNN on ragged images, added out of order, one image never added: equal to
    live COCOeval on the notebook's results file and to evaluate() of detect_images' results."""
    import coco_eval_cases as cc
    from detectorch_b200.utils import blob, coco_eval
    from oracle import cocoapi
    ims, results, ds, gt = _model_case(mask_rcnn)
    acc = coco_eval.DeviceResults()
    for part in ([5, 2, 0], [6, 3, 1]):
        data, sizes, scales, orig = blob.images_to_batch([ims[p] for p in part], 128, 200, canvas=CANVAS)
        out = mask_rcnn.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
        acc.add(out, [10 * (p + 1) for p in part], original_sizes=orig)
    all_boxes = [[[] for _ in ims]] + [[r[2][j] for r in results] for j in range(1, 81)]
    all_segms = [[[] for _ in ims]] + [[r[3][j] for r in results] for j in range(1, 81)]
    have_oracle = cocoapi.available()
    mods = cocoapi.load() if have_oracle else None
    for t in ('bbox', 'segm'):
        got = coco_eval.evaluate(gt, acc, t)
        _same_eval(got, coco_eval.evaluate(gt, results, t))
        assert got.stats[0] > 0, t
        if have_oracle:
            E = cc.oracle_eval(mods, ds, all_boxes, all_segms, t)
            for k in ('precision', 'recall', 'scores'):
                assert np.array_equal(got.eval[k], E.eval[k]), (t, k)
            assert np.array_equal(got.stats, np.array(E.stats)), t
    if not have_oracle:
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh): compared with evaluate() of detect_images only")


def test_host_input_back_to_back(dev, mask_rcnn):
    """Pinned-host detect() calls back to back (the third and later replay a captured graph), each followed by add with no
    synchronisation, evaluate as device input with a synchronisation after each call."""
    from detectorch_b200.utils import blob, coco_eval
    ims, results, ds, gt = _model_case(mask_rcnn)
    parts = [[0, 1], [2, 3], [5, 6], [1, 0]]
    staged = []
    for part in parts:
        data, sizes, scales, orig = blob.images_to_batch([ims[p] for p in part], 128, 200, canvas=CANVAS)
        staged.append((data, data.cpu().pin_memory(), sizes, scales, orig, part))
    for with_masks in (False, True):
        eager = coco_eval.DeviceResults()
        host = coco_eval.DeviceResults()
        for n, (data, _, sizes, scales, orig, part) in enumerate(staged):
            out = mask_rcnn.detect(data, scaling_factor=scales, image_sizes=sizes, original_sizes=orig, with_masks=with_masks)
            torch.cuda.synchronize()
            eager.add(out, [10 * (p + 1) + 1000 * n for p in part], original_sizes=orig)
        for n, (_, pinned, sizes, scales, orig, part) in enumerate(staged):
            out = mask_rcnn.detect(pinned, scaling_factor=scales, image_sizes=sizes, original_sizes=orig, with_masks=with_masks)
            host.add(out, [10 * (p + 1) + 1000 * n for p in part], original_sizes=orig)
        ds2 = dict(ds, images=[dict(im, id=im['id'] + 1000 * n) for n in range(len(parts)) for im in ds['images']],
                   annotations=[dict(a, id=a['id'] + 100000 * n, image_id=a['image_id'] + 1000 * n) for n in range(len(parts)) for a in ds['annotations']])
        gt2 = coco_eval.CocoGroundTruth(ds2)
        for t in (('bbox', 'segm') if with_masks else ('bbox',)):
            a, b = coco_eval.evaluate(gt2, host, t), coco_eval.evaluate(gt2, eager, t)
            _same_eval(a, b)
            assert a.stats[0] > 0

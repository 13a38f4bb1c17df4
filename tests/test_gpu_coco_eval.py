"""COCO evaluation on the device (detectorch_b200.utils.coco_eval): bit-identical to the reference's pycocotools COCOeval.
Golden arrays (tests/golden/make_coco_eval_golden.py) are compared with np.array_equal, float64, no tolerance; GT polygon masks
byte for byte with COCO.annToRLE; detect_images output of the synthetic-weight Mask R-CNN against COCOeval run live (oracle/_ref)."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "coco_eval_golden.npz")


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLD)
    case = json.loads(z['case'].tobytes().decode())
    boxes = [[np.array(b, np.float32).reshape(-1, 5) if len(b) else [] for b in c] for c in case['all_boxes']]
    return z, case['dataset'], boxes, case['all_segms']


def test_golden_bit_identical(dev, golden):
    from detectorch_b200.utils import coco_eval
    z, ds, boxes, segms = golden
    gt = coco_eval.CocoGroundTruth(ds)
    for t in ('bbox', 'segm'):
        E = coco_eval.evaluate(gt, boxes, t, segms if t == 'segm' else None, keep_ious=True)
        for k in ('precision', 'recall', 'scores'):
            assert E.eval[k].dtype == np.float64 and np.array_equal(E.eval[k], z[t + '_' + k]), (t, k)
        assert np.array_equal(E.stats, z[t + '_stats']), t
        o = 0
        for key, shape in zip(z[t + '_iou_keys'], z[t + '_iou_shapes']):
            n = int(shape[0] * shape[1])
            assert np.array_equal(E.ious[tuple(int(v) for v in key)], z[t + '_iou_values'][o:o + n].reshape(shape)), (t, key)
            o += n


def test_gt_masks_equal_ann_to_rle(dev, golden):
    from detectorch_b200.utils import coco_eval
    from oracle import ref
    z, ds, _, _ = golden
    want = json.loads(z['gt_rles'].tobytes().decode())
    gt = coco_eval.CocoGroundTruth(ds)
    got = gt.rles()
    assert len(got) == len(want)
    for aid, counts in zip(gt.ann_ids, got):
        assert ref.rle_to_string(counts) == want[str(aid)].encode(), aid


def test_ground_truth_reused_across_evaluations(dev, golden):
    from detectorch_b200.utils import coco_eval
    z, ds, boxes, segms = golden
    gt = coco_eval.CocoGroundTruth(ds)
    a = coco_eval.evaluate(gt, boxes, 'segm', segms)
    coco_eval.evaluate(gt, boxes, 'bbox')
    b = coco_eval.evaluate(gt, boxes, 'segm', segms)
    assert np.array_equal(a.eval['precision'], b.eval['precision']) and np.array_equal(a.stats, z['segm_stats'])


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


def test_detect_images_equals_cocoeval(dev):
    """detect_images of the synthetic-weight Mask R-CNN, evaluated on the device, equals COCOeval on the notebook's results file."""
    import coco_eval_cases as cc
    from detectorch_b200.utils import coco_eval
    from oracle import cocoapi
    from oracle import network as net
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh)")
    mods = cocoapi.load()
    rng = np.random.RandomState(5)
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(60, 80), (90, 50), (64, 64), (41, 97), (77, 70), (58, 66)]]
    results = _model(net.synthetic_params("resnet50")).detect_images(ims, target_size=128, max_size=200)
    assert sum(len(r[0]) for r in results) > 0
    cat_ids = list(range(80, 0, -1))                  # contiguous class j is json category 81 - j
    images = [dict(id=10 * (i + 1), height=im.shape[0], width=im.shape[1]) for i, im in enumerate(ims)]
    anns = []
    for i, r in enumerate(results):
        if i == 4:
            continue                                    # an image whose detections are all false positives
        for j in range(1, 81):
            for b in np.asarray(r[2][j]).reshape(-1, 5)[:3]:
                x, y = float(b[0]) + rng.uniform(-3, 3), float(b[1]) + rng.uniform(-3, 3)
                w, h = float(b[2] - b[0]) + rng.uniform(-3, 3), float(b[3] - b[1]) + rng.uniform(-3, 3)
                anns.append(dict(id=len(anns) + 1, image_id=10 * (i + 1), category_id=81 - j, bbox=[x, y, w, h], area=max(w * h, 0.),
                                 iscrowd=int(rng.rand() < .1), segmentation=[[x, y, x + w, y, x + w / 2, y + h, x, y + h]]))
    ds = dict(images=images, annotations=anns, categories=[dict(id=c, name="c%d" % c) for c in cat_ids])
    gt = coco_eval.CocoGroundTruth(ds)
    all_boxes = [[[] for _ in ims]] + [[r[2][j] for r in results] for j in range(1, 81)]
    all_segms = [[[] for _ in ims]] + [[r[3][j] for r in results] for j in range(1, 81)]
    for t in ('bbox', 'segm'):
        E = cc.oracle_eval(mods, ds, all_boxes, all_segms, t)
        got = coco_eval.evaluate(gt, results, t)
        for k in ('precision', 'recall', 'scores'):
            assert np.array_equal(got.eval[k], E.eval[k]), (t, k)
        assert np.array_equal(got.stats, np.array(E.stats)), t
        assert E.stats[0] > 0, t


def test_json_dataset_evaluator(dev, golden):
    """evaluate_boxes / evaluate_masks with the reference's signatures: JsonDataset-like object in, the same numbers out, no file."""
    from detectorch_b200.utils import json_dataset_evaluator as jde
    z, ds, boxes, segms = golden

    class _Coco:
        dataset = ds

    class _JsonDataset:
        name = 'coco_2014_minival'
        COCO = _Coco()
        classes = ['__background__'] + [c['name'] for c in ds['categories']]
        category_to_id_map = {c['name']: c['id'] for c in ds['categories']}

    out = "/nonexistent-output-dir"
    jd = _JsonDataset()
    E = jde.evaluate_boxes(jd, boxes, out, use_salt=True, cleanup=False)
    assert np.array_equal(E.eval['precision'], z['bbox_precision']) and np.array_equal(E.stats, z['bbox_stats'])
    E = jde.evaluate_masks(jd, boxes, segms, out)
    assert np.array_equal(E.eval['precision'], z['segm_precision']) and np.array_equal(E.stats, z['segm_stats'])
    jd.name = 'coco_2015_test'
    assert jde.evaluate_boxes(jd, boxes, out) is None

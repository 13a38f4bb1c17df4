"""Proposal recall on the device (utils.coco_eval.box_proposal_recall, json_dataset_evaluator.evaluate_box_proposals) against the
reference's own evaluate_box_proposals on its compiled bbox_overlaps -- the committed golden file and live random roidbs, compared with
np.array_equal -- and batched RPN proposals (detector.propose_images, dt_engine_proposals) against batch-1 forward()."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

import proposal_recall_cases as cases

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "proposal_recall_golden.npz")
DETECTRON = [(a, l) for a in ('all', 'small', 'medium', 'large') for l in (100, 1000)]


def _same(got, want):
    # a combination without positives divides 0 by 0, in the reference too
    assert np.array_equal(got['recalls'], want['recalls'], equal_nan=True)
    assert np.array_equal(got['gt_overlaps'], want['gt_overlaps'])
    assert np.array_equal(np.float64(got['ar']), np.float64(want['ar']), equal_nan=True)
    assert got['num_pos'] == want['num_pos']


def _oracle():
    from oracle import cython_bbox
    if not cython_bbox.available():
        pytest.skip("oracle/_ref cython_bbox / reflib.zip not built (oracle/build_cython_bbox.sh needs the reference tree once)")
    return cython_bbox.load()


def test_golden(built):
    from detectorch_b200.utils import json_dataset_evaluator as jde
    g = np.load(GOLDEN)
    names = list(g["names"])
    assert len(names) == len(cases.edge_cases())
    for name, roidb, area, limit, thr in cases.edge_cases():
        got = jde.evaluate_box_proposals(None, roidb, thresholds=thr, area=area, limit=limit)
        want = {k: g["%s/%s" % (name, k)] for k in ('recalls', 'gt_overlaps', 'ar', 'num_pos')}
        want['num_pos'] = int(want['num_pos'])
        _same(got, want)
        assert np.array_equal(np.asarray(got['thresholds']), g["%s/thresholds" % name]), name


def test_random_roidbs_against_oracle(built):
    from detectorch_b200.utils import coco_eval
    ref, _ = _oracle()
    for seed in range(6):
        roidb = cases.random_roidb(seed)
        got = coco_eval.box_proposal_recall(roidb, areas=list(coco_eval.PROPOSAL_AREAS), limits=(None, 0, 7, 100, 1000))
        for (area, limit), r in got.items():
            _same(r, ref.evaluate_box_proposals(None, roidb, area=area, limit=limit))
    # Detectron's 8 combinations in one launch equal 8 single ones
    roidb = cases.random_roidb(99, 60)
    all8 = coco_eval.box_proposal_recall(roidb)
    assert sorted(all8) == sorted(DETECTRON)
    for key in DETECTRON:
        _same(all8[key], ref.evaluate_box_proposals(None, roidb, area=key[0], limit=key[1]))


def _model(params):
    from detectorch_b200.model.detector import detector
    model = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                     conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                     roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                     use_rpn_head=True, use_mask_head=False)
    sd = model.state_dict()
    for k, v in params.items():
        if k in sd:
            sd[k].copy_(v)
    return model.cuda()


@pytest.fixture(scope="module")
def params(built):
    from oracle import network as net
    return net.synthetic_params("resnet50", mask=False)


def _uint8_images():
    rng = np.random.RandomState(5)
    return [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(60, 80), (90, 50), (64, 64), (41, 97), (77, 70)]]


def _forward_proposals(model, im):
    """Batch-1 forward() RoIs divided by the image's scale (fp32, as postprocess_output divides them)."""
    from detectorch_b200.utils import blob
    data, s = blob.image_to_blob(im, target_size=128, max_size=200, fpn_on=True)
    rois = model(data, scaling_factor=s)[2].cpu().numpy()
    return rois / np.float32(s)


@pytest.mark.parametrize("conv_kind", ["f16", "tf32"])
def test_propose_images_equals_forward(params, monkeypatch, conv_kind):
    monkeypatch.setenv("DT_CONV_KIND", conv_kind)
    model = _model(params)
    ims = _uint8_images()
    total = 0
    for call in range(3):                 # eager, then captured, then replayed
        got = model.propose_images(ims, target_size=128, max_size=200, canvas=(224, 224))
        assert len(got) == len(ims)
        for b, im in enumerate(ims):
            boxes, scores = got[b]
            want = _forward_proposals(model, im)
            assert boxes.dtype == np.float32 and scores.dtype == np.float32
            assert np.array_equal(boxes, want), (conv_kind, call, b)
            assert scores.shape == (len(boxes),) and np.all(np.diff(scores) <= 0) and np.all(scores > 0)
            total += len(boxes)
    assert total > 0
    assert model.engine_for(len(ims), 224, 224)._proposal_state["graph"] is not None


def test_engine_proposals_on_nan_canvas(params):
    """dt_engine_proposals on a NaN-padded ragged canvas: every image's boxes equal its batch-1 rois / scale, its scores the collect's."""
    from detectorch_b200.engine import Engine, ST_COLLECT, ST_TRUNK
    from oracle import network as net
    dev = torch.device("cuda:0")
    canvas, sizes, scales = (192, 256), [(192, 256), (128, 160), (192, 128), (96, 224)], [1.0, 0.8, 1.25, 0.6]
    crops = [net.synthetic_image(1, h, w, seed=b) for b, (h, w) in enumerate(sizes)]
    img = torch.full((len(sizes), 3) + canvas, float("nan"))
    for b, (h, w) in enumerate(sizes):
        img[b, :, :h, :w] = crops[b][0]
    eng = Engine(batch=len(sizes), height=canvas[0], width=canvas[1], use_mask=False, det_cap=128)
    eng.load_state_dict(params)
    eng.set_image_info(sizes, scales)
    eng.run(img.to(dev), 1.0, ST_TRUNK, ST_COLLECT)
    R = eng.cfg.post_nms_top_n
    boxes = torch.full((len(sizes), R, 4), 7.0, device=dev)
    scores = torch.full((len(sizes), R), 7.0, device=dev)
    eng.proposals(boxes, scores)
    torch.cuda.synchronize()
    for b, (h, w) in enumerate(sizes):
        ref = Engine(batch=1, height=h, width=w, use_mask=False, det_cap=128, share_weights_with=eng)
        ref.run(crops[b].to(dev), scales[b], ST_TRUNK, ST_COLLECT)
        torch.cuda.synchronize()
        n = int(ref.buffer("roi_counts")[0])
        assert n > 0 and int(eng.buffer("roi_counts")[b]) == n
        want = ref.buffer("rois")[0, :n, 1:5].cpu().numpy() / np.float32(scales[b])
        assert np.array_equal(boxes[b, :n].cpu().numpy(), want), b
        assert int(torch.count_nonzero(boxes[b, n:])) == 0 and int(torch.count_nonzero(scores[b, n:])) == 0
        # the scores are the collected proposals' RPN scores: each one is in its level's prop_scores, sorted descending
        sc = scores[b, :n].cpu().numpy()
        pool = ref.buffer("prop_scores")[0].cpu().numpy().reshape(-1)
        assert np.all(np.diff(sc) <= 0) and np.all(np.isin(sc, pool))


def test_proposals_file_roundtrip_through_reference_json_dataset(params, tmp_path):
    """propose_images -> write_proposals_file -> the reference's JsonDataset.get_roidb(proposal_file=) -> the same recall on the device
    as in the reference."""
    from detectorch_b200.utils import coco_eval, proposal_file
    ref_eval, json_dataset = _oracle()
    from oracle import cocoapi
    if not cocoapi.available():
        pytest.skip("reference pycocotools not built")
    model = _model(params)
    ims = _uint8_images()
    ids = [42, 7, 19, 3, 11]                                # not sorted: the writer and the reader sort by id
    rng = np.random.RandomState(3)
    images, anns = [], []
    for i, (iid, im) in enumerate(zip(ids, ims)):
        h, w = im.shape[:2]
        images.append({'id': iid, 'width': w, 'height': h, 'file_name': "%d.jpg" % iid})
        open(os.path.join(tmp_path, "%d.jpg" % iid), "wb").close()
        for k in range(4):
            x, y = float(rng.uniform(0, w / 2)), float(rng.uniform(0, h / 2))
            bw, bh = float(rng.uniform(4, w / 2)), float(rng.uniform(4, h / 2))
            anns.append({'id': len(anns) + 1, 'image_id': iid, 'category_id': 1 + k % 2, 'bbox': [x, y, bw, bh], 'area': bw * bh,
                         'iscrowd': int(k == 3 and i == 0), 'segmentation': [[x, y, x + bw, y, x + bw, y + bh, x, y + bh]]})
    ann_file = os.path.join(tmp_path, "ann.json")
    with open(ann_file, "w") as f:
        json.dump({'images': images, 'annotations': anns, 'categories': [{'id': 1, 'name': 'a'}, {'id': 2, 'name': 'b'}]}, f)
    pkl = os.path.join(tmp_path, "proposals.pkl")
    props = model.propose_images(ims, target_size=128, max_size=200)
    proposal_file.write_proposals_file(pkl, ids, props)
    with open(pkl, "rb") as f:
        d = pickle.load(f, encoding='latin1')
    assert d['ids'] == sorted(ids)
    ds = json_dataset.JsonDataset(ann_file, str(tmp_path))
    roidb = ds.get_roidb(gt=True, proposal_file=pkl)
    assert [e['id'] for e in roidb] == sorted(ids)
    assert sum(int((e['gt_classes'] == 0).sum()) for e in roidb) > 0
    got = coco_eval.box_proposal_recall(roidb)
    for (area, limit), r in got.items():
        _same(r, ref_eval.evaluate_box_proposals(ds, roidb, area=area, limit=limit))


def test_propose_images_model_checks(built):
    from detectorch_b200.model.detector import detector
    fast = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                    conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=False,
                    roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                    use_rpn_head=False)
    with pytest.raises(RuntimeError):
        fast.propose_images(_uint8_images())
    c4 = detector(arch='resnet50', use_rpn_head=True)
    with pytest.raises(NotImplementedError):
        c4.propose_images(_uint8_images())

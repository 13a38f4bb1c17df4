"""Batched Fast R-CNN on the FPN body (detect(..., proposals=), detect_images(ims, proposals=), Engine.set_proposals): the device stage that
scales, deduplicates and maps each image's pre-computed proposals to the FPN levels equals the reference's preprocess_sample +
add_multilevel_rois_for_test bit for bit (tests/golden/fast_props_golden.npz), and every image's detections equal the batch-1 notebook flow
of eval_fast_FPN.ipynb (preprocess_sample(fpn_on=True), forward(image, [rois_fpn2..5], roi_original_idx), postprocess_output)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fast_props_golden.npz")
CASES = ["dups", "near", "half", "levels", "single", "full"]
CANVAS = (192, 256)
SIZES = [(192, 256), (128, 160), (192, 128), (96, 224)]
SCALES = [1.0, 0.8, 1.25, 0.6]
ORIG = [(190.0, 250.0), (161.0, 203.0), (150.0, 101.0), (161.0, 371.0)]
FAST_FPN = dict(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], roi_height=7, roi_width=7,
                roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2)


@pytest.fixture(scope="module")
def params(built):
    from oracle import network as net
    return net.synthetic_params("resnet50", fpn=True, rpn=False, mask=False)


def _fast_model(params, conv_kind=None):
    from detectorch_b200.model.detector import detector
    model = detector(**FAST_FPN)
    sd = model.state_dict()
    for k, v in params.items():
        sd[k].copy_(v)
    model = model.cuda()
    if conv_kind is not None:
        model.engine_defaults["conv_kind"] = conv_kind
    return model


def _canvas_batch(sizes, seed0=0, fill=float("nan")):
    from oracle import network as net
    crops = [net.synthetic_image(1, h, w, seed=seed0 + b) for b, (h, w) in enumerate(sizes)]
    img = torch.full((len(sizes), 3) + CANVAS, fill)
    for b, (h, w) in enumerate(sizes):
        img[b, :, :h, :w] = crops[b][0]
    return img, crops


def _proposals(rng, n, oh, ow):
    """n float32 roidb-style boxes inside an oh x ow original image: Detectron-like sizes and aspect ratios, ~5 % exact duplicates and
    ~5 % boxes within 2 px of another one (most of which hash to the same cell)."""
    m = n - 2 * (n // 20)
    side = np.exp(rng.uniform(np.log(6), np.log(max(ow, oh)), m))
    ar = np.exp(rng.uniform(np.log(0.4), np.log(2.5), m))
    w, h = np.minimum(side * np.sqrt(ar), ow - 1), np.minimum(side / np.sqrt(ar), oh - 1)
    x1, y1 = rng.uniform(0, ow - w), rng.uniform(0, oh - h)
    b = np.stack([x1, y1, x1 + w, y1 + h], 1)
    near = b[rng.choice(m, n // 20)] + rng.uniform(-2, 2, (n // 20, 4))
    near[:, 2:] = np.maximum(near[:, 2:], near[:, :2])
    b = np.concatenate([b, b[rng.choice(m, n // 20)], near])
    return b[rng.permutation(n)].astype(np.float32)


def _mirror_rois(boxes, scale):
    """preprocess_sample's proposal half (preprocess_sample.py:36-45), through the mirror's own code."""
    from detectorch_b200.utils.multilevel_rois import add_multilevel_rois_for_test
    from detectorch_b200.utils.preprocess_sample import preprocess_sample
    proposals, _ = preprocess_sample(fpn_on=True).remove_dup_prop(boxes * scale)
    return add_multilevel_rois_for_test({'rois': proposals}, 'rois')


def _notebook_flow(model, image, boxes, sf, orig):
    """eval_fast_FPN.ipynb's loop body for one image -> (scores_final, boxes_final, per-detection class)."""
    from detectorch_b200.utils import result_utils
    dev = torch.device("cuda:0")
    blobs = _mirror_rois(boxes, sf)
    lst = [torch.FloatTensor(blobs['rois_fpn%d' % l]).to(dev) for l in range(2, 6)]
    with torch.no_grad():
        cls, box, _, _ = model(image.to(dev), lst, roi_original_idx=torch.from_numpy(blobs['rois_idx_restore_int32']).long().to(dev))
    scores, bxs, cb = result_utils.postprocess_output(torch.FloatTensor(blobs['rois']), sf, torch.tensor([orig[0], orig[1], 3.0]), cls, box)
    classes = np.concatenate([np.full(len(cb[j]), j) for j in range(1, 81)]).astype(np.int32)
    return scores, bxs, classes


def _snap(out):
    return {k: v.clone() for k, v in out.items() if k != "range_flag"}


def test_kernel_vs_golden(params):
    """The ST_COLLECT stage of a batch engine with the per-image table on: rois / roi_levels / roi_counts equal the reference's
    remove_dup_prop + add_multilevel_rois_for_test (golden) and the mirror's, in order, bit for bit."""
    from detectorch_b200.engine import Engine, ST_TRUNK, ST_DETECT
    g = np.load(GOLDEN)
    sizes = [(192, 256), (128, 160), (192, 128), (96, 224), (64, 64), (160, 256)]
    dev = torch.device("cuda:0")
    eng = Engine(batch=len(CASES), height=CANVAS[0], width=CANVAS[1], use_rpn=False, use_mask=False, post_nms_top_n=1000)
    eng.load_state_dict(params)
    img, _ = _canvas_batch(sizes)
    eng.set_image_info(sizes, [float(g[c + "_scale"]) for c in CASES])
    eng.set_proposals([g[c + "_boxes"] for c in CASES])
    eng.run(img.to(dev), 1.0, ST_TRUNK, ST_DETECT)
    torch.cuda.synchronize()
    rois, levels, counts = eng.buffer("rois").cpu(), eng.buffer("roi_levels").cpu(), eng.buffer("roi_counts").cpu()
    for b, c in enumerate(CASES):
        want, lv = torch.from_numpy(g[c + "_props"]), torch.from_numpy(g[c + "_levels"].astype(np.int32) - 2)
        m = want.shape[0]
        assert int(counts[b]) == m, c
        assert torch.equal(rois[b, :m, 1:5], want), c
        assert torch.equal(levels[b, :m], lv), c
        assert bool((rois[b, :, 0] == b).all()) and int(torch.count_nonzero(rois[b, m:, 1:5])) == 0 and int(torch.count_nonzero(levels[b, m:])) == 0
        blobs = _mirror_rois(g[c + "_boxes"], float(g[c + "_scale"]))
        assert np.array_equal(blobs['rois'], g[c + "_props"]) and np.array_equal(blobs['rois_idx_restore_int32'], g[c + "_restore"]), c
    assert int(counts[CASES.index("single")]) == 1 and int(counts[CASES.index("full")]) > 900


@pytest.mark.parametrize("conv_kind", ["f16", "tf32"])
def test_per_image_equality(params, conv_kind):
    """detect(canvas, scales, proposals=, image_sizes=, original_sizes=) against the notebook flow of each image alone (an engine sized
    by its rounded proposal count there, 1000 here)."""
    dev = torch.device("cuda:0")
    model = _fast_model(params, conv_kind)
    rng = np.random.RandomState(1)
    props = [_proposals(rng, n, int(o[0]), int(o[1])) for n, o in zip([300, 1000, 517, 760], ORIG)]
    img, crops = _canvas_batch(SIZES)
    out = model.detect(img.to(dev), scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG, proposals=props)
    torch.cuda.synchronize()
    assert int(out["range_flag"].item()) == 0
    assert "masks" not in out
    counts, boxes, scores, classes = (out[k].cpu() for k in ("counts", "boxes", "scores", "classes"))
    total = 0
    for b in range(len(SIZES)):
        sf, bf, cl = _notebook_flow(model, crops[b], props[b], SCALES[b], ORIG[b])
        n = int(counts[b])
        assert n == len(sf), b
        assert torch.equal(boxes[b, :n], torch.from_numpy(bf)) and torch.equal(scores[b, :n], torch.from_numpy(sf)), b
        assert torch.equal(classes[b, :n], torch.from_numpy(cl)), b
        total += n
    assert total > 0


def test_detect_images(params):
    """uint8 photos + roidb boxes -> what eval_fast_FPN.ipynb files per image: (scores_final, boxes_final, boxes_per_class, None)."""
    from detectorch_b200.utils import result_utils
    from detectorch_b200.utils.preprocess_sample import preprocess_sample
    dev = torch.device("cuda:0")
    model = _fast_model(params)
    rng = np.random.RandomState(2)
    shapes = [(60, 80), (90, 50), (64, 64), (41, 97), (75, 75)]
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    props = [_proposals(rng, n, h, w) for n, (h, w) in zip([400, 1000, 350, 620, 999], shapes)]
    res = model.detect_images(ims, target_size=128, max_size=200, proposals=props)
    assert len(res) == len(ims)
    total = 0
    for im, p, (sc, bx, cb, segms) in zip(ims, props, res):
        s = preprocess_sample(target_sizes=128, max_size=200, fpn_on=True)({'image': im, 'dbentry': {'boxes': p}})
        lst = [s['rois_fpn%d' % l].to(dev) for l in range(2, 6)]
        with torch.no_grad():
            cls, box, _, _ = model(s['image'], lst, roi_original_idx=s['rois_idx_restore_int32'].long().to(dev))
        w_sc, w_bx, w_cb = result_utils.postprocess_output(s['rois'], s['scaling_factors'], s['original_im_size'], cls, box)
        assert segms is None
        assert np.array_equal(sc, w_sc) and np.array_equal(bx, w_bx)
        for j in range(1, 81):
            assert np.array_equal(np.asarray(cb[j]).reshape(-1, 5), np.asarray(w_cb[j]).reshape(-1, 5)), j
        total += len(sc)
    assert total > 0


def test_graph_replay(params):
    """Host input replays a captured graph; the proposals are written on the run's stream, so back-to-back calls with different
    proposals and size mixes each get their own results."""
    dev = torch.device("cuda:0")
    model = _fast_model(params)
    rng = np.random.RandomState(3)
    mix_b = ([(96, 128), (192, 256), (160, 96), (64, 64)], [0.9, 1.1, 1.0, 0.5], [(107.0, 142.0), (175.0, 233.0), (160.0, 96.0), (128.0, 128.0)])
    img_a, _ = _canvas_batch(SIZES, seed0=0)
    img_b, _ = _canvas_batch(mix_b[0], seed0=10)
    calls = {"a": (img_a, dict(scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG,
                               proposals=[_proposals(rng, n, int(o[0]), int(o[1])) for n, o in zip([500, 800, 300, 1000], ORIG)])),
             "b": (img_b, dict(scaling_factor=mix_b[1], image_sizes=mix_b[0], original_sizes=mix_b[2],
                               proposals=[_proposals(rng, n, int(o[0]), int(o[1])) for n, o in zip([1000, 420, 640, 200], mix_b[2])]))}
    want = {k: {n: v.cpu() for n, v in _snap(model.detect(im.to(dev), **kw)).items()} for k, (im, kw) in calls.items()}
    host = {k: im.pin_memory() for k, (im, _) in calls.items()}
    for k in ["a", "b", "a", "b"]:             # the first round runs eagerly, the second captures one graph per staging buffer
        model.detect(host[k], **calls[k][1])
    torch.cuda.synchronize()
    st = model.engine_for(4, *CANVAS, post_nms_top_n=1000)._stage_state
    assert len(st["graphs"]) == 2
    got = [(k, _snap(model.detect(host[k], **calls[k][1]))) for k in ["b", "a", "a", "b"]]     # no synchronisation in between
    torch.cuda.synchronize()
    for k, out in got:
        for n, v in out.items():
            assert torch.equal(v.cpu(), want[k][n]), (k, n)


def test_zero_and_full(params):
    """An image without proposals has no detections and leaves its neighbours' results as they are; 1000 proposals fit."""
    dev = torch.device("cuda:0")
    model = _fast_model(params)
    rng = np.random.RandomState(4)
    props = [_proposals(rng, n, int(o[0]), int(o[1])) for n, o in zip([600, 300, 1000, 450], ORIG)]
    img, _ = _canvas_batch(SIZES)
    kw = dict(scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG)
    full = _snap(model.detect(img.to(dev), proposals=props, **kw))
    empty = _snap(model.detect(img.to(dev), proposals=props[:1] + [np.zeros((0, 4), np.float32)] + props[2:], **kw))
    torch.cuda.synchronize()
    assert int(empty["counts"][1].item()) == 0 and int(full["counts"][1].item()) > 0
    assert int(full["counts"][2].item()) > 0
    for b in (0, 2, 3):
        for k in full:
            assert torch.equal(empty[k][b], full[k][b]), (k, b)


def test_validation_before_launch(params):
    from detectorch_b200.model.detector import detector
    model = _fast_model(params)
    img = torch.zeros((4, 3) + CANVAS)
    ok = [np.array([[0, 0, 10, 10]], np.float32)] * 4
    kw = dict(scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG)
    bad = [(ValueError, ok[:3]), (TypeError, [ok[0].astype(np.float64)] + ok[1:]), (ValueError, [ok[0].reshape(1, 2, 2)] + ok[1:]),
           (ValueError, [np.array([[0, 0, np.nan, 10]], np.float32)] + ok[1:]), (ValueError, [np.zeros((1001, 4), np.float32)] + ok[1:]),
           (ValueError, [np.array([[0, 0, 2e5, 10]], np.float32)] + ok[1:]), (ValueError, [np.array([[10, 0, 0, 10]], np.float32)] + ok[1:]),
           (TypeError, np.zeros((4, 1, 4), np.float32))]
    for exc, p in bad:
        with pytest.raises(exc):
            model.detect(img, proposals=p, **kw)
    with pytest.raises(RuntimeError):
        model.detect(img, **kw)
    assert len(model._engines) == 0
    rpn = detector(**dict(FAST_FPN, use_rpn_head=True))
    with pytest.raises(ValueError):
        rpn.detect(img, proposals=ok, **kw)
    c4 = detector(arch='resnet50')
    with pytest.raises(NotImplementedError):
        c4.detect(img, proposals=ok)

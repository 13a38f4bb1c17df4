"""Batches of differently-sized images on one padded canvas (detect(..., image_sizes, original_sizes), Engine.set_image_info):
every image's maps, proposals, detections and masks are bit-identical to a batch-1 run of that image at its own size, whatever the
canvas holds around it (NaN here), on every conv kind and RoIAlign variant; a captured graph replays for any size mix."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CANVAS = (192, 256)
SIZES = [(192, 256), (128, 160), (192, 128), (96, 224)]
SCALES = [1.0, 0.8, 1.25, 0.6]
ORIG = [(190.0, 250.0), (161.0, 203.0), (150.0, 101.0), (161.0, 371.0)]
# image-shaped maps and their strides: valid region ceil(size / stride), exactly zero outside
MAPS = [("C2", 4), ("C3", 8), ("C4", 16), ("C5", 32), ("P2", 4), ("P3", 8), ("P4", 16), ("P5", 32), ("P6", 64),
        ("rpn_out2", 4), ("rpn_out3", 8), ("rpn_out4", 16), ("rpn_out5", 32), ("rpn_out6", 64)]
DETS = ["det_boxes", "det_scores", "det_classes", "det_counts", "det_roi_idx"]


def _canvas_batch(sizes, seed0=0, fill=float("nan")):
    from oracle import network as net
    crops = [net.synthetic_image(1, h, w, seed=seed0 + b) for b, (h, w) in enumerate(sizes)]
    img = torch.full((len(sizes), 3) + CANVAS, fill)
    for b, (h, w) in enumerate(sizes):
        img[b, :, :h, :w] = crops[b][0]
    return img, crops


@pytest.fixture(scope="module")
def params(built):
    from oracle import network as net
    return net.synthetic_params("resnet50")


def _mask_model(params):
    from detectorch_b200.model.detector import detector
    model = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                     conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                     roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                     use_rpn_head=True, use_mask_head=True, mask_head_type='1up4convs')
    sd = model.state_dict()
    for k, v in params.items():
        sd[k].copy_(v)
    return model.cuda()


@pytest.mark.parametrize("conv_kind,exact", [("f16", False), ("f16", True), ("tf32", False)])
def test_per_image_equality(params, conv_kind, exact):
    from detectorch_b200.engine import Engine
    dev = torch.device("cuda:0")
    kw = dict(arch="resnet50", det_cap=128, exact_roialign=exact, conv_kind=conv_kind)
    img, crops = _canvas_batch(SIZES)
    eng = Engine(batch=len(SIZES), height=CANVAS[0], width=CANVAS[1], **kw)
    eng.load_state_dict(params)
    eng.set_image_info(SIZES, SCALES, ORIG)
    eng.run(img.to(dev), 1.0)
    torch.cuda.synchronize()
    assert int(eng.buffer("range_flag").item()) == 0
    cap = eng.cfg.det_cap
    masks = eng.buffer("masks").view(len(SIZES), cap, 28, 28)
    total = 0
    for b, (h, w) in enumerate(SIZES):
        ref = Engine(batch=1, height=h, width=w, share_weights_with=eng, **kw)
        ref.set_original_size(*ORIG[b])
        ref.run(crops[b].to(dev), SCALES[b])
        torch.cuda.synchronize()
        assert int(ref.buffer("range_flag").item()) == 0
        for name, s in MAPS:
            got, want = eng.buffer(name)[b], ref.buffer(name)[0]
            eh, ew = -(-h // s), -(-w // s)
            assert tuple(want.shape[:2]) == (eh, ew)
            assert torch.equal(got[:eh, :ew], want), (name, b)
            pad = got.clone()
            pad[:eh, :ew] = 0
            assert int(torch.count_nonzero(pad)) == 0, (name, b)       # exact zeros (NaN would count as non-zero)
        assert torch.equal(eng.buffer("roi_counts")[b], ref.buffer("roi_counts")[0])
        assert torch.equal(eng.buffer("rois")[b, :, 1:5], ref.buffer("rois")[0, :, 1:5])
        for name in DETS:
            assert torch.equal(eng.buffer(name)[b], ref.buffer(name)[0]), (name, b)
        assert torch.equal(masks[b], ref.buffer("masks").view(1, cap, 28, 28)[0]), b
        total += int(ref.buffer("det_counts")[0].item())
        del ref
    assert total > 0


def _notebook_flow(model, image, sf, orig):
    """eval_mask_FPN.ipynb cell 10 for one image: forward, postprocess_output, the mask RoIs (boxes_final * scaling_factor distributed over
    the FPN levels), mask_head -> (scores_final, boxes_final, per-detection class, masks of that class [D,28,28])."""
    from detectorch_b200.utils import result_utils
    from detectorch_b200.utils.multilevel_rois import add_multilevel_rois_for_test
    dev = torch.device("cuda:0")
    with torch.no_grad():
        cls, box, rois, feats = model(image.to(dev), scaling_factor=torch.tensor([sf]))
    scores, boxes, cb = result_utils.postprocess_output(rois, torch.tensor([sf]), torch.tensor([orig]), cls, box)
    classes = np.concatenate([np.full(len(cb[j]), j) for j in range(1, 81)]).astype(np.int64)
    blobs = add_multilevel_rois_for_test({"mask_rois": boxes * np.float32(sf)}, "mask_rois")
    lst = [torch.from_numpy(blobs["mask_rois_fpn%d" % l]).to(dev) if len(blobs["mask_rois_fpn%d" % l]) else None for l in range(2, 6)]
    masks = torch.zeros((0, 28, 28))
    if len(boxes):
        full = model.mask_head(feats, lst, torch.from_numpy(blobs["mask_rois_idx_restore_int32"].astype(np.int64)).to(dev))
        masks = full[torch.arange(len(boxes), device=dev), torch.from_numpy(classes).to(dev)].cpu()
    return scores, boxes, classes, masks


def test_reference_flow(params):
    """detect(..., image_sizes, original_sizes) against the notebook flow (forward + postprocess_output + mask_head) of each image alone."""
    dev = torch.device("cuda:0")
    model = _mask_model(params)
    img, crops = _canvas_batch(SIZES)
    out = model.detect(img.to(dev), scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG)
    torch.cuda.synchronize()
    assert int(out["range_flag"].item()) == 0
    counts, boxes = out["counts"].cpu().numpy(), out["boxes"].cpu().numpy()
    scores, classes, masks = out["scores"].cpu().numpy(), out["classes"].cpu().numpy(), out["masks"].cpu()
    total = 0
    for b in range(len(SIZES)):
        sf, bf, cls, mk = _notebook_flow(model, crops[b], SCALES[b], ORIG[b])
        n = int(counts[b])
        assert n == len(sf)
        assert np.array_equal(boxes[b, :n], bf) and np.array_equal(scores[b, :n], sf)
        assert np.array_equal(classes[b, :n], cls)
        assert torch.equal(masks[b, :n], mk), b
        total += n
    assert total > 0


def test_table_does_not_outlive_detect(params):
    """A batch-1 detect() with per-image sizes shares its engine with forward() on the same input shape; the table must not leak into the
    notebook flow that follows (different image, scale and original size): it must equal that flow on a model that never saw a table."""
    from oracle import network as net
    dev = torch.device("cuda:0")
    model, fresh = _mask_model(params), _mask_model(params)
    img, _ = _canvas_batch([(128, 160)], seed0=5)
    out = model.detect(img.to(dev), scaling_factor=[0.8], image_sizes=[(128, 160)], original_sizes=[(161.0, 203.0)])
    torch.cuda.synchronize()
    assert int(out["counts"][0].item()) >= 0
    image = net.synthetic_image(1, CANVAS[0], CANVAS[1], seed=7)
    got = _notebook_flow(model, image, 1.25, (153.0, 204.0))
    want = _notebook_flow(fresh, image, 1.25, (153.0, 204.0))
    assert len(want[0]) > 0
    for g, w in zip(got, want):
        assert (torch.equal(g, w) if torch.is_tensor(g) else np.array_equal(g, w))
    # and the uniform detect() on that engine afterwards equals the fresh model's
    a, b = _snap(model.detect(image.to(dev), 1.25)), _snap(fresh.detect(image.to(dev), 1.25))
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k].cpu(), b[k].cpu()), k


def _snap(out):
    return {k: v.clone() for k, v in out.items() if k != "range_flag"}


def test_uniform_sizes_unchanged(params):
    dev = torch.device("cuda:0")
    model = _mask_model(params)
    img, _ = _canvas_batch([CANVAS] * 4, fill=0.0)
    img = img.to(dev)
    a = _snap(model.detect(img, 0.9))
    b = _snap(model.detect(img, 0.9, image_sizes=[CANVAS] * 4))
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_graph_replay_with_changing_sizes(params):
    """Host input is replayed from captured graphs; the table is written on the run's stream, so back-to-back calls with different size
    mixes (and then none) each get their own results, and no new graph is captured for a new mix."""
    dev = torch.device("cuda:0")
    model = _mask_model(params)
    mix_b = ([(96, 128), (192, 256), (160, 96), (64, 64)], [0.9, 1.1, 1.0, 0.5], [(107.0, 142.0), (175.0, 233.0), (160.0, 96.0), (128.0, 128.0)])
    img_a, _ = _canvas_batch(SIZES, seed0=0)
    img_b, _ = _canvas_batch(mix_b[0], seed0=10)
    img_u, _ = _canvas_batch([CANVAS] * 4, seed0=20, fill=0.0)
    calls = {"a": (img_a, dict(scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG)),
             "b": (img_b, dict(scaling_factor=mix_b[1], image_sizes=mix_b[0], original_sizes=mix_b[2])),
             "u": (img_u, dict(scaling_factor=1.0))}
    want = {}
    for k, (im, kw) in calls.items():          # device input: the eager path
        want[k] = {n: v.cpu() for n, v in _snap(model.detect(im.to(dev), **kw)).items()}
    host = {k: im.pin_memory() for k, (im, _) in calls.items()}
    # staging buffers alternate: the first round sees every (buffer, table on/off) key once, the second captures each of them
    for k in ["a", "b", "u", "u", "a", "b", "u", "u"]:
        model.detect(host[k], **calls[k][1])
    torch.cuda.synchronize()
    st = model.engine_for(4, *CANVAS)._stage_state
    graphs = dict(st["graphs"])
    assert len(graphs) == 4
    got = []
    for k in ["b", "a", "u", "a", "b"]:        # replays of graphs captured under the other mix; no synchronisation in between
        got.append((k, _snap(model.detect(host[k], **calls[k][1]))))
    torch.cuda.synchronize()
    assert st["graphs"] == graphs and all(st["graphs"][g] is graphs[g] for g in graphs)
    for k, out in got:
        for n, v in out.items():
            assert torch.equal(v.cpu(), want[k][n]), (k, n)


def test_validation_before_launch(params):
    model = _mask_model(params)
    img = torch.zeros((4, 3) + CANVAS)
    bad = [dict(image_sizes=[(100, 128)] * 4), dict(image_sizes=[(224, 256)] + SIZES[1:]), dict(image_sizes=[(0, 64)] + SIZES[1:]),
           dict(image_sizes=SIZES[:3]), dict(scaling_factor=[1.0, 1.0, 0.0, 1.0]), dict(scaling_factor=[1.0, -2.0, 1.0, 1.0], image_sizes=SIZES),
           dict(scaling_factor=[1.0, 1.0]), dict(image_sizes=SIZES, original_sizes=ORIG[:2]), dict(image_sizes=SIZES, original_sizes=[(0, 1)] * 4)]
    for kw in bad:
        with pytest.raises(ValueError):
            model.detect(img, **kw)
    assert len(model._engines) == 0              # nothing was built or launched
    from detectorch_b200.model.detector import detector
    c4 = detector(arch='resnet50', use_rpn_head=True, use_mask_head=True, mask_head_type='upshare', roi_height=14, roi_width=14,
                  roi_spatial_scale=0.0625, roi_sampling_ratio=0)
    with pytest.raises(NotImplementedError):
        c4.detect(img, image_sizes=SIZES)


def test_images_to_batch(built):
    from detectorch_b200.utils import blob
    rng = np.random.RandomState(3)
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(60, 80), (90, 50), (64, 64), (41, 97)]]
    for canvas in (None, (256, 256)):
        data, sizes, scales, orig = blob.images_to_batch(ims, target_size=128, max_size=200, canvas=canvas)
        torch.cuda.synchronize()
        if canvas is not None:
            assert tuple(data.shape[2:]) == canvas
        for b, im in enumerate(ims):
            one, s = blob.image_to_blob(im, target_size=128, max_size=200, fpn_on=True)
            h, w = one.shape[2:]
            assert (int(sizes[b, 0]), int(sizes[b, 1])) == (h, w) and h % 32 == 0 and w % 32 == 0
            assert float(scales[b]) == s == blob.im_scale_for(im.shape, 128, 200)
            assert (int(orig[b, 0]), int(orig[b, 1])) == im.shape[:2]
            assert torch.equal(data[b, :, :h, :w], one[0])
            rest = data[b].clone()
            rest[:, :h, :w] = 0
            assert int(torch.count_nonzero(rest)) == 0

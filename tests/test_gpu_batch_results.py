"""Batched COCO results: dt_segm_rle_batch (ops.segm_rle_batch), result_utils.batch_results and detector.detect_images.  The batched
paste + RLE must equal the one-image dt_segm_rle, the oracle and the reference-produced golden strings per image; batch_results and
detect_images must return, per image, exactly what the notebook flow (forward, postprocess_output, mask_head, segm_results) returns for
that image alone."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
M, K, CAP = 28, 4, 100

CANVAS = (192, 256)
SIZES = [(192, 256), (128, 160), (192, 128), (96, 224)]
SCALES = [1.0, 0.8, 1.25, 0.6]
ORIG = [(190.0, 250.0), (161.7, 203.2), (150.0, 101.9), (161.0, 371.5)]     # the RLE canvas is int() of each value


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def ref_mod():
    from oracle import ref
    return ref


# ------------------------------------------------------------------------------------------------ the batched kernel
def _blob_masks(rng, n):
    yy, xx = np.mgrid[0:M, 0:M].astype(np.float32) / M
    out = np.zeros((n, K, M, M), np.float32)
    for d in range(n):
        for k in range(K):
            cx, cy, r = rng.uniform(.3, .7), rng.uniform(.3, .7), rng.uniform(.15, .45)
            out[d, k] = np.clip(1.0 / (1.0 + np.exp(((xx - cx) ** 2 + (yy - cy) ** 2 - r * r) * 40)) + 0.25 * rng.randn(M, M), 0, 1)
    return out


def _random_boxes(rng, n, W, H):
    cx, cy = rng.uniform(0, W, n), rng.uniform(0, H, n)
    w = np.exp(rng.uniform(np.log(4), np.log(max(W, H)), n)); a = np.exp(rng.uniform(-0.7, 0.7, n))
    b = np.stack([cx - w * np.sqrt(a) / 2, cy - w / np.sqrt(a) / 2, cx + w * np.sqrt(a) / 2, cy + w / np.sqrt(a) / 2], 1)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, W - 1); b[:, 1::2] = np.clip(b[:, 1::2], 0, H - 1)    # detections are clipped to the image
    return b.astype(np.float32)


def _kernel_batch():
    """Five images on CAP slots: 800x1216 with 100 live detections, a small image whose expanded boxes cross every border, the m28 golden
    case, an image with no live detection and another with every slot live.  Dead slots hold NaN boxes."""
    rng = np.random.RandomState(7)
    S = np.load(os.path.join(GOLD, "segm_golden.npz"))
    h, w = 37, 53
    border = np.array([[0, 0, w - 1, h - 1], [0, 0, 4, 4], [w - 5, h - 5, w - 1, h - 1], [0, 10, 3, 30], [w - 3, 5, w - 1, 20],
                       [10, 0, 20, 2], [15, h - 3, 40, h - 1], [0.5, 0.5, 1.5, h - 1.5], [w - 1.5, 0, w - 1, h - 1], [2.2, 3.3, 50.1, 33.9]],
                      np.float32)
    big = _random_boxes(rng, 100, 1216, 800)
    big[:6] = [[0, 0, 1215, 799], [0, 0, 3, 3], [1207, 791, 1215, 799], [600, 0, 620, 799], [0, 400, 1215, 410], [100, 100, 113, 113]]
    images = [((800, 1216), big), ((h, w), border), (tuple(int(v) for v in S["m28_size"]), S["m28_boxes"]), ((480, 640), np.zeros((0, 4))),
              ((333, 517), _random_boxes(rng, CAP, 517, 333))]
    B = len(images)
    masks = np.zeros((B, CAP, K, M, M), np.float32)
    boxes = np.full((B, CAP, 4), np.nan, np.float32)
    classes = np.zeros((B, CAP), np.int32)
    counts = np.zeros((B,), np.int32)
    for b, ((ih, iw), bx) in enumerate(images):
        n = len(bx)
        counts[b] = n
        masks[b] = _blob_masks(rng, CAP)
        boxes[b, :n] = bx
        classes[b, :n] = np.sort(rng.randint(1, K, n))
    masks[0, 0] = 1.0                                          # the whole image set: runs touch every border
    n = int(counts[2])
    masks[2, :n], classes[2, :n] = S["m28_masks"], S["m28_cls"]
    sizes = np.array([s for s, _ in images], np.int64)
    return masks, boxes, classes, counts, sizes, [str(x) for x in S["m28_rle"]]


def test_segm_rle_batch_matches_single_image_oracle_and_golden(dev):
    from detectorch_b200 import ops
    ref = ref_mod()
    masks, boxes, classes, counts, sizes, golden = _kernel_batch()
    B = len(counts)
    assert counts[0] == 100 and sizes[0].tolist() == [800, 1216] and counts[3] == 0 and counts[4] == CAP
    tm, tb, tc, tn = (torch.from_numpy(x).to(dev) for x in (masks, boxes, classes, counts))
    sel = tm[torch.arange(B, device=dev)[:, None], torch.arange(CAP, device=dev)[None, :], tc.long()]        # [B,CAP,M,M]
    full = ops.segm_rle_batch(tm, tc, tb, tn, sizes)
    assert full == ops.segm_rle_batch(sel, None, tb, tn, sizes)
    assert full == ops.segm_rle_batch(tm, tc, tb, tn, torch.from_numpy(sizes), runs_cap=8)      # grow and redo, same strings
    assert [len(f) for f in full] == counts.tolist()
    assert full[2] == [g.encode() for g in golden]
    for b in range(B):
        n, (ih, iw) = int(counts[b]), (int(sizes[b, 0]), int(sizes[b, 1]))
        if n == 0:
            continue
        _, single = ops.segm_rle(tm[b, :n], tc[b, :n], tb[b, :n], ih, iw)
        assert full[b] == single, b
        exp = ref.expand_boxes(boxes[b, :n], (M + 2.0) / M).astype(np.int32)
        crossing = set()
        for d in range(n):
            e = exp[d]
            crossing |= {s for s, c in zip("ltrb", (e[0] < 0, e[1] < 0, e[2] >= iw, e[3] >= ih)) if c}
            want = ref.rle_to_string(ref.rle_encode(ref.paste_mask(masks[b, d, classes[b, d]], e, ih, iw)))
            assert full[b][d] == want, (b, d)
        if b == 1:
            assert crossing == set("ltrb")


def test_segm_rle_batch_arguments(dev):
    from detectorch_b200 import ops
    tm = torch.zeros((2, 3, M, M), device=dev)
    tb = torch.zeros((2, 3, 4), device=dev)
    tn = torch.tensor([1, 0], dtype=torch.int32, device=dev)
    for bad in ([(10, 10)], [(10, 10), (0, 5)], [(10, 10), (5, -3)], [(10, 10, 1), (5, 5)], [(10, 10), (float("nan"), 5)], [(2 ** 16, 2 ** 16)] * 2):
        with pytest.raises(ValueError):
            ops.segm_rle_batch(tm, None, tb, tn, bad)
    with pytest.raises(ValueError):
        ops.segm_rle_batch(tm, torch.zeros((2, 3), dtype=torch.int32, device=dev), tb, tn, [(10, 10)] * 2)     # classes need K planes
    with pytest.raises(RuntimeError):
        ops.segm_rle_batch(tm, None, tb, tn, [(20000, 10), (10, 10)])          # row table beyond the shared-memory limit
    # an empty mask in a box: one run of zeros per live slot, nothing for dead ones
    got = ops.segm_rle_batch(tm, None, tb, tn, [(10, 10), (4, 6)])
    assert got == [[ref_mod().rle_to_string(np.array([100], np.uint32))], []]


# ------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def params(built):
    from oracle import network as net
    return net.synthetic_params("resnet50")


def _model(params, mask=True):
    from detectorch_b200.model.detector import detector
    model = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                     conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                     roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2,
                     use_rpn_head=True, use_mask_head=mask, mask_head_type='1up4convs')
    sd = model.state_dict()
    for k, v in params.items():
        if k in sd:
            sd[k].copy_(v)
    return model.cuda()


def _notebook_flow(model, image, sf, orig):
    """eval_mask_FPN.ipynb cell 10 for one image -> (scores_final, boxes_final, boxes_per_class, cls_segms); cls_segms is None without a
    mask head."""
    from detectorch_b200.utils import result_utils
    from detectorch_b200.utils.multilevel_rois import add_multilevel_rois_for_test
    dev = torch.device("cuda:0")
    with torch.no_grad():
        cls, box, rois, feats = model(image.to(dev), scaling_factor=torch.tensor([sf]))
    scores, boxes, cls_boxes = result_utils.postprocess_output(rois, torch.tensor([sf]), torch.tensor([orig]), cls, box)
    if not model.use_mask_head:
        return scores, boxes, cls_boxes, None
    masks = torch.zeros((0, 81, M, M), device=dev)
    if len(boxes):
        blobs = add_multilevel_rois_for_test({"mask_rois": boxes * np.float32(sf)}, "mask_rois")
        lst = [torch.from_numpy(blobs["mask_rois_fpn%d" % l]).to(dev) if len(blobs["mask_rois_fpn%d" % l]) else None for l in range(2, 6)]
        masks = model.mask_head(feats, lst, torch.from_numpy(blobs["mask_rois_idx_restore_int32"].astype(np.int64)).to(dev))
    segms = result_utils.segm_results(cls_boxes, masks, boxes, int(orig[0]), int(orig[1]), M=M)
    return scores, boxes, cls_boxes, segms


def _assert_same(got, want, what):
    sc, bx, cb, segms = got
    assert np.array_equal(sc, want[0]) and np.array_equal(bx, want[1]), what
    assert len(cb) == len(want[2]) == 81 and cb[0] == want[2][0] == []
    for j in range(1, 81):
        assert np.array_equal(cb[j], want[2][j]) and cb[j].dtype == want[2][j].dtype, (what, j)
    assert segms == want[3], what


def test_batch_results_equals_notebook_flow(params):
    """NaN-padded ragged canvas -> detect() -> batch_results: each image's four values equal the notebook flow on its crop."""
    from detectorch_b200.utils import result_utils
    from oracle import network as net
    dev = torch.device("cuda:0")
    model = _model(params)
    crops = [net.synthetic_image(1, h, w, seed=b) for b, (h, w) in enumerate(SIZES)]
    img = torch.full((len(SIZES), 3) + CANVAS, float("nan"))
    for b, (h, w) in enumerate(SIZES):
        img[b, :, :h, :w] = crops[b][0]
    out = model.detect(img.to(dev), scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG)
    got = result_utils.batch_results(out, ORIG)
    counts, classes = out["counts"].cpu().numpy(), out["classes"].cpu().numpy()
    assert int(out["range_flag"].item()) == 0
    total = 0
    for b in range(len(SIZES)):
        n = int(counts[b])
        assert np.all(np.diff(classes[b, :n]) >= 0)                  # slots are class-major, which segm_results relies on
        want = _notebook_flow(model, crops[b], SCALES[b], ORIG[b])
        _assert_same(got[b], want, b)
        assert all(s["size"] == [int(ORIG[b][0]), int(ORIG[b][1])] for j in range(1, 81) for s in got[b][3][j])
        total += n
    assert total > 0
    # without masks the same boxes, and no segmentations
    got_nm = result_utils.batch_results(model.detect(img.to(dev), scaling_factor=SCALES, image_sizes=SIZES, original_sizes=ORIG,
                                                     with_masks=False), ORIG)
    for b in range(len(SIZES)):
        assert got_nm[b][3] is None
        _assert_same(got_nm[b][:3] + (None,), got[b][:3] + (None,), b)


def _uint8_images():
    rng = np.random.RandomState(11)
    return [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(60, 80), (90, 50), (64, 64), (41, 97), (77, 70)]]


def _flow_on_uint8(model, im):
    from detectorch_b200.utils import blob
    data, s = blob.image_to_blob(im, target_size=128, max_size=200, fpn_on=True)
    return _notebook_flow(model, data, s, (float(im.shape[0]), float(im.shape[1])))


def test_detect_images_equals_notebook_flow(params):
    model = _model(params)
    ims = _uint8_images()
    for canvas in (None, (224, 224)):
        got = model.detect_images(ims, target_size=128, max_size=200, canvas=canvas)
        assert len(got) == len(ims)
        total = 0
        for b, im in enumerate(ims):
            _assert_same(got[b], _flow_on_uint8(model, im), b)
            total += len(got[b][0])
        assert total > 0


def test_detect_images_faster_rcnn(built):
    from oracle import network as net
    model = _model(net.synthetic_params("resnet50", mask=False), mask=False)
    ims = _uint8_images()
    got = model.detect_images(ims, target_size=128, max_size=200)
    total = 0
    for b, im in enumerate(ims):
        assert got[b][3] is None
        _assert_same(got[b], _flow_on_uint8(model, im), b)
        total += len(got[b][0])
    assert total > 0


def test_validation_before_launch(params):
    from detectorch_b200.model.detector import detector
    from detectorch_b200.utils import result_utils
    dev = torch.device("cuda:0")
    out = {"boxes": torch.zeros((2, CAP, 4), device=dev), "scores": torch.zeros((2, CAP), device=dev),
           "classes": torch.zeros((2, CAP), dtype=torch.int32, device=dev), "counts": torch.zeros((2,), dtype=torch.int32, device=dev),
           "masks": torch.zeros((2, CAP, M, M), device=dev)}
    for bad in ([(10, 10)], [(10, 10)] * 3, [(10, 10), (0, 10)], [(10, 10), (10, -1)], [(10, 10), (0.5, 10)], [(10, 10, 3)] * 2,
                [(float("inf"), 10), (10, 10)]):
        with pytest.raises(ValueError):
            result_utils.batch_results(out, bad)
    empty = result_utils.batch_results(out, [(10, 10), (20, 30)])
    assert len(empty) == 2
    for sc, bx, cb, segms in empty:
        assert sc.shape == (0,) and bx.shape == (0, 4) and all(cb[j].shape == (0, 5) for j in range(1, 81))
        assert segms == [[] for _ in range(81)]
    model = _model(params)
    with pytest.raises(TypeError):
        model.detect_images([np.zeros((10, 10), np.uint8)])
    assert len(model._engines) == 0
    c4 = detector(arch='resnet50', use_rpn_head=True, use_mask_head=True, mask_head_type='upshare', roi_height=14, roi_width=14,
                  roi_spatial_scale=0.0625, roi_sampling_ratio=0)
    with pytest.raises(NotImplementedError):
        c4.detect_images(_uint8_images())
    fast = detector(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                    conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], fpn_extra_lvl=True,
                    roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2)
    with pytest.raises(RuntimeError):
        fast.detect_images(_uint8_images())
    assert len(c4._engines) == len(fast._engines) == 0

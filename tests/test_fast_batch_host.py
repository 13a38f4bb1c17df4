"""Host side of batched Fast R-CNN (detect(..., proposals=)): the proposal checks that run before any engine is built, the padded block
Engine.set_proposals uploads, and the bound under which preprocess_sample's float64 duplicate hash is an exact integer.  No GPU needed."""
import numpy as np
import pytest
import torch

FAST_FPN = dict(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
                conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'], roi_height=7, roi_width=7,
                roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2)
BOX = np.array([[0, 0, 10, 10]], np.float32)


def test_pad_proposals():
    from detectorch_b200.engine import pad_proposals
    rng = np.random.RandomState(0)
    boxes = [rng.uniform(0, 100, (n, 4)).astype(np.float32) for n in (3, 0, 7)]
    block, counts = pad_proposals(boxes, 3, 8)
    assert block.shape == (3, 8, 4) and block.dtype == np.float32 and counts.dtype == np.int32
    assert counts.tolist() == [3, 0, 7]
    for b, bx in enumerate(boxes):
        assert np.array_equal(block[b, :len(bx)], bx) and not block[b, len(bx):].any()
    with pytest.raises(ValueError):
        pad_proposals(boxes[:2], 3, 8)
    with pytest.raises(ValueError):
        pad_proposals(boxes, 3, 6)


def test_check_proposals():
    from detectorch_b200.model.detector import detector
    scales = np.array([1.0, 2.0])
    out = detector._check_proposals([BOX, torch.from_numpy(np.zeros((0, 4), np.float32))], scales)
    assert len(out) == 2 and all(o.dtype == np.float32 for o in out) and out[1].shape == (0, 4)
    bad = [(TypeError, (BOX, BOX)[0]), (ValueError, [BOX]), (TypeError, [BOX, BOX.astype(np.float64)]), (TypeError, [BOX, BOX.tolist()]),
           (ValueError, [BOX, BOX.reshape(2, 2)]), (ValueError, [BOX, BOX.reshape(1, 1, 4)]), (ValueError, [BOX, np.zeros((1001, 4), np.float32)]),
           (ValueError, [BOX, np.array([[0, 0, np.inf, 1]], np.float32)]), (ValueError, [BOX, np.array([[5, 0, 4, 1]], np.float32)]),
           (ValueError, [BOX, np.array([[0, 5, 1, 4]], np.float32)])]
    for exc, p in bad:
        with pytest.raises(exc):
            detector._check_proposals(p, scales)
    detector._check_proposals([BOX, np.zeros((1000, 4), np.float32)], scales)
    # the hash bound applies to the scaled coordinate: 8990 * 16 px passes, one cell further does not (image 1 has scale 2)
    lim = detector.FAST_MAX_HASH_COORD * 16
    detector._check_proposals([BOX, np.array([[-lim / 2, 0, lim / 2, 1]], np.float32)], scales)
    for x in (lim / 2 + 8, -lim / 2 - 8):
        with pytest.raises(ValueError):
            detector._check_proposals([BOX, np.array([[min(x, 0), 0, max(x, 0), 1]], np.float32)], scales)


def test_hash_is_exact_within_bound():
    """preprocess_sample.remove_dup_prop hashes r0*1e3 + r1*1e6 + r2*1e9 + r3*1e12 in float64; at the extremes of the accepted range every
    partial sum is an exact integer, so the engine's int64 key has the same equalities and order."""
    from detectorch_b200.model.detector import detector
    m = detector.FAST_MAX_HASH_COORD
    v = np.array([1e3, 1e6, 1e9, 1e12])
    r = np.array([[m, m, m, m], [-m, -m, -m, -m], [m, -m, m, -m], [m - 1, m, m, m], [m, m, m, m - 1]], np.float32)
    exact = r.astype(np.int64) @ np.array([10 ** 3, 10 ** 6, 10 ** 9, 10 ** 12], np.int64)
    assert np.all(np.abs(exact) < 2 ** 53)
    assert np.array_equal(r.dot(v), exact.astype(np.float64)) and np.array_equal(r.dot(v).astype(np.int64), exact)


def test_detect_validates_before_any_engine():
    """On a CPU model every rejected call raises before engine_for (which would refuse a CPU model with RuntimeError)."""
    from detectorch_b200.model.detector import detector
    model = detector(**FAST_FPN)
    img = torch.zeros((2, 3, 64, 96))
    kw = dict(scaling_factor=[1.0, 0.5], image_sizes=[(64, 96), (32, 64)], original_sizes=[(64.0, 96.0), (60.0, 120.0)])
    for exc, p in [(ValueError, [BOX]), (TypeError, [BOX, BOX.astype(np.float16)]), (ValueError, [BOX, np.zeros((3, 5), np.float32)]),
                   (ValueError, [BOX, np.full((1, 4), np.nan, np.float32)]), (ValueError, [BOX, np.zeros((1200, 4), np.float32)]),
                   (ValueError, [BOX, np.array([[0, 0, 3e5, 1]], np.float32)])]:
        with pytest.raises(exc):
            model.detect(img, proposals=p, **kw)
    with pytest.raises(RuntimeError):
        model.detect(img, **kw)                       # the Fast model still needs proposals
    with pytest.raises(RuntimeError, match="CUDA"):
        model.detect(img, proposals=[BOX, BOX], **kw)  # valid: reaches engine_for
    assert len(model._engines) == 0
    with pytest.raises(ValueError):
        detector(**dict(FAST_FPN, use_rpn_head=True)).detect(img, proposals=[BOX, BOX], **kw)
    with pytest.raises(NotImplementedError):
        detector(arch='resnet50').detect(img, proposals=[BOX, BOX])
    with pytest.raises(ValueError):
        detector(**dict(FAST_FPN, use_rpn_head=True)).detect_images([np.zeros((8, 8, 3), np.uint8)], proposals=[BOX])

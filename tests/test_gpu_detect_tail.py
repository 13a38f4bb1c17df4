"""Differential tests of the device detection tail (ST_DETECT: det_class_kernel + det_limit_kernel) on the adversarial and
randomised cases of tests/detect_tail_cases.py.  Each case is teacher-forced into an engine (rois, roi_counts, cls_prob,
bbox_pred, per-image scales and original sizes) and only ST_DETECT runs; every image's rows are compared with
oracle/ref.expected_device: counts, classes and RoI indices exactly, scores bit for bit, boxes bit for bit where the deltas are
zero (within 2e-4 elsewhere: expf against numpy's exp).  On the cases whose result does not depend on the NMS tie order the rows
also equal the reference's own (numpy-order) result."""
import numpy as np
import pytest
import torch

import detect_tail_cases as dtc

pytestmark = pytest.mark.gpu

CASES = dtc.all_cases()
H, W = 128, 160


@pytest.fixture(scope="module")
def engines(built):
    """One engine per (B, R, NC, det_cap) group; engines of one class count share their weights."""
    from detectorch_b200 import engine as E
    from oracle import network as net
    out, by_nc = {}, {}
    for B, R, NC, cap in sorted({c.group for c in CASES}):
        kw = dict(batch=B, height=H, width=W, post_nms_top_n=R, num_classes=NC, det_cap=cap, use_mask=False)
        if NC in by_nc:
            eng = E.Engine(share_weights_with=by_nc[NC], **kw)
        else:
            eng = by_nc[NC] = E.Engine(**kw)
            eng.load_state_dict(net.synthetic_params("resnet50", mask=False, n_classes=NC))
        out[(B, R, NC, cap)] = eng
    return E, out


def _run(E, eng, case):
    dev = eng.device
    eng.set_image_info([(H, W)] * case.B, case.scale, case.orig_hw)
    eng.buffer("rois").copy_(torch.from_numpy(case.rois).to(dev))
    eng.buffer("roi_counts").copy_(torch.from_numpy(case.roi_counts).to(dev))
    eng.buffer("cls_prob").copy_(torch.from_numpy(case.cls_prob).to(dev))
    eng.buffer("bbox_pred").copy_(torch.from_numpy(case.bbox_pred).to(dev))
    eng.run(None, 1.0, E.ST_DETECT, E.ST_DETECT)
    torch.cuda.synchronize()
    return {k: eng.buffer(k).cpu().numpy() for k in ("det_counts", "det_total", "det_classes", "det_roi_idx", "det_scores", "det_boxes")}


def _check(got, b, want, exact, tag):
    cls, idx, sc, bx, total = want
    n = len(sc)
    assert int(got["det_total"][b]) == total, (tag, "det_total", int(got["det_total"][b]), total)
    assert int(got["det_counts"][b]) == n, (tag, "det_counts", int(got["det_counts"][b]), n)
    assert np.array_equal(got["det_classes"][b, :n], cls), (tag, "det_classes")
    assert np.array_equal(got["det_roi_idx"][b, :n], idx), (tag, "det_roi_idx")
    assert np.array_equal(got["det_scores"][b, :n].view(np.uint32), sc.astype(np.float32).view(np.uint32)), (tag, "det_scores")
    if exact:
        assert np.array_equal(got["det_boxes"][b, :n].view(np.uint32), bx.astype(np.float32).view(np.uint32)), (tag, "det_boxes")
    else:
        assert n == 0 or np.abs(got["det_boxes"][b, :n].astype(np.float64) - bx).max() < 2e-4, (tag, "det_boxes")
    assert np.all(got["det_roi_idx"][b, n:] == -1) and not np.any(got["det_scores"][b, n:]), (tag, "rows past det_counts")


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_detection_tail_matches_oracle(engines, case):
    from oracle import ref
    E, eng = engines[0], engines[1][case.group]
    got = _run(E, eng, case)
    for b, want in enumerate(ref.expected_device(case, case.det_cap)):
        _check(got, b, want, case.exact, (case.id, b))
    if case.tie_free:
        for b, want in enumerate(ref.expected_device(case, case.det_cap, tie_order="numpy")):
            _check(got, b, want, case.exact, (case.id, b, "numpy order"))

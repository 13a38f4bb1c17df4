"""The generated detection-tail cases of tests/detect_tail_cases.py, without a GPU: every case has the property it is built to
have under the oracle (an fp32 IoU of exactly 0.5, a tie at the image threshold, more detections than det_cap, poisoned rows past
roi_counts, ...), the stable-order and numpy-order oracles agree on every case declared tie-free, and the cases whose boxes are
not bit-exact keep every IoU away from the NMS threshold.  A generator that silently stopped testing what it claims fails here."""
import numpy as np
import pytest

import detect_tail_cases as dtc
from oracle import ref

CASES = dtc.all_cases()


def _iou(a, b):
    """fp32 IoU in the oracle's operation order (oracle/nms_ref.c): a is the box visited first."""
    f = np.float32
    a, b = np.asarray(a, f), np.asarray(b, f)
    area = lambda d: f(f(f(d[2] - d[0]) + f(1)) * f(f(d[3] - d[1]) + f(1)))
    w = max(f(0), f(f(min(a[2], b[2]) - max(a[0], b[0])) + f(1)))
    h = max(f(0), f(f(min(a[3], b[3]) - max(a[1], b[1])) + f(1)))
    inter = f(w * h)
    return f(inter / f(f(area(a) + area(b)) - inter))


def _decoded(case, b):
    """The oracle's decoded, clipped boxes of image b: [n, 4NC]."""
    R, n = case.R, int(case.roi_counts[b])
    boxes = (case.rois[b, :n, 1:5] / np.float32(case.scale[b])).astype(np.float32)
    return ref.clip_tiled_boxes(ref.bbox_transform(boxes, case.bbox_pred[b * R:b * R + n], (10.0, 10.0, 5.0, 5.0)),
                                np.asarray(case.orig_hw[b], np.float32))


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_case_claims(case):
    assert case.claims or case.family in ("sizes", "classes", "fuzz"), case.id
    for cl in case.claims:
        kind, b = cl[0], cl[1]
        cls, idx, sc, bx, thresh = ref.detection_tail(case, b, "stable")
        if kind in ("kept", "dropped"):
            mine = set(idx[cls == cl[2]].tolist())
            want = set(int(r) for r in cl[3])
            assert (want <= mine) if kind == "kept" else not (want & mine), (case.id, cl, sorted(mine))
        elif kind in ("iou", "iou_rounds"):
            j, ri, rk = cl[2], cl[3], cl[4]
            d = _decoded(case, b)
            assert case.exact and np.array_equal(d[[ri, rk], 4 * j:4 * j + 4], case.rois[b, [ri, rk], 1:5] / case.scale[b]), cl
            a, c = d[ri, 4 * j:4 * j + 4], d[rk, 4 * j:4 * j + 4]
            assert case.cls_prob[b * case.R + ri, j] > case.cls_prob[b * case.R + rk, j], cl
            v = _iou(a, c)
            if kind == "iou_rounds" or cl[5] == "eq":
                assert v == np.float32(0.5), (case.id, cl, v)
            else:
                assert np.float32(0.49) < v < np.float32(0.5), (case.id, cl, v)
            if kind == "iou_rounds":                   # the exact rational IoU is below one half
                ai = [int(x) for x in a]; ci = [int(x) for x in c]
                area = lambda q: (q[2] - q[0] + 1) * (q[3] - q[1] + 1)
                inter = (min(ai[2], ci[2]) - max(ai[0], ci[0]) + 1) * (min(ai[3], ci[3]) - max(ai[1], ci[1]) + 1)
                assert 2 * inter < area(ai) + area(ci) - inter, cl
        elif kind == "count":
            assert len(sc) == cl[2], (case.id, cl, len(sc))
        elif kind == "tie_at_limit":
            assert thresh is not None and np.count_nonzero(sc == thresh) > 1, (case.id, cl)
        elif kind == "overflow":
            assert len(sc) > case.det_cap, (case.id, len(sc))
            lost = np.arange(case.det_cap, len(sc))         # what cutting the reference's list at det_cap would lose
            assert np.any(sc[lost] > thresh), case.id
            e = ref.expected_device(case, case.det_cap)[b]
            assert len(e[2]) == case.det_cap and e[4] == len(sc) and np.all(e[2] >= thresh)
            assert np.count_nonzero(e[2] > thresh) == np.count_nonzero(sc > thresh)
        elif kind == "poison":
            n, R = int(case.roi_counts[b]), case.R
            for a in (case.rois[b, n:, 1:5], case.cls_prob[b * R + n:(b + 1) * R], case.bbox_pred[b * R + n:(b + 1) * R]):
                assert a.size and np.all(~np.isfinite(a) | (np.abs(a) >= 1e29)), (case.id, b)
        else:
            raise AssertionError("unknown claim %r" % (kind,))


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_tie_order_and_margins(case):
    """Tie-free cases: numpy's order and (score desc, RoI asc) give the same detections.  Cases without bit-exact boxes: every
    pair of candidates of a class keeps its fp32 IoU at least 1e-5 away from the NMS threshold 0.5, so that an ulp of expf
    cannot flip a suppression."""
    for b in range(case.B):
        st = ref.detection_tail(case, b, "stable")
        if case.tie_free:
            nu = ref.detection_tail(case, b, "numpy")
            for x, y in zip(st[:4], nu[:4]):
                assert np.array_equal(x, y), (case.id, b)
        if not case.exact:
            d = _decoded(case, b)
            n = int(case.roi_counts[b])
            for j in range(1, case.NC):
                cand = np.flatnonzero(case.cls_prob[b * case.R:b * case.R + n, j] > dtc.THRESH)
                for p in range(len(cand)):
                    for q in range(p + 1, len(cand)):
                        v = _iou(d[cand[p], 4 * j:4 * j + 4], d[cand[q], 4 * j:4 * j + 4])
                        assert abs(float(v) - 0.5) >= 1e-5, (case.id, j, cand[p], cand[q], v)


def test_expected_device_keeps_reference_order():
    """expected_device is the reference's own list whenever it fits, and otherwise that list minus its last ties at the threshold."""
    for case in CASES:
        for b, (cls, idx, sc, bx, total) in enumerate(ref.expected_device(case, case.det_cap)):
            rc, ri, rs, rb, thresh = ref.detection_tail(case, b, "stable")
            assert total == len(rs)
            if total <= case.det_cap:
                assert np.array_equal(cls, rc) and np.array_equal(idx, ri) and np.array_equal(sc, rs) and np.array_equal(bx, rb)
            else:
                key = lambda c, i: c.astype(np.int64) * case.R + i
                assert np.all(np.diff(key(cls, idx)) > 0)                      # class-major, RoI ascending
                dropped = np.setdiff1d(key(rc, ri), key(cls, idx))
                assert len(dropped) == total - case.det_cap and np.all(rs[np.isin(key(rc, ri), dropped)] == thresh)
                assert key(rc, ri)[rs == thresh][-1] in dropped


def test_nms_tie_orders():
    """ref.nms: with unique scores both orders agree; with tied identical boxes the stable order keeps the lowest index."""
    rng = np.random.RandomState(0)
    d = np.concatenate([dtc.clustered_boxes(rng, 200, 5), rng.permutation(200)[:, None] / np.float32(200)], 1).astype(np.float32)
    assert np.array_equal(ref.nms(d, 0.5), ref.nms(d, 0.5, order="stable"))
    t = np.tile(np.array([[10, 10, 49, 49, 0.5]], np.float32), (7, 1))
    assert ref.nms(t, 0.5, order="stable").tolist() == [0]
    with pytest.raises(ValueError):
        ref.nms(t, 0.5, order="unstable")

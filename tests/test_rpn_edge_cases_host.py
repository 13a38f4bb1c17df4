"""The generated RPN proposal cases of tests/rpn_edge_cases.py and the FPN level boundary boxes, without a GPU: every case reaches
the branch of the device's top-k it names (a numpy mirror of float_desc_key and the 11 + 11-bit digit split gives n, K, b1, b2 and
the boundary total), and has the property it is built to have under the oracle (an fp32 IoU of exactly 0.7, widths on min_size,
ties across the cut, empty levels, ...).  The boundary boxes hit the intended float32 areas, on which the oracle's and the
package's map_rois_to_fpn_levels agree.  A generator that silently stopped testing what it claims fails here."""
import numpy as np
import pytest

import rpn_edge_cases as rec
from oracle import ref

CASES = rec.all_cases()
F32 = np.float32


def _iou(a, b):
    """fp32 IoU in the oracle's operation order (oracle/nms_ref.c)."""
    f = F32
    area = lambda d: f(f(f(d[2] - d[0]) + f(1)) * f(f(d[3] - d[1]) + f(1)))
    w = max(f(0), f(f(min(a[2], b[2]) - max(a[0], b[0])) + f(1)))
    h = max(f(0), f(f(min(a[3], b[3]) - max(a[1], b[1])) + f(1)))
    inter = f(w * h)
    return f(inter / f(f(area(a) + area(b)) - inter))


def _iou_matrix(p):
    """fp32 IoU of every pair of boxes p [n, 4], same operation order."""
    p = np.asarray(p, F32)
    area = ((p[:, 2] - p[:, 0] + F32(1)) * (p[:, 3] - p[:, 1] + F32(1))).astype(F32)
    w = np.maximum(F32(0), (np.minimum(p[:, None, 2], p[None, :, 2]) - np.maximum(p[:, None, 0], p[None, :, 0])) + F32(1))
    h = np.maximum(F32(0), (np.minimum(p[:, None, 3], p[None, :, 3]) - np.maximum(p[:, None, 1], p[None, :, 1])) + F32(1))
    inter = (w * h).astype(F32)
    return (inter / ((area[:, None] + area[None, :]).astype(F32) - inter)).astype(F32)


def _decoded(case, b, l):
    """The oracle's clipped boxes of every anchor of (b, l), in anchor order (pre_nms = 0: no top-k, no NMS)."""
    import torch
    h, w = case.net_hw[b]
    p, _, st = ref.generate_proposals_level(torch.from_numpy(case.scores[b][l][None]), torch.from_numpy(case.deltas[b][l][None]), h, w,
                                            float(case.scale[b]), 1.0 / rec.stride(l), (32 << l,), pre_nms_top_n=0, post_nms_top_n=0,
                                            nms_thresh=0, min_size=0, return_stages=True, tie_order="stable")
    box = np.zeros((case.scores[b][l].size, 4), F32)
    box[st["order"]] = p.numpy()
    return box


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_case_claims(case):
    assert case.claims or case.id == "filter-dw_clip", case.id
    exp = rec.expected(case)
    for cl in case.claims:
        kind, b = cl[0], cl[1]
        if kind in ("collect_cut", "cross_level_tie"):
            lv = exp[b][0]
            if kind == "collect_cut":
                assert sum(len(s) for _, s, _ in lv) > case.post, (case.id, cl)
            else:
                vals = [set(s[:, 0].numpy().tolist()) for _, s, _ in lv]
                assert any(vals[i] & vals[j] for i in range(len(vals)) for j in range(i + 1, len(vals))), (case.id, cl)
            continue
        l = cl[2]
        props, scores, st = exp[b][0][l]
        sel = rec.select_stats(case.get_scores(b, l), case.pre)
        if kind == "branch":
            assert sel["branch"] == cl[3], (case.id, cl, {k: v for k, v in sel.items() if k != "keys"})
        elif kind == "total":
            assert sel["total"] == cl[3], (case.id, cl, sel["total"])
        elif kind == "slot":
            keys, K = sel["keys"], sel["K"]
            kth = int(keys[K - 1])
            shift = 21 if cl[3].startswith("bin") else 10
            if cl[3].endswith("first"):
                assert K == 1 or int(keys[K - 2]) >> shift < kth >> shift, (case.id, cl)
                assert kth & ((1 << shift) - 1) == 0, (case.id, cl, hex(kth))
            else:
                assert K == len(keys) or int(keys[K]) >> shift > kth >> shift, (case.id, cl)
                assert kth & ((1 << shift) - 1) == (1 << shift) - 1, (case.id, cl, hex(kth))
            assert int(keys[K - 2]) != kth and int(keys[K]) != kth, "the K-th key is unique"
        elif kind == "tie_cut":
            keys, K = sel["keys"], sel["K"]
            assert K < len(keys) and keys[K - 1] == keys[K], (case.id, cl)
        elif kind == "cands":
            assert len(st["filter_keep"]) == cl[3], (case.id, cl, len(st["filter_keep"]))
        elif kind == "filtered_all":
            assert sel["K"] > 0 and len(st["filter_keep"]) == 0 and len(props) == 0, (case.id, cl)
        elif kind in ("survivors", "survivors_over"):
            _, _, full = rec.oracle_level(case, b, l, post=0)
            k = len(full["nms_keep"])
            assert (k == cl[3]) if kind == "survivors" else (k > cl[3] and len(props) == cl[3]), (case.id, cl, k)
        elif kind == "iou":
            i, j, v = cl[3], cl[4], cl[5]
            d = _decoded(case, b, l)
            assert case.get_scores(b, l)[i] > case.get_scores(b, l)[j]
            assert _iou(d[i], d[j]) == F32(v), (case.id, cl, _iou(d[i], d[j]))
            pos = {int(a): r for r, a in enumerate(st["order"])}
            cand = {int(st["filter_keep"][r]): r for r in range(len(st["filter_keep"]))}
            kept = set(int(st["filter_keep"][r]) for r in st["nms_keep"])
            ri, rj = pos[i], pos[j]
            assert ri in kept and ri in cand and rj in cand, (case.id, cl)
            assert (rj not in kept) == (F32(v) >= F32(rec.NMS)), (case.id, cl)
        elif kind == "edge":
            what, i = cl[3], cl[4]
            d = _decoded(case, b, l)[i]
            ws, hs = F32(d[2] - d[0]) + F32(1), F32(d[3] - d[1]) + F32(1)
            ms = F32(case.min_size * float(case.scale[b]))
            h, w = case.net_hw[b]
            pos = {int(a): r for r, a in enumerate(st["order"])}
            passed = pos[i] in set(st["filter_keep"].tolist())
            if what in ("ws_eq", "hs_eq"):
                assert (ws if what == "ws_eq" else hs) == ms and passed, (case.id, cl, ws, hs, ms)
            elif what in ("ws_below", "hs_below"):
                assert (ws if what == "ws_below" else hs) == ms - 1 and not passed, (case.id, cl, ws, hs, ms)
            elif what == "xc_max":
                assert d[0] == d[2] == w - 1 and F32(d[0] + ws / F32(2)) == F32(w - 0.5) and passed, (case.id, cl, d)
            else:
                assert d[1] == d[3] == h - 1 and F32(d[1] + hs / F32(2)) == F32(h - 0.5) and passed, (case.id, cl, d)
        else:
            raise AssertionError("unknown claim %r" % (kind,))


def test_branches_covered():
    """Every branch of the top-k is reached, in a single-image and in a mixed launch, and every pre_nms edge."""
    seen = set()
    for c in CASES:
        seen |= {(cl[3], c.B > 1) for cl in c.claims if cl[0] == "branch"}
    for br in ("small", "k4", "narrowed", "fallback"):
        assert (br, False) in seen, br
    assert {("small", True), ("narrowed", True), ("fallback", True)} <= seen
    pres = {c.pre for c in CASES}
    assert {1, 63, 64, 65, 127, 128, 129, 3071, 3072, 8192} <= pres and {1, 100} <= {c.post for c in CASES}
    assert {w for c in CASES for cl in c.claims if cl[0] == "slot" for w in [cl[3]]} == {"bin_first", "bin_last", "sub_first", "sub_last"}


@pytest.mark.parametrize("case", [c for c in CASES if not c.exact], ids=lambda c: c.id)
def test_inexact_margins(case):
    """Cases whose boxes are not bit-exact (expf of a non-zero size delta): every candidate pair with such a box keeps its fp32 IoU
    1e-5 away from the NMS threshold, and every such width / height stays 1e-3 away from min_size, so that an ulp of expf cannot flip a
    decision."""
    for b in range(case.B):
        for l in range(rec.LEVELS):
            _, _, st = rec.oracle_level(case, b, l, post=0)
            dl = case.deltas[b][l]
            sized = ((dl[2::4] != 0) | (dl[3::4] != 0)).transpose(1, 2, 0).reshape(-1)
            d = _decoded(case, b, l)[st["order"]]
            inexact = sized[st["order"]]
            ws, hs = d[:, 2] - d[:, 0] + 1, d[:, 3] - d[:, 1] + 1
            ms = case.min_size * float(case.scale[b])
            assert np.all(np.abs(ws - ms)[inexact] > 1e-3) and np.all(np.abs(hs - ms)[inexact] > 1e-3), (case.id, b, l)
            keep = st["filter_keep"]
            if len(keep) > 1 and inexact[keep].any():
                m = _iou_matrix(d[keep])
                pair = inexact[keep][:, None] | inexact[keep][None, :]
                assert np.all(np.abs(m.astype(np.float64) - rec.NMS)[pair] >= 1e-5), (case.id, b, l)


def test_tie_free_cases_match_numpy_order():
    """On levels without equal scores the stable oracle is the reference's own."""
    for case in CASES:
        if any(cl[0] in ("tie_cut", "cross_level_tie", "total") for cl in case.claims) or case.id in ("select-all_equal", "select-fallback",
                                                                                                    "mixed-narrow_fallback"):
            continue
        for l in range(rec.LEVELS):
            st = rec.oracle_level(case, 0, l)
            nu = rec.oracle_level(case, 0, l, tie_order="numpy")
            assert np.array_equal(st[2]["order"], nu[2]["order"]) and np.array_equal(st[0].numpy(), nu[0].numpy()), (case.id, l)


# ------------------------------------------------------------------------------------------------ FPN level boundaries
def test_boundary_boxes_hit_areas():
    areas = rec.boundary_areas()
    assert len(areas) == 3 * (2 * rec.BOUNDARY_ULPS + 1) and len(np.unique(areas)) == len(areas)
    assert set(F32(a) for a in rec.NAMED_AREAS) <= set(areas.tolist())
    boxes = rec.boundary_boxes(areas)
    assert np.array_equal(rec.box_areas(boxes).view(np.uint32), areas.view(np.uint32))
    assert boxes.min() >= 0 and boxes[:, 2:].max() < 512


def test_boundary_levels_agree():
    """The oracle's map_rois_to_fpn_levels and the package's host mirror give the same levels on every boundary box, every level
    changes inside the set, and the named areas sit on either side of their boundary."""
    from detectorch_b200.utils import multilevel_rois
    boxes = rec.boundary_boxes(rec.boundary_areas())
    a = ref.map_rois_to_fpn_levels(boxes, 2, 5)
    b = multilevel_rois.map_rois_to_fpn_levels(boxes, 2, 5)
    assert a.dtype == np.float32 and np.array_equal(a, b)
    n = 2 * rec.BOUNDARY_ULPS + 1
    for k, (lo, hi) in enumerate(((2, 3), (3, 4), (4, 5))):
        seg = a[k * n:(k + 1) * n]
        assert seg[0] == lo and seg[-1] == hi and np.all(np.diff(seg) >= 0)
    named = ref.map_rois_to_fpn_levels(rec.boundary_boxes(np.asarray(rec.NAMED_AREAS, F32)), 2, 5)
    assert named.tolist() == [2, 3, 3, 5, 5]

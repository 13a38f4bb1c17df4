"""Differential tests of the device RPN proposal stage and collect step (ST_PROPOSALS..ST_COLLECT) on the adversarial cases of
tests/rpn_edge_cases.py, and of the FPN level map on boxes at every float32 area around the level boundaries.

Each case's RPN maps are teacher-forced into rpn_out* (the canvas outside each image holds 2.0, a score no real anchor has) and
only the proposal and collect stages run.  Every image and level is compared with oracle/ref.generate_proposals_level with
(score desc, anchor index asc) tie order, the order the device documents: rpn_order exactly, prop_counts exactly, prop_scores bit for
bit, props bit for bit where the size deltas are zero (within 2e-4 elsewhere: expf against torch.exp), the device's top-k plan
(rpn_sel_info) against the numpy mirror of the selection, and rois / roi_levels / roi_counts against collect_and_distribute.
Where the scores have no ties the order is also the reference's own.  Each case runs after a decoy input on the same engine, so
that every checked run reuses the engine's selection histograms.

The FPN level boundary boxes go through all three callers of fpn_level: collect_kernel (teacher-forced props), fast_props_kernel
(pre-computed proposals at scale 1) and mask_rois_kernel (teacher-forced detections); every level must equal
map_rois_to_fpn_levels."""
import numpy as np
import pytest
import torch

import rpn_edge_cases as rec
from test_gpu_fullsize import assert_same_order_up_to_ties

pytestmark = pytest.mark.gpu

CASES = rec.all_cases()
F32 = np.float32
POISON = 2.0


@pytest.fixture(scope="module")
def engines(built):
    """RPN engines on a 256 x 256 canvas, one per (B, pre_nms, post_nms, min_size) group, sharing one set of weights."""
    from detectorch_b200 import engine as E
    from oracle import network as net
    made = {}

    def get(group, canvas=rec.CANVAS):
        key = (group, canvas)
        if key not in made:
            B, pre, post, min_size = group
            kw = dict(batch=B, height=canvas, width=canvas, pre_nms_top_n=pre, post_nms_top_n=post, rpn_min_size=min_size, use_mask=False)
            if not made:
                made["base"] = E.Engine(**kw)
                made["base"].load_state_dict(net.synthetic_params("resnet50", mask=False))
                made[key] = made["base"]
            else:
                made[key] = E.Engine(share_weights_with=made["base"], **kw)
        return made[key]
    get(CASES[0].group)
    return E, get


def _run(E, eng, case):
    dev = eng.device
    eng.set_image_info(case.net_hw, case.scale)
    for l in range(rec.LEVELS):
        o = eng.buffer("rpn_out%d" % (l + 2))
        o.fill_(POISON)
        for b in range(case.B):
            blk = torch.from_numpy(case.rpn_out(b, l))
            o[b, :blk.shape[0], :blk.shape[1], :blk.shape[2]] = blk.to(dev)
    eng.run(None, 1.0, E.ST_PROPOSALS, E.ST_COLLECT)
    torch.cuda.synchronize()
    return {k: eng.buffer(k).cpu().numpy().copy() for k in ("rpn_order", "prop_counts", "props", "prop_scores", "rpn_sel_info", "rois",
                                                         "roi_levels", "roi_counts")}


def _bits(x):
    return np.ascontiguousarray(x, F32).view(np.uint32)


def _check(got, case, tag):
    exp = rec.expected(case)
    for b in range(case.B):
        lv, (rois, lvls) = exp[b]
        for l in range(rec.LEVELS):
            props, scores, st = lv[l]
            t = (tag, b, l)
            order = st["order"]
            sc = case.get_scores(b, l)
            assert np.array_equal(got["rpn_order"][b, l, :len(order)], order), (t, "rpn_order")
            sel = rec.select_stats(sc, case.pre)
            keys, K = sel["keys"], sel["K"]
            if K == len(keys) or keys[K - 1] != keys[K]:        # no run of equal scores across the cut: the reference's own top-k set
                nu = rec.oracle_level(case, b, l, tie_order="numpy")[2]["order"]
                assert_same_order_up_to_ties(got["rpn_order"][b, l, :len(order)], nu, lambda o: sc[o])
            info = got["rpn_sel_info"][b, l]
            if sel["branch"] == "narrowed":
                assert info[:3].tolist() == [sel["b1"], sel["b2"], sel["total"]], (t, "rpn_sel_info", info, sel["total"])
            elif sel["branch"] == "fallback":
                assert info[:2].tolist() == [sel["b1"], sel["b2"]] and info[2] == -1, (t, "rpn_sel_info", info)
            k = len(props)
            assert int(got["prop_counts"][b, l]) == k, (t, "prop_counts", int(got["prop_counts"][b, l]), k)
            assert np.array_equal(_bits(got["prop_scores"][b, l, :k]), _bits(scores[:, 0].numpy())), (t, "prop_scores")
            if case.exact:
                assert np.array_equal(_bits(got["props"][b, l, :k]), _bits(props.numpy())), (t, "props")
            else:
                assert k == 0 or np.abs(got["props"][b, l, :k].astype(np.float64) - props.numpy()).max() <= 2e-4, (t, "props")
        n = len(rois)
        assert int(got["roi_counts"][b]) == n, ((tag, b), "roi_counts", int(got["roi_counts"][b]), n)
        assert np.all(got["rois"][b, :n, 0] == b)
        if case.exact:
            assert np.array_equal(_bits(got["rois"][b, :n, 1:5]), _bits(rois)), ((tag, b), "rois")
        else:
            assert n == 0 or np.abs(got["rois"][b, :n, 1:5].astype(np.float64) - rois).max() <= 2e-4, ((tag, b), "rois")
        assert np.array_equal(got["roi_levels"][b, :n] + 2, lvls.astype(np.int64)), ((tag, b), "roi_levels")
        assert not got["rois"][b, n:, 1:5].any() and not got["roi_levels"][b, n:].any(), ((tag, b), "rows past roi_counts")


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_proposals_match_oracle(engines, case):
    E, get = engines
    eng = get(case.group)
    decoy = case.decoy()
    _check(_run(E, eng, decoy), decoy, decoy.id)
    _check(_run(E, eng, case), case, case.id)


# ------------------------------------------------------------------------------------------------ FPN level boundaries
FB, FCAP, FCANVAS = 4, 1024, 512


def _boundary_chunks(per_run):
    """The boundary boxes (one per float32 area within 4096 ulps of 112^2, 224^2, 448^2), in runs of at most per_run."""
    boxes = rec.boundary_boxes(rec.boundary_areas(), FCANVAS)
    return [boxes[i:i + per_run] for i in range(0, len(boxes), per_run)]


def _want_levels(boxes):
    from oracle import ref
    return ref.map_rois_to_fpn_levels(np.asarray(boxes, F32), 2, 5).astype(np.int64)


def test_fpn_levels_collect(engines):
    """collect_kernel: teacher-forced props (boxes spread over the five RPN levels, distinct scores), ST_COLLECT only."""
    from oracle import ref
    E, get = engines
    eng = get((FB, 1000, FCAP, 0.0), FCANVAS)
    dev = eng.device
    eng.clear_image_info()
    bad = 0
    for chunk in _boundary_chunks(FB * FCAP):
        props = np.zeros((FB, rec.LEVELS, FCAP, 4), F32)
        scores = np.zeros((FB, rec.LEVELS, FCAP), F32)
        counts = np.zeros((FB, rec.LEVELS), np.int32)
        want = []
        for b in range(FB):
            bx = chunk[b * FCAP:(b + 1) * FCAP]
            sc = np.linspace(0.99, 0.01, max(len(bx), 1)).astype(F32)[:len(bx)]
            rl, sl = [], []
            for l in range(rec.LEVELS):
                p, s = bx[l::rec.LEVELS], sc[l::rec.LEVELS]
                props[b, l, :len(p)], scores[b, l, :len(p)], counts[b, l] = p, s, len(p)
                rl.append(torch.from_numpy(p.copy()))
                sl.append(torch.from_numpy(s.copy()[:, None]))
            _, _, rois, lvls = ref.collect_and_distribute(rl, sl, post_nms_top_n=FCAP, stable=True)
            want.append((rois.numpy(), lvls.astype(np.int64)))
        eng.buffer("props").copy_(torch.from_numpy(props).to(dev))
        eng.buffer("prop_scores").copy_(torch.from_numpy(scores).to(dev))
        eng.buffer("prop_counts").copy_(torch.from_numpy(counts).to(dev))
        eng.run(None, 1.0, E.ST_COLLECT, E.ST_COLLECT)
        torch.cuda.synchronize()
        rois_d, lv_d, cnt_d = eng.buffer("rois").cpu().numpy(), eng.buffer("roi_levels").cpu().numpy(), eng.buffer("roi_counts").cpu().numpy()
        for b, (rois, lvls) in enumerate(want):
            n = len(rois)
            assert int(cnt_d[b]) == n
            assert np.array_equal(_bits(rois_d[b, :n, 1:5]), _bits(rois))
            bad += int(np.count_nonzero(lv_d[b, :n] + 2 != lvls))
    assert bad == 0, "collect_kernel: %d boundary RoIs on another FPN level than map_rois_to_fpn_levels" % bad


def test_fpn_levels_fast_props(built):
    """fast_props_kernel: the boxes as pre-computed proposals at scale 1 (moved down by 16 pixels each so that no two share the
    deduplication hash)."""
    from detectorch_b200 import engine as E
    from oracle import network as net
    eng = E.Engine(batch=FB, height=FCANVAS, width=FCANVAS, post_nms_top_n=FCAP, use_rpn=False, use_mask=False)
    eng.load_state_dict(net.synthetic_params("resnet50", mask=False))
    bad = 0
    for chunk in _boundary_chunks(FB * FCAP):
        per = []
        for b in range(FB):
            bx = chunk[b * FCAP:(b + 1) * FCAP].copy()
            off = (16 * np.arange(len(bx))).astype(F32)
            bx[:, 1] += off
            bx[:, 3] += off
            assert np.array_equal(_bits(rec.box_areas(bx)), _bits(rec.box_areas(chunk[b * FCAP:(b + 1) * FCAP])))
            per.append(bx)
        eng.set_proposals(per)
        eng.run(None, 1.0, E.ST_COLLECT, E.ST_COLLECT)
        torch.cuda.synchronize()
        rois_d, lv_d, cnt_d = eng.buffer("rois").cpu().numpy(), eng.buffer("roi_levels").cpu().numpy(), eng.buffer("roi_counts").cpu().numpy()
        for b, bx in enumerate(per):
            n = len(bx)
            assert int(cnt_d[b]) == n
            got = rois_d[b, :n, 1:5]
            key = lambda r: np.lexsort(r.T[::-1])
            assert np.array_equal(_bits(got[key(got)]), _bits(bx[key(bx)]))
            bad += int(np.count_nonzero(lv_d[b, :n] + 2 != _want_levels(got)))
    assert bad == 0, "fast_props_kernel: %d boundary RoIs on another FPN level than map_rois_to_fpn_levels" % bad


def test_fpn_levels_mask_rois(built):
    """mask_rois_kernel: the boxes as teacher-forced detections at scale 1, ST_MASK_ROIS only."""
    from detectorch_b200 import engine as E
    from oracle import network as net
    B = 2
    eng = E.Engine(batch=B, height=FCANVAS, width=FCANVAS, post_nms_top_n=FCAP, det_cap=FCAP, use_mask=True)
    eng.load_state_dict(net.synthetic_params("resnet50"))
    dev = eng.device
    bad = 0
    for chunk in _boundary_chunks(B * FCAP):
        boxes = np.zeros((B, FCAP, 4), F32)
        counts = np.zeros((B,), np.int32)
        for b in range(B):
            bx = chunk[b * FCAP:(b + 1) * FCAP]
            boxes[b, :len(bx)], counts[b] = bx, len(bx)
        eng.buffer("det_boxes").copy_(torch.from_numpy(boxes).to(dev))
        eng.buffer("det_counts").copy_(torch.from_numpy(counts).to(dev))
        eng.run(None, 1.0, E.ST_MASK_ROIS, E.ST_MASK_ROIS)
        torch.cuda.synchronize()
        rois_d = eng.buffer("mask_rois").cpu().numpy().reshape(B, FCAP, 5)
        lv_d = eng.buffer("mask_levels").cpu().numpy().reshape(B, FCAP)
        for b in range(B):
            n = int(counts[b])
            assert np.array_equal(_bits(rois_d[b, :n, 1:5]), _bits(boxes[b, :n]))
            bad += int(np.count_nonzero(lv_d[b, :n] + 2 != _want_levels(boxes[b, :n])))
    assert bad == 0, "mask_rois_kernel: %d boundary RoIs on another FPN level than map_rois_to_fpn_levels" % bad

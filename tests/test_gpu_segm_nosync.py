"""Masks added without a host synchronisation: ops.segm_rle_batch_append (dt_segm_rle_batch_append) and the masked
DeviceResults.add built on it.  The appended strings must be byte-identical to ops.segm_rle_batch, eagerly and replayed from a captured
CUDA graph; every overflow must be flagged and leave the arena as it was; adds must pass under sync-debug mode "error"; and every
evaluation must equal evaluate() on batch_results of the same batches, np.array_equal throughout."""
import numpy as np
import pytest
import torch

import test_gpu_batch_results as tbr
import test_gpu_device_results as tdr

pytestmark = pytest.mark.gpu
NC = tdr.NC


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _five(dev):
    """test_gpu_batch_results' five images (800 x 1216 with 100 detections, boxes crossing every border, the golden case, no live
    detection, every slot live) on the device, with the class-selected masks."""
    masks, boxes, classes, counts, sizes, _ = tbr._kernel_batch()
    tm, tb, tc, tn = (torch.from_numpy(x).to(dev) for x in (masks, boxes, classes, counts))
    B, cap = tm.shape[:2]
    sel = tm[torch.arange(B, device=dev)[:, None], torch.arange(cap, device=dev)[None, :], tc.long()].contiguous()
    return tm, sel, tb, tc, tn, sizes


def _strings(arena, offs, counts, cap):
    """Per image, the appended strings of its live slots (bytes)."""
    a, o = arena.cpu().numpy().tobytes(), offs.cpu().numpy()
    return [[a[o[b * cap + d]:o[b * cap + d + 1]] for d in range(int(n))] for b, n in enumerate(counts)]


def _append(ops, masks, classes, boxes, counts, sizes, dev, base=17, capacity=1 << 22, runs_cap=4096):
    arena = torch.full((capacity,), 0xAB, dtype=torch.uint8, device=dev)
    cursor = torch.tensor([base], dtype=torch.int64, device=dev)
    sz = torch.from_numpy(np.asarray(sizes, np.int32)).to(dev)
    offs, flags = ops.segm_rle_batch_append(masks, classes, boxes, counts, sz, arena, cursor, runs_cap=runs_cap)
    return arena, cursor, offs, flags


def test_append_bytes_equal_segm_rle_batch(dev):
    from detectorch_b200 import ops
    tm, sel, tb, tc, tn, sizes = _five(dev)
    cap = tm.shape[1]
    want = ops.segm_rle_batch(tm, tc, tb, tn, sizes)
    counts = tn.cpu().numpy()
    for masks, classes in ((tm, tc), (sel, None)):
        arena, cursor, offs, flags = _append(ops, masks, classes, tb, tn, sizes, dev)
        o = offs.cpu().numpy()
        total = sum(len(s) for img in want for s in img)
        assert flags.cpu().tolist() == [0, 0, 0]
        assert int(cursor) == 17 + total and o[0] == 17 and o[-1] == 17 + total
        assert _strings(arena, offs, counts, cap) == want
        live = np.zeros((len(counts), cap), bool)
        for b, n in enumerate(counts):
            live[b, :n] = True
        assert np.all(np.diff(o)[~live.reshape(-1)] == 0)                  # dead slots have empty strings
        a = arena.cpu().numpy()
        assert np.all(a[:17] == 0xAB) and np.all(a[17 + total:] == 0xAB)     # nothing written outside the batch's range


def test_append_flags(dev):
    from detectorch_b200 import ops
    tm, sel, tb, tc, tn, sizes = _five(dev)
    cap = tm.shape[1]
    want = ops.segm_rle_batch(tm, tc, tb, tn, sizes)
    total = sum(len(s) for img in want for s in img)
    untouched = lambda arena: bool(torch.all(arena == 0xAB))
    # runs: a slot above runs_cap reports what it needed, nothing is appended; growing to the reported need and redoing gives the strings
    runs_cap = 8
    arena, cursor, offs, flags = _append(ops, sel, None, tb, tn, sizes, dev, runs_cap=runs_cap)
    f = flags.cpu().tolist()
    assert f[0] > runs_cap and f[1:] == [0, 0] and int(cursor) == 17 and untouched(arena)
    while f[0]:
        runs_cap = max(2 * runs_cap, f[0] + 1)
        arena, cursor, offs, flags = _append(ops, sel, None, tb, tn, sizes, dev, runs_cap=runs_cap)
        f = flags.cpu().tolist()
    assert f == [0, 0, 0] and _strings(arena, offs, tn.cpu().numpy(), cap) == want
    # arena: one byte short sets "full" and leaves the cursor (offsets still give the need); the exact size fits
    arena, cursor, offs, flags = _append(ops, sel, None, tb, tn, sizes, dev, capacity=17 + total - 1)
    o = offs.cpu().numpy()
    assert flags.cpu().tolist() == [0, 0, 1] and int(cursor) == 17 and o[-1] - o[0] == total and untouched(arena)
    arena, cursor, offs, flags = _append(ops, sel, None, tb, tn, sizes, dev, capacity=17 + total)
    assert flags.cpu().tolist() == [0, 0, 0] and int(cursor) == 17 + total
    # sizes: an image beyond the tables (or empty) raises the size flag and the batch is not emitted -- not emitted empty
    for bad in ((ops.SEGM_APPEND_MAX_SIDE + 1, 40), (60, ops.SEGM_APPEND_MAX_SIDE + 1), (0, 50)):
        sz = sizes.copy()
        sz[1] = bad
        arena, cursor, offs, flags = _append(ops, sel, None, tb, tn, sz, dev)
        f = flags.cpu().tolist()
        assert f[1] == 1 and f[2] == 0 and int(cursor) == 17 and untouched(arena), bad
    # the largest side is within the tables
    sz = sizes.copy()
    sz[3] = (ops.SEGM_APPEND_MAX_SIDE, ops.SEGM_APPEND_MAX_SIDE)
    _, _, _, flags = _append(ops, sel, None, tb, tn, sz, dev)
    assert flags.cpu().tolist() == [0, 0, 0]


def test_append_in_captured_graph(dev):
    """Captured once, replayed with a changed im_sizes table, counts and cursor: each replay equals segm_rle_batch of its inputs."""
    from detectorch_b200 import ops
    tm, sel, tb, tc, tn, sizes = _five(dev)
    cap = tm.shape[1]
    arena = torch.zeros((1 << 22,), dtype=torch.uint8, device=dev)
    cursor = torch.zeros((1,), dtype=torch.int64, device=dev)
    sz = torch.from_numpy(sizes.astype(np.int32)).to(dev)
    counts = tn.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                               # warm-up outside the capture
        ops.segm_rle_batch_append(tm, tc, tb, counts, sz, arena, cursor)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        offs, flags = ops.segm_rle_batch_append(tm, tc, tb, counts, sz, arena, cursor)
    cases = [(sizes, tn.cpu().numpy(), 0),
             (np.array([[600, 900], [40, 50], [500, 700], [333, 517], [2000, 3000]], np.int64), np.array([100, 10, 3, 0, 57], np.int32), 5),
             (np.array([[800, 1216], [37, 53], [64, 64], [480, 640], [8, 9]], np.int64), np.array([0, 10, 7, 0, 100], np.int32), 1000)]
    for new_sizes, new_counts, base in cases:
        sz.copy_(torch.from_numpy(new_sizes.astype(np.int32)))
        counts.copy_(torch.from_numpy(new_counts))
        cursor.fill_(base)
        g.replay()
        want = ops.segm_rle_batch(tm, tc, tb, counts, new_sizes)
        total = sum(len(s) for img in want for s in img)
        assert flags.cpu().tolist() == [0, 0, 0] and int(cursor) == base + total
        assert _strings(arena, offs, new_counts, cap) == want


# ---------------------------------------------------------------------------------------------------------------- DeviceResults
def _batches(dev, seed, n_batches, B=3, cap=12):
    """n_batches detect()-shaped batches of B images over distinct ids (counts include 0 and cap, two images never added), their
    ground truth and per-image batch_results."""
    from detectorch_b200.utils import result_utils
    rng = np.random.RandomState(seed)
    n = n_batches * B + 2
    ids = [int(v) for v in rng.permutation(np.arange(10, 10 + n)) * 7]
    hw = tdr._sizes(rng, n)
    batches, near = [], []
    for k in range(n_batches):
        part = list(range(k * B, (k + 1) * B))
        counts = [int(v) for v in rng.randint(0, cap + 1, B)]
        counts[k % B] = (0, cap)[k % 2]
        sz = [hw[p] for p in part]
        out = tdr._batch(rng, sz, cap, counts, dev)
        orig = np.array([[h + .25, w + .75] for h, w in sz])
        batches.append((out, [ids[p] for p in part], orig))
        bx, cl = out["boxes"].cpu().numpy(), out["classes"].cpu().numpy()
        for b, p in enumerate(part):
            for d in range(0, counts[b], 2):
                if cl[b, d] <= len(tdr.CATS):
                    near.append((ids[p], tdr.CATS[cl[b, d] - 1]) + tuple(float(v) for v in bx[b, d]))
    ds, gt = tdr._ground_truth(rng, ids, hw, True, near)
    idx = {v: i for i, v in enumerate(gt.img_ids)}
    per_batch = [dict(zip([idx[v] for v in bids], result_utils.batch_results(out, orig, num_classes=NC))) for out, bids, orig in batches]
    return gt, batches, per_batch


def _results(gt, per_batch, upto=None, masks=True):
    res = [tdr._empty() for _ in gt.img_ids]
    for pb in per_batch[:upto]:
        for i, r in pb.items():
            res[i] = r if masks else (r[0], r[1], r[2], [[] for _ in range(NC)])
    return res


def _same(gt, acc, results, types=('bbox', 'segm')):
    from detectorch_b200.utils import coco_eval
    for t in types:
        got = coco_eval.evaluate(gt, acc, t, keep_ious=True)
        want = coco_eval.evaluate(gt, results, t, keep_ious=True)
        tdr._same_eval(got, want)
        assert got.ious.keys() == want.ious.keys() and any(np.any(v > 0) for v in want.ious.values()), t
        for k in want.ious:
            assert np.array_equal(got.ious[k], want.ious[k]), (t, k)


def _small(dev, runs_cap=2, ring=None):
    from detectorch_b200.utils import coco_eval
    acc = coco_eval.DeviceResults(dev)
    acc._MIN_CHARS, acc._MIN_RECORDS, acc._runs_cap = 1, 1, runs_cap
    if ring is not None:
        acc._RING = ring
    return acc


def test_segm_add_does_not_synchronise(dev):
    """Fewer batches than the ring holds, a one-byte arena and runs_cap 2: every batch overflows, is redone, and nothing waits."""
    from detectorch_b200.utils import coco_eval
    gt, batches, per_batch = _batches(dev, 0, coco_eval.DeviceResults._RING - 1)
    acc = _small(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for out, ids, orig in batches:
            acc.add(out, ids, original_sizes=orig, num_classes=NC)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _same(gt, acc, _results(gt, per_batch))
    assert acc._runs_cap > 2 and acc._chars.shape[0] > 1 and not acc._ring


@pytest.mark.parametrize("ring", [1, 2, 4])
def test_ring_wraps(dev, ring):
    """More batches than the ring holds, with overflows forcing redos while later batches are in flight."""
    gt, batches, per_batch = _batches(dev, 1, 9)
    acc = _small(dev, runs_cap=6, ring=ring)
    for out, ids, orig in batches:
        acc.add(out, ids, original_sizes=orig, num_classes=NC)
        assert len(acc._ring) <= ring
    _same(gt, acc, _results(gt, per_batch))
    assert acc._chars.shape[0] < 2 * acc._num_chars


def test_masked_and_bbox_adds_interleaved(dev):
    from detectorch_b200.utils import coco_eval
    gt, batches, per_batch = _batches(dev, 2, 8)
    acc = _small(dev, runs_cap=4, ring=2)
    for k, (out, ids, orig) in enumerate(batches):
        if k % 2:
            out = {n: v for n, v in out.items() if n != "masks"}
        acc.add(out, ids, original_sizes=orig, num_classes=NC)
    _same(gt, acc, _results(gt, per_batch, masks=False), ('bbox',))
    with pytest.raises(ValueError, match="without masks"):
        coco_eval.evaluate(gt, acc, 'segm')


def test_add_after_evaluate(dev):
    gt, batches, per_batch = _batches(dev, 3, 7)
    acc = _small(dev, runs_cap=3, ring=3)
    for out, ids, orig in batches[:4]:
        acc.add(out, ids, original_sizes=orig, num_classes=NC)
    _same(gt, acc, _results(gt, per_batch, upto=4))
    for out, ids, orig in batches[4:]:
        acc.add(out, ids, original_sizes=orig, num_classes=NC)
    _same(gt, acc, _results(gt, per_batch))


def test_add_refuses_images_beyond_the_tables(dev):
    from detectorch_b200 import ops
    from detectorch_b200.utils import coco_eval
    _, batches, _ = _batches(dev, 4, 1)
    out, ids, orig = batches[0]
    acc = coco_eval.DeviceResults(dev)
    big = orig.copy()
    big[1] = (ops.SEGM_APPEND_MAX_SIDE + 1, 30)
    with pytest.raises(ValueError, match="beyond"):
        acc.add(out, ids, original_sizes=big, num_classes=NC)
    assert len(acc) == 0 and not acc._ring
    acc.add({k: v for k, v in out.items() if k != "masks"}, ids, original_sizes=big, num_classes=NC)     # boxes only: no canvas needed


@pytest.fixture(scope="module")
def mask_rcnn(dev):
    from oracle import network as net
    return tdr._model(net.synthetic_params("resnet50"))


def test_pinned_detect_then_add_equals_cocoeval(dev, mask_rcnn):
    """detect() from pinned host batches (the third replays a captured graph), each followed at once by a masked add: equal to
    evaluate() of detect_images' results and to live COCOeval on the notebook's results file."""
    import coco_eval_cases as cc
    from detectorch_b200.utils import blob, coco_eval
    from oracle import cocoapi
    ims, results, ds, gt = tdr._model_case(mask_rcnn)
    staged = []
    for part in ([5, 2], [0, 6], [3, 1]):
        data, sizes, scales, orig = blob.images_to_batch([ims[p] for p in part], 128, 200, canvas=tdr.CANVAS)
        staged.append((data.cpu().pin_memory(), sizes, scales, orig, part))
    torch.cuda.synchronize()
    acc = coco_eval.DeviceResults()
    for pinned, sizes, scales, orig, part in staged:
        out = mask_rcnn.detect(pinned, scaling_factor=scales, image_sizes=sizes, original_sizes=orig)
        acc.add(out, [10 * (p + 1) for p in part], original_sizes=orig)
    all_boxes = [[[] for _ in ims]] + [[r[2][j] for r in results] for j in range(1, 81)]
    all_segms = [[[] for _ in ims]] + [[r[3][j] for r in results] for j in range(1, 81)]
    have_oracle = cocoapi.available()
    mods = cocoapi.load() if have_oracle else None
    for t in ('bbox', 'segm'):
        got = coco_eval.evaluate(gt, acc, t)
        tdr._same_eval(got, coco_eval.evaluate(gt, results, t))
        assert got.stats[0] > 0, t
        if have_oracle:
            E = cc.oracle_eval(mods, ds, all_boxes, all_segms, t)
            for k in ('precision', 'recall', 'scores'):
                assert np.array_equal(got.eval[k], E.eval[k]), (t, k)
            assert np.array_equal(got.stats, np.array(E.stats)), t
    if not have_oracle:
        pytest.skip("reference pycocotools not built (oracle/build_cocoapi.sh): compared with evaluate() of detect_images only")

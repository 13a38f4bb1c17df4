"""Differential tests of the OpenCV-exact device resizes on the edge cases of tests/resize_edge_cases.py, bit for bit against what the
reference's own blob.py and segm_results computed with the real cv2 (tests/golden/resize_edges_golden.npz).

  prep   prep_image_kernel through image_to_blob (fpn_on off and on), prep_im_for_blob, images_to_batch (a ragged batch of the odd-size
         exact 2x down-scales on a fixed canvas) and dt_prep_image at fx a few ulp from 0.5; full-size 1600x2003 @ 800 and 2666x1003
         capped at 1333 (im_scale == 0.5 with an odd side whose half rounds up) against the oracle computed here
  masks  segm_paste_kernel and segm_rle_kernel through segm_paste, segm_rle (counts and strings, class-specific and class-agnostic
         masks, a runs_cap of 2 that forces the grow-and-redo), segm_rle_batch (every image of a mask size in one launch, per-image
         sizes, num_dets trimming, regrow) and segm_rle_batch_append into an arena; the 8192-side table bound of the arena launch at
         1x8192 and 8192x1 (against the oracle) and 8193 (flag raised, arena and cursor untouched)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import resize_edge_cases as rec

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "resize_edges_golden.npz")
SETS = rec.mask_sets()


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def G():
    return np.load(GOLD)


def _fpn_pad(blob):
    h, w = blob.shape[2:]
    out = np.zeros(blob.shape[:2] + (-(-h // 32) * 32, -(-w // 32) * 32), np.float32)
    out[:, :, :h, :w] = blob
    return out


# ------------------------------------------------------------------------------------------------ image pre-processing
@pytest.mark.parametrize("i", range(len(rec.PREP_CASES)), ids=lambda i: "%dx%d@%d,%d" % rec.PREP_CASES[i])
def test_prep_cases(dev, G, i):
    from detectorch_b200.utils import blob as B
    h, w, ts, ms = rec.PREP_CASES[i]
    im, want, scale = rec.prep_image(i, h, w), G["prep%d_blob" % i], float(G["prep%d_scale" % i])
    blob, s = B.image_to_blob(im, target_size=ts, max_size=ms, fpn_on=False)
    assert s == scale and np.array_equal(blob.cpu().numpy(), want)
    blob, s = B.image_to_blob(im, target_size=ts, max_size=ms, fpn_on=True)
    assert s == scale and np.array_equal(blob.cpu().numpy(), _fpn_pad(want))
    ims, scales = B.prep_im_for_blob(im, target_sizes=[ts], max_size=ms)
    assert scales == [scale] and np.array_equal(ims[0].cpu().numpy(), want[0].transpose(1, 2, 0))


def _prep_direct(im, fx, pad, dev):
    """dt_prep_image at a given factor (image_to_blob computes its own) into a blob `pad` pixels larger than the resized image."""
    from detectorch_b200 import _lib
    t = torch.from_numpy(im).to(dev)
    h, w = im.shape[:2]
    oh, ow = rec.cv_round(h * fx), rec.cv_round(w * fx)
    blob = torch.full((3, oh + pad, ow + pad), 7.0, dtype=torch.float32, device=dev)
    means = (ctypes.c_double * 3)(*rec.MEANS)
    ok = _lib.lib().dt_prep_image(ctypes.c_void_p(t.data_ptr()), h, w, ctypes.cast(means, ctypes.c_void_p), float(fx), oh, ow,
                                  ctypes.c_void_p(blob.data_ptr()), oh + pad, ow + pad,
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(ok, "dt_prep_image")
    return blob.cpu().numpy(), oh, ow


@pytest.mark.parametrize("i", range(len(rec.FX_CASES)), ids=lambda i: "%dx%d@%r" % rec.FX_CASES[i])
def test_prep_fx_cases(dev, G, i):
    h, w, fx = rec.FX_CASES[i]
    got, oh, ow = _prep_direct(rec.prep_image(100 + i, h, w), fx, 3, dev)
    assert np.array_equal(got[:, :oh, :ow], G["fx%d_out" % i].transpose(2, 0, 1))
    assert not got[:, oh:].any() and not got[:, :, ow:].any()


def test_images_to_batch_ragged_odd(dev, G):
    """The odd-size exact 2x down-scales of one target size as one ragged batch on a fixed canvas: each slot is its image's blob in the
    top-left corner and zeros elsewhere."""
    from detectorch_b200.utils import blob as B
    idx = [i for i, (h, w, ts, ms) in enumerate(rec.PREP_CASES) if (ts, ms) == (8, 1333)]
    assert len(idx) >= 6
    ims = [rec.prep_image(i, *rec.PREP_CASES[i][:2]) for i in idx]
    blob, sizes, scales, orig = B.images_to_batch(ims, target_size=8, max_size=1333, canvas=(64, 96))
    got = blob.cpu().numpy()
    for b, i in enumerate(idx):
        want = G["prep%d_blob" % i][0]
        oh, ow = want.shape[1:]
        assert float(scales[b]) == float(G["prep%d_scale" % i]) and tuple(orig[b].tolist()) == rec.PREP_CASES[i][:2]
        assert tuple(sizes[b].tolist()) == (-(-oh // 32) * 32, -(-ow // 32) * 32)
        assert np.array_equal(got[b, :, :oh, :ow], want), i
        assert not got[b, :, oh:].any() and not got[b, :, :, ow:].any(), i


@pytest.mark.parametrize("case", rec.FULL_CASES, ids=lambda c: "%dx%d" % c[:2])
def test_prep_full_size_half_scale(dev, case):
    from detectorch_b200.utils import blob as B
    from oracle import ref
    h, w, ts, ms = case
    im = rec.prep_image(0, h, w, seed=3)
    ims, scales = ref.prep_im_for_blob(im, target_sizes=[ts], max_size=ms)
    blob, s = B.image_to_blob(im, target_size=ts, max_size=ms, fpn_on=True)
    assert s == scales[0] == 0.5
    assert np.array_equal(blob.cpu().numpy(), ref.im_list_to_blob(ims, fpn_on=True))


# ------------------------------------------------------------------------------------------------ mask paste + RLE
def _want(G, s):
    bits = np.unpackbits(G[s.tag + "_bits"], axis=1)[:, :s.H * s.W].reshape(s.D, s.H, s.W)
    raw, off = G[s.tag + "_rle"].tobytes(), G[s.tag + "_rle_off"]
    return bits, [raw[off[d]:off[d + 1]] for d in range(s.D)]


@pytest.mark.parametrize("s", SETS, ids=lambda s: s.tag)
def test_segm_cases(dev, G, s):
    from detectorch_b200 import ops
    from oracle import ref
    bits, strings = _want(G, s)
    tm, tc, tb = (torch.from_numpy(a).to(dev) for a in (s.masks, s.cls, s.boxes))
    assert np.array_equal(ops.segm_paste(tm, tc, tb, s.H, s.W).cpu().numpy(), bits)
    counts, got = ops.segm_rle(tm, tc, tb, s.H, s.W)
    assert got == strings
    for d in range(s.D):
        assert np.array_equal(counts[d], ref.rle_encode(bits[d])), d
    sel = torch.from_numpy(np.ascontiguousarray(s.selected())).to(dev)
    assert ops.segm_rle(sel, None, tb, s.H, s.W, runs_cap=2)[1] == strings          # class-agnostic planes, grow-and-redo
    assert np.array_equal(ops.segm_paste(sel, None, tb, s.H, s.W).cpu().numpy(), bits)


def _batch(sets, cap):
    """Mask sets as one padded batch: masks [B, cap, K, M, M], classes, boxes (dead slots hold a full-image box of ones)."""
    B, K, M = len(sets), max(s.K for s in sets), sets[0].M
    masks = np.ones((B, cap, K, M, M), np.float32)
    cls = np.ones((B, cap), np.int32)
    boxes = np.zeros((B, cap, 4), np.float32)
    for b, s in enumerate(sets):
        masks[b, :s.D, :s.K] = s.masks
        cls[b, :s.D] = s.cls
        boxes[b, :s.D] = s.boxes
        boxes[b, s.D:] = [0, 0, s.W - 1, s.H - 1]
    return masks, cls, boxes


@pytest.mark.parametrize("M", rec.MASK_SIZES)
def test_segm_batch_and_append(dev, G, M):
    """Every image of one mask size in one launch of segm_rle_batch (per-image canvas sizes, num_dets trimming three images, runs_cap 2
    forcing the regrow) and of segm_rle_batch_append into an arena behind existing bytes."""
    from detectorch_b200 import ops
    from oracle import ref
    sets = [s for s in SETS if s.M == M]
    cap = max(s.D for s in sets) + 2
    masks, cls, boxes = _batch(sets, cap)
    nd = np.array([s.D - (3 if b % 3 == 1 else 0) for b, s in enumerate(sets)], np.int32)
    want = [_want(G, s)[1][:nd[b]] for b, s in enumerate(sets)]
    tm, tc, tb, tn = (torch.from_numpy(a).to(dev) for a in (masks, cls, boxes, nd))
    sizes = np.array([[s.H, s.W] for s in sets], np.int32)
    assert ops.segm_rle_batch(tm, tc, tb, tn, sizes) == want
    assert ops.segm_rle_batch(tm, tc, tb, tn, sizes, runs_cap=2) == want
    runs = max(len(ref.rle_encode(m)) for b, s in enumerate(sets) for m in _want(G, s)[0][:nd[b]])
    total = sum(len(x) for w in want for x in w)
    prefix = b"prefix"
    arena = torch.zeros((len(prefix) + total + 64,), dtype=torch.uint8, device=dev)
    arena[:len(prefix)] = torch.frombuffer(bytearray(prefix), dtype=torch.uint8).to(dev)
    cursor = torch.tensor([len(prefix)], dtype=torch.int64, device=dev)
    ts = torch.from_numpy(sizes).to(dev)
    before = arena.clone()
    offs, flags = ops.segm_rle_batch_append(tm, tc, tb, tn, ts, arena, cursor, runs_cap=runs - 1)    # one run short: flagged
    assert flags.cpu().tolist()[0] >= runs and torch.equal(arena, before) and int(cursor.item()) == len(prefix)
    offs, flags = ops.segm_rle_batch_append(tm, tc, tb, tn, ts, arena, cursor, runs_cap=runs)
    assert flags.cpu().tolist() == [0, 0, 0] and int(cursor.item()) == len(prefix) + total
    a, o = arena.cpu().numpy().tobytes(), offs.cpu().numpy()
    assert a[:len(prefix)] == prefix and not any(a[len(prefix) + total:])
    for b in range(len(sets)):
        got = [a[o[b * cap + d]:o[b * cap + d + 1]] for d in range(cap)]
        assert got[:nd[b]] == want[b] and all(x == b"" for x in got[nd[b]:]), sets[b].tag


def test_segm_bounded_table_limits(dev):
    """segm_rle_batch_append's tables hold a side of 8192: 1x8192 and 8192x1 images encode as the oracle does; a side of 8193 raises
    flags[1] and leaves the arena and the cursor as they were."""
    from detectorch_b200 import ops
    from oracle import ref
    M, n = 28, 8192
    rng = np.random.RandomState(8192)
    rows = []
    for (H, W) in ((1, n), (n, 1)):
        L = max(H, W) - 1
        spans = [(0, L), (0, 0), (L, L), (100.5, 4000.25), (L - 40.5, L), (3.0, 3.0 + 30 * M)]
        bx = [[a, 0, b, 0] if H == 1 else [0, a, 0, b] for a, b in spans]
        rows.append((H, W, np.asarray(bx, np.float32)))
    D = len(rows[0][2])
    masks = np.stack([rec.make_mask(("ones", "checker", "uniform", "eighths", "checker", "half")[d], M, rng) for d in range(D)])
    masks = np.stack([masks, masks[::-1]]).astype(np.float32)                          # [2, D, M, M]
    boxes = np.stack([r[2] for r in rows])
    want = []
    for b, (H, W, bx) in enumerate(rows):
        e = rec.expand(M, bx)
        want.append([ref.rle_to_string(ref.rle_encode(ref.paste_mask(masks[b, d], e[d], H, W))) for d in range(D)])
    tm, tb = torch.from_numpy(masks).to(dev), torch.from_numpy(boxes).to(dev)
    tn = torch.full((2,), D, dtype=torch.int32, device=dev)
    arena = torch.zeros((1 << 16,), dtype=torch.uint8, device=dev)
    cursor = torch.zeros((1,), dtype=torch.int64, device=dev)
    sizes = torch.tensor([[1, n], [n, 1]], dtype=torch.int32, device=dev)
    offs, flags = ops.segm_rle_batch_append(tm, None, tb, tn, sizes, arena, cursor)
    assert flags.cpu().tolist() == [0, 0, 0]
    a, o = arena.cpu().numpy().tobytes(), offs.cpu().numpy()
    assert [[a[o[b * D + d]:o[b * D + d + 1]] for d in range(D)] for b in range(2)] == want
    assert int(cursor.item()) == sum(len(x) for w in want for x in w)
    for big in ([[1, n + 1], [n, 1]], [[1, n], [n + 1, 1]]):
        before, cur = arena.clone(), int(cursor.item())
        offs, flags = ops.segm_rle_batch_append(tm, None, tb, tn, torch.tensor(big, dtype=torch.int32, device=dev), arena, cursor)
        assert flags.cpu().tolist()[1] == 1 and torch.equal(arena, before) and int(cursor.item()) == cur, big

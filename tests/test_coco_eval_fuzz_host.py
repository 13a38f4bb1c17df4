"""Host side of the device COCO evaluation on the generated cases of tests/coco_eval_fuzz_cases.py, without a GPU: _flatten_results
equals the notebooks' results file row for row (and, where oracle/build_cocoapi.sh has built it, what the reference's COCO.loadRes
makes of that file): keys, scores, boxes, RLE strings, sizes and order.  Also the host's decoding of RLE string sums."""
import numpy as np
import pytest

import coco_eval_cases as cc
import coco_eval_fuzz_cases as fz

CASES = [(f, None) for f in fz.FAMILIES] + [('mixed', s) for s in (0, 7, 13, 21)]


def _encode():
    from oracle import cocoapi, ref
    if cocoapi.available():
        mask = cocoapi.load()[2]
        return lambda m: mask.encode(np.asfortranarray(m[:, :, None]))[0]['counts'].decode()
    return lambda m: ref.rle_to_string(ref.rle_encode(m)).decode()


def _case(family, seed):
    return fz.make_mixed_case(seed, _encode()) if family == 'mixed' else fz.make_case(family, 0, _encode())


def _bbox_gt(ds):
    from detectorch_b200.utils import coco_eval
    d = dict(ds, annotations=[{k: v for k, v in a.items() if k != 'segmentation'} for a in ds['annotations']])
    return coco_eval.CocoGroundTruth(d, device='cpu')


@pytest.mark.parametrize("family,seed", CASES)
def test_flatten_equals_results_file(family, seed):
    from detectorch_b200.utils import coco_eval
    from oracle import cocoapi
    ds, boxes, segms = _case(family, seed)
    gt = _bbox_gt(ds)
    for t in ('bbox', 'segm'):
        res = cc.results_file(ds, boxes, segms, t)
        if cocoapi.available():
            COCO = cocoapi.load()[0]
            g = COCO()
            g.dataset = dict(ds)
            import contextlib
            import io
            with contextlib.redirect_stdout(io.StringIO()):
                g.createIndex()
                res = g.loadRes(res).dataset['annotations']
            assert [r['id'] for r in res] == list(range(1, len(res) + 1))
        key = np.array([gt.cat_ids.index(r['category_id']) * gt.num_images + gt.img_ids.index(r['image_id']) for r in res])
        order = np.argsort(key, kind='stable')                # COCOeval's per-pair lists keep file order
        k, f, i, chars = coco_eval._flatten_results(gt, boxes, segms, t, gt.category_ids)
        assert len(k) == len(res) and np.array_equal(k, key[order]), (family, t)
        assert np.array_equal(f[:, 0], np.array([res[n]['score'] for n in order], np.float64)), (family, t)
        if t == 'bbox':
            assert np.array_equal(f[:, 1:], np.array([res[n]['bbox'] for n in order], np.float64)), family
        else:
            assert [chars[a:a + b] for a, b in i[:, :2]] == [res[n]['segmentation']['counts'].encode() for n in order], family
            assert np.array_equal(i[:, 2:], np.array([res[n]['segmentation']['size'] for n in order])), family


def test_string_sums_equal_decoded_counts():
    """_string_sums == the sum of rleFrString's uint32 counts (oracle/ref.rle_from_string), for strings with negative deltas,
    6-char values and zero runs, and for counts that do not sum to a mask."""
    from detectorch_b200.utils import coco_eval
    from oracle import ref
    rng = np.random.RandomState(4)
    strs, want = [], []
    for n in range(300):
        m = int(rng.randint(0, 40))
        c = rng.randint(0, [3, 300, 2 ** 20, 2 ** 28][n % 4], m)
        c[rng.rand(m) < .1] = 0
        s = ref.rle_to_string(c)
        strs.append(s)
        want.append(sum(int(v) for v in ref.rle_from_string(s)))
    lens = np.array([len(s) for s in strs])
    buf = b"".join(strs)
    coco_eval._check_strings(buf, lens, "test")
    assert np.array_equal(coco_eval._string_sums(buf, lens), np.array(want, np.int64))


def test_string_sums_wrap_in_uint32(monkeypatch):
    """A negative delta that takes a running count below zero: rleFrString's (uint) cast wraps it, and the sum counts the wrapped
    value.  Without the wrap these runs would sum to 5 and pass for a 1 x 5 mask."""
    from detectorch_b200.utils import coco_eval
    from oracle import ref
    s = ref.rle_to_string([5, 3, 2, -7, 2])          # deltas 5, 3, 2, -10, 0: count 3 = 3 - 10 -> 2^32 - 7, count 4 = 2 + 0
    assert s == b"532F0"
    want = 5 + 3 + 2 + (2 ** 32 - 7) + 2
    for blk in (1 << 20, 2):
        monkeypatch.setattr(coco_eval, "_SUM_BLOCK_CHARS", blk)
        assert list(coco_eval._string_sums(s + b"1" + s, np.array([len(s), 1, len(s)]))) == [want, 1, want]
    with pytest.raises(ValueError):
        coco_eval._check_sums(coco_eval._string_sums(s, np.array([len(s)])), 1, 5, "test")

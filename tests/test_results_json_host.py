"""Host side of the results json writer (coco_eval.write_results): malformed input is refused before anything is launched or
written; and the test restatement of the reference's writers (results_json_cases) is pinned against the reference's own, where
they are staged (oracle/_ref)."""
import numpy as np
import pytest

import results_json_cases as rj


def _gt():
    from detectorch_b200.utils import coco_eval
    return coco_eval.CocoGroundTruth(dict(images=[dict(id=1, height=10, width=10)], categories=[dict(id=5)]), device='cpu')


GOOD = np.array([[1, 1, 5, 5, .5]], np.float32)
BAD = [
    ([[[]], [np.array([[1, 1, np.nan, 5, .5]])]], 'bbox', None),
    ([[[]], [np.array([[1, 1, 5, 5, -np.inf]])]], 'bbox', None),
    ([[[]], [GOOD[:, :4]]], 'bbox', None),
    ([[[]], [GOOD, GOOD]], 'bbox', None),
    ([[[]], [GOOD]], 'segm', None),
    ([[[]], [GOOD]], 'segm', [[[]], [[{'size': [10, 10], 'counts': 'L9', 'extra': 0}]]]),
    ([[[]], [GOOD]], 'segm', [[[]], [[{'size': [10, 10], 'counts': b'L9'}]]]),
    ([[[]], [GOOD]], 'segm', [[[]], [[{'size': [10, True], 'counts': 'L9'}]]]),
    ([[[]], [GOOD]], 'segm', [[[]], [[{'size': [10, 10], 'counts': 'L9~'}]]]),
    ([[[]], [GOOD]], 'segm', [[[]], [[]]]),
]


@pytest.mark.parametrize("case", range(len(BAD)))
def test_refused_before_launch(tmp_path, monkeypatch, case):
    from detectorch_b200 import _lib
    from detectorch_b200.utils import coco_eval

    def no_launch():
        raise AssertionError("a kernel was reached")
    monkeypatch.setattr(_lib, "lib", no_launch)
    results, t, segms = BAD[case]
    p = tmp_path / "r.json"
    p.write_bytes(b"keep")
    with pytest.raises(ValueError):
        coco_eval.write_results(_gt(), results, t, str(p), segms)
    assert p.read_bytes() == b"keep"
    with pytest.raises(ValueError):
        coco_eval.write_results(_gt(), results, t, str(tmp_path / "new.json"), segms)
    assert sorted(x.name for x in tmp_path.iterdir()) == ["r.json"]


def test_bad_arguments(tmp_path):
    from detectorch_b200.utils import coco_eval
    with pytest.raises(ValueError):
        coco_eval.write_results(_gt(), [[[]], [GOOD]], 'keypoints', str(tmp_path / "r.json"))
    with pytest.raises(TypeError):
        coco_eval.write_results(object(), [[[]], [GOOD]], 'bbox', str(tmp_path / "r.json"))
    with pytest.raises(ValueError):
        coco_eval.write_results(_gt(), [[[]], [GOOD]], 'bbox', str(tmp_path / "r.json"), category_ids=[6])
    assert not list(tmp_path.iterdir())


def test_restatement_equals_reference_writers(tmp_path):
    from oracle import cython_bbox
    if not cython_bbox.available():
        pytest.skip("the reference's writers are not staged under oracle/_ref")
    jde = cython_bbox.load()[0]
    rng = np.random.RandomState(0)
    ids, cats = [9, 4, 7], [3, 8]
    boxes = [[[] for _ in ids]] + [[rng.rand(int(rng.randint(0, 4)), 5).astype(np.float32) * 100 for _ in ids] for _ in cats]
    boxes[1][1] = []
    segms = [[[{'size': [5, 6], 'counts': '0' + chr(48 + k)} for k in range(len(b))] if len(b) else [] for b in c] for c in boxes]
    jd = rj.FakeJsonDataset(ids, cats)
    for t in ('bbox', 'segm'):
        p = str(tmp_path / ("%s.json" % t))
        if t == 'bbox':
            jde._write_coco_bbox_results_file(jd, boxes, p)
        else:
            jde._write_coco_segms_results_file(jd, boxes, segms, p)
        with open(p, "rb") as f:
            assert f.read() == rj.reference_text(ids, cats, boxes, segms, t)

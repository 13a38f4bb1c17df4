"""CPU checks of the proposal-recall host side: malformed roidbs, unknown areas and bad limits raise ValueError before anything is
launched; the roidb flattening selects the rows the reference selects; the proposals pickle has the reader's keys and id order."""
import pickle

import numpy as np
import pytest

import proposal_recall_cases as cases


def test_unknown_area_raises():
    from detectorch_b200.utils import coco_eval, json_dataset_evaluator as jde
    roidb = [cases.random_entry(np.random.RandomState(0), 5, 2)]
    with pytest.raises(ValueError):
        jde.evaluate_box_proposals(None, roidb, area='huge')
    with pytest.raises(ValueError):
        coco_eval.box_proposal_recall(roidb, areas=['all', 'tiny'])


@pytest.mark.parametrize("limit", [-1, 2.5, True, "10"])
def test_bad_limit_raises(limit):
    from detectorch_b200.utils import coco_eval
    with pytest.raises(ValueError):
        coco_eval.box_proposal_recall([cases.random_entry(np.random.RandomState(0), 5, 2)], limits=[limit])


def _bad_entries():
    e = cases.random_entry(np.random.RandomState(1), 6, 3)
    out = []
    for k, v in (('boxes', e['boxes'][:, :3]), ('gt_classes', e['gt_classes'][:-1]), ('gt_classes', e['gt_classes'].astype(np.float32)),
                 ('is_crowd', e['is_crowd'][:-1]), ('seg_areas', e['seg_areas'].astype(np.float16)), ('seg_areas', e['seg_areas'][:2])):
        d = dict(e)
        d[k] = v
        out.append(d)
    for bad in (np.nan, np.inf, 1e20):
        d = dict(e)
        d['boxes'] = e['boxes'].copy()
        d['boxes'][4, 2] = bad
        out.append(d)
    d = dict(e)
    del d['seg_areas']
    out.append(d)
    out.append("not an entry")
    return out


@pytest.mark.parametrize("i", range(len(_bad_entries())))
def test_malformed_entries_raise(i):
    from detectorch_b200.utils import coco_eval
    good = cases.random_entry(np.random.RandomState(2), 4, 2)
    with pytest.raises(ValueError):
        coco_eval.box_proposal_recall([good, _bad_entries()[i]])


def test_tables_select_the_reference_rows():
    from detectorch_b200.utils import coco_eval
    roidb = cases.random_roidb(3, 12)
    prop_off, props, gt_off, gts, gt_area = coco_eval._proposal_tables(roidb)
    for i, e in enumerate(roidb):
        g = np.where((e['gt_classes'] > 0) & (e['is_crowd'] == 0))[0]
        p = np.where(e['gt_classes'] == 0)[0]
        assert np.array_equal(gts[gt_off[i]:gt_off[i + 1]], e['boxes'][g].astype(np.float32))
        assert np.array_equal(gt_area[gt_off[i]:gt_off[i + 1]], e['seg_areas'][g].astype(np.float64))
        assert np.array_equal(props[prop_off[i]:prop_off[i + 1]], e['boxes'][p].astype(np.float32))


def test_proposals_file_layout(tmp_path):
    from detectorch_b200.utils import proposal_file
    rng = np.random.RandomState(0)
    ids = [9, 2, 5]
    props = [(rng.rand(n, 4).astype(np.float32), rng.rand(n).astype(np.float32)) for n in (3, 0, 5)]
    path = str(tmp_path / "p.pkl")
    proposal_file.write_proposals_file(path, ids, props)
    with open(path, "rb") as f:
        d = pickle.load(f, encoding='latin1')
    assert set(d) == {'boxes', 'scores', 'ids'} and d['ids'] == [2, 5, 9]
    for k, i in enumerate(d['ids']):
        j = ids.index(i)
        assert np.array_equal(d['boxes'][k], props[j][0]) and np.array_equal(d['scores'][k], props[j][1])
    with pytest.raises(ValueError):
        proposal_file.write_proposals_file(path, [1, 1, 2], props)
    with pytest.raises(ValueError):
        proposal_file.write_proposals_file(path, [1, 2], props)
    with pytest.raises(ValueError):
        proposal_file.write_proposals_file(path, [1], [(np.zeros((2, 4)), np.zeros(3))])

"""CPU test of the Detectron caffe2-pickle weight import (SURVEY.md 8f "next" row 2): a synthetic pickle written with the
reference's own blob names loads identically into the reference detector and into the detectorch_b200 mirror, for the
constructor kwargs of every eval_*.ipynb notebook (Fast / Faster / Mask R-CNN on the C4 and on the FPN body: the loader
branches on use_rpn_head / use_fpn_body / mask_head_type / two_layer_mlp exactly like detector.py:317-374).
The reference side (its utils.utils.parse_th_to_caffe2 name mapping, its detector's trunk keys, and what its loader read from the
pickle) is stored in tests/golden/ref_golden.npz by tests/golden/make_ref_golden.py."""
import os

import numpy as np
import pytest
import torch

import ref_cases as rc
from oracle import network as net

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_golden.npz")


@pytest.fixture(scope="module")
def G():
    return np.load(GOLD)


@pytest.mark.parametrize("name", sorted(rc.CONFIGS))
def test_detectron_pickle_loads_like_the_reference(tmp_path, built, G, name):
    from detectorch_b200.model.detector import detector as b200_detector
    kw, flags = rc.CONFIGS[name]
    P = net.synthetic_params("resnet50", **flags)
    trunk = [str(k) for k in G["pkl_%s_trunk" % name]]
    layout = {"trunk": trunk, "c2": dict(zip(trunk, [str(c) for c in G["pkl_%s_trunk_c2" % name]])), "fpn": [str(c) for c in G["pkl_%s_fpn" % name]]}
    pkl = os.path.join(str(tmp_path), "model_final.pkl")
    rc.write_detectron_pickle(pkl, layout, P, flags)
    mine = b200_detector(detector_pkl_file=pkl, **kw)                   # exactly the notebook's cell 7
    sm = mine.state_dict()
    # the reference loader read the same pickle into exactly these parameters (names, shapes, bit-pattern sums, leading values)
    keys = [str(k) for k in G["pkl_%s_keys" % name]]
    assert keys == sorted(P)
    for i, k in enumerate(keys):
        v = P[k]
        assert list(G["pkl_%s_shapes" % name][i][:v.dim()]) == list(v.shape), "reference loader: " + k
        assert int(G["pkl_%s_bitsums" % name][i]) == rc.bitsum(v), "reference loader: " + k
        assert np.array_equal(G["pkl_%s_head" % name][i], rc.head8(v), equal_nan=True), "reference loader: " + k
        assert torch.equal(sm[k], v), "mirror loader: " + k
    # and the engine's parameter table accepts exactly these names
    from detectorch_b200 import engine
    t = engine.param_table("resnet50", use_mask=flags["mask"], model="fpn" if flags["fpn"] else "c4", use_rpn=flags["rpn"])
    assert set(t) == set(P) and all(t[k] == int(np.prod(P[k].shape)) for k in P)


def test_caffe2_blob_names_match_the_reference_helper(G):
    """The mirror's own torchvision-name -> caffe2-blob-name mapping equals utils/utils.py:44-71 (parse_th_to_caffe2) on every trunk key."""
    import torchvision.models as models
    from detectorch_b200.model.detector import caffe2_blob_name
    for arch in ("resnet50", "resnet101"):
        keys = [k for k in getattr(models, arch)().state_dict().keys() if not ('running' in k or 'fc' in k or 'num_batches' in k)]
        assert len(keys) > 150 and keys == [str(k) for k in G["name_%s_th" % arch]]
        for k, want in zip(keys, G["name_%s_c2" % arch]):
            assert caffe2_blob_name(k) == str(want), k

"""The OpenCV-exact resizes of the oracle on the edge cases of tests/resize_edge_cases.py, without a GPU: bit for bit against the
fixture the reference's own blob.py and segm_results produced with the real cv2 (tests/golden/make_resize_edges_golden.py); against
the live reference on fresh seeds where it is importable; and oracle.resize_linear_f32_scale against a live cv2.resize(fx=...) sweep of
odd and even sizes at fx = 0.5 and around it.  The cases are also checked to reach the edges they are built for, so that a generator
that silently stopped testing them fails here."""
import os

import numpy as np
import pytest

import resize_edge_cases as rec
from oracle import ref
from oracle import reference_shim as rs

GOLD = os.path.join(os.path.dirname(__file__), "golden", "resize_edges_golden.npz")
SETS = rec.mask_sets()


@pytest.fixture(scope="module")
def G():
    return np.load(GOLD)


def _unbits(G, s):
    return np.unpackbits(G[s.tag + "_bits"], axis=1)[:, :s.H * s.W].reshape(s.D, s.H, s.W)


def _strings(G, s):
    raw, off = G[s.tag + "_rle"].tobytes(), G[s.tag + "_rle_off"]
    return [raw[off[d]:off[d + 1]].decode() for d in range(s.D)]


def test_fixture_matches_cases(G):
    assert G["prep_cases"].tolist() == [list(c) for c in rec.PREP_CASES]
    assert np.array_equal(G["fx_cases"], np.asarray(rec.FX_CASES, np.float64))
    assert G["mask_tags"].tolist() == [s.tag for s in SETS]
    for s in SETS:
        assert G[s.tag + "_digest"] == s.digest(), s.tag


@pytest.mark.parametrize("i", range(len(rec.PREP_CASES)), ids=lambda i: "%dx%d@%d,%d" % rec.PREP_CASES[i])
def test_prep_oracle_matches_fixture(G, i):
    h, w, ts, ms = rec.PREP_CASES[i]
    ims, scales = ref.prep_im_for_blob(rec.prep_image(i, h, w), target_sizes=[ts], max_size=ms)
    assert scales[0] == float(G["prep%d_scale" % i])
    assert np.array_equal(ref.im_list_to_blob(ims), G["prep%d_blob" % i])


@pytest.mark.parametrize("i", range(len(rec.FX_CASES)), ids=lambda i: "%dx%d@%r" % rec.FX_CASES[i])
def test_fx_oracle_matches_fixture(G, i):
    h, w, fx = rec.FX_CASES[i]
    got = ref.resize_linear_f32_scale(rec.fx_input(rec.prep_image(100 + i, h, w)), fx)
    assert np.array_equal(got, G["fx%d_out" % i])


@pytest.mark.parametrize("s", SETS, ids=lambda s: s.tag)
def test_mask_oracle_matches_fixture(G, s):
    pasted, strings = rec.oracle_segm(s)
    assert np.array_equal(pasted, _unbits(G, s))
    assert strings == _strings(G, s)
    for d in range(s.D):
        assert np.array_equal(ref.rle_from_string(strings[d]), ref.rle_encode(pasted[d])), (s.tag, d)


def test_prep_cases_reach_their_edges():
    """Exact 0.5 scales with an odd side whose half rounds up and one whose half rounds down, from the target size and from the
    max_size cap; 1xN, Nx1, 1x1; a 50x up-scale; ordinary down-scales; fx cases a few ulp from 0.5 that are not area-fast."""
    from detectorch_b200.utils import blob as B
    up = down = capped = 0
    for (h, w, ts, ms) in rec.PREP_CASES:
        s, oh, ow, _, _ = B.blob_geometry((h, w), ts, ms)
        if s == 0.5:
            up += bool(oh * 2 > h or ow * 2 > w)
            down += bool((h % 2 and oh * 2 < h) or (w % 2 and ow * 2 < w))
            capped += float(ts) / min(h, w) != 0.5
    assert up >= 6 and down >= 3 and capped >= 4, (up, down, capped)
    shapes = {(h, w) for h, w, _, _ in rec.PREP_CASES}
    assert {(1, 1), (1, 37), (41, 1)} <= shapes
    assert max(B.blob_geometry((h, w), ts, ms)[0] for h, w, ts, ms in rec.PREP_CASES) == 50.0
    assert any(0.5 < B.blob_geometry((h, w), ts, ms)[0] < 1 for h, w, ts, ms in rec.PREP_CASES)
    fx = [f for _, _, f in rec.FX_CASES]
    assert any(h % 2 and w % 2 for h, w, f in rec.FX_CASES if f == 0.5)
    near = [f for f in fx if f != 0.5 and abs(f - 0.5) < 8 * np.finfo(np.float64).eps]
    assert len(near) >= 8 and all(abs(1.0 / f - 2.0) >= np.finfo(np.float64).eps for f in near)
    assert sum(rec.cv_round(h * f) == h and rec.cv_round(w * f) == w and f != 1 for h, w, f in rec.FX_CASES) >= 3
    for (h, w, ts, ms) in rec.FULL_CASES:
        s, oh, ow, _, _ = B.blob_geometry((h, w), ts, ms)
        assert s == 0.5 and ((h % 2 and oh * 2 > h) or (w % 2 and ow * 2 > w))


def test_mask_cases_reach_their_edges(G):
    """Every box family is present for both mask sizes, and each does what it is named for under the oracle: zero-size boxes, an
    expanded origin in (-1, 0) (truncation is not floor) and at or below -1, expanded size S/2 x S/2 (OpenCV's area-fast kernel)
    with the whole SIMD tail pasted, S/2 on one axis only, exactly S x S, boxes 10-50x the mask size; and regions whose runs cross
    column boundaries, end at the last image column and set pixel (0, 0)."""
    for M in rec.MASK_SIZES:
        S = M + 2
        mine = [s for s in SETS if s.M == M]
        assert {f for s in mine for f in s.families} == set(rec.FAMILIES), M
        seen = set()
        for s in mine:
            b = s.boxes.astype(np.float64)
            e = rec.expand(M, s.boxes)
            ef = ref.expand_boxes(s.boxes, (M + 2.0) / M)
            w, h = e[:, 2] - e[:, 0] + 1, e[:, 3] - e[:, 1] + 1
            x0, x1 = np.maximum(e[:, 0], 0), np.minimum(e[:, 2] + 1, s.W)
            pasted = _unbits(G, s)
            for d, fam in enumerate(s.families):
                if fam == "point":
                    assert b[d, 0] == b[d, 2] and b[d, 1] == b[d, 3]
                    seen.add("point")
                elif fam == "trunc" and -1 < ef[d, 0] < 0:
                    assert e[d, 0] == 0
                    seen.add("trunc")
                elif fam == "neg" and e[d, 0] <= -1:
                    seen.add("neg")
                elif fam == "area2":
                    assert w[d] * 2 == S and h[d] * 2 == S, (s.tag, d)
                    if x1[d] - x0[d] == w[d]:
                        seen.add("area2_tail")
                elif fam in ("half_x", "half_y"):
                    assert (w[d] * 2 == S) != (h[d] * 2 == S), (s.tag, d)
                    seen.add(fam)
                elif fam == "exact":
                    assert w[d] == S and h[d] == S
                    seen.add("exact")
                elif fam == "big":
                    r = max(b[d, 2] - b[d, 0], b[d, 3] - b[d, 1]) / M
                    assert 10 <= r <= 50, (s.tag, d, r)
                    seen.add("big")
            for d in range(s.D):
                m = pasted[d]
                if s.H > 1 and s.W > 1 and np.any(m[-1, :-1] & m[0, 1:]):
                    seen.add("cross_column")
                if m[:, -1].any():
                    seen.add("last_column")
                if m[0, 0]:
                    seen.add("origin")
        assert seen >= {"point", "trunc", "neg", "area2_tail", "half_x", "half_y", "exact", "big", "cross_column", "last_column",
                        "origin"}, (M, seen)
    kinds = {k for s in SETS for k in s.kinds}
    assert kinds == set(rec.KINDS)


@pytest.mark.skipif(not rs.available(), reason="the reference tree is not available")
@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_against_live_reference(seed):
    """Fresh seeded inputs of every case through the reference's own blob.py and segm_results (real cv2, IPP off) and the oracle,
    compared bit for bit by the fixture's generator in a subprocess (the reference's modules must not shadow the package's here)."""
    pytest.importorskip("cv2")
    import subprocess
    import sys
    gen = os.path.join(os.path.dirname(__file__), "golden", "make_resize_edges_golden.py")
    r = subprocess.run([sys.executable, gen, "--check-seed", str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "the oracle reproduces the reference" in r.stdout


def test_fx_form_against_cv2():
    """oracle.resize_linear_f32_scale == cv2.resize(x, None, None, fx, fx, INTER_LINEAR) bit for bit (IPP off) on odd and even
    sizes at fx = 0.5 (area-fast, partial cells on odd sides), a few ulp either side of it, and scales around it."""
    cv2 = pytest.importorskip("cv2")
    ipp = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        rng = np.random.RandomState(5)
        e = np.finfo(np.float64).eps
        scales = [0.5, 0.5 + e / 2, 0.5 - e / 4, 0.5 + 2 * e, 0.5 - e, 0.49, 0.51, 0.5 + 1e-7, 0.25, 1.0 / 3]
        sizes = [(h, w) for h in (1, 2, 3, 4, 5, 7, 8, 11) for w in (1, 2, 3, 5, 6, 9, 13)] + [(23, 16), (37, 54), (101, 63), (2, 199)]
        n = 0
        for fx in scales:
            for (h, w) in sizes:
                if rec.cv_round(h * fx) < 1 or rec.cv_round(w * fx) < 1:
                    continue
                x = rec.fx_input(rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
                want = cv2.resize(x, None, None, fx=fx, fy=fx, interpolation=cv2.INTER_LINEAR)
                assert np.array_equal(ref.resize_linear_f32_scale(x, fx), want), (h, w, fx)
                n += 1
        assert n > 300
    finally:
        cv2.ipp.setUseIPP(ipp)

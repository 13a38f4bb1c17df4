"""Generates tests/golden/resize_edges_golden.npz by RUNNING THE REFERENCE's own lib/utils/blob.py (prep_im_for_blob +
im_list_to_blob) and lib/utils/result_utils.py segm_results, imported unmodified through oracle/reference_shim.py, with the real cv2
of this container (OpenCV 4.13, IPP off = OpenCV's own resize kernels) on the edge cases of tests/resize_edge_cases.py.  The fx cases
call cv2.resize(fx=fy=fx) directly on the mean-subtracted image, as prep_im_for_blob does.  The inputs are not stored (they are
seeded in resize_edge_cases.py); a digest of each mask set is.  The oracle must reproduce every reference result bit for bit.
With --check-seed N the same comparisons run on fresh inputs of seed N and nothing is written (tests/test_resize_edges_host.py runs
that in a subprocess: importing the reference's modules would shadow the package's lib/ overlay in the test process).

    python tests/golden/make_resize_edges_golden.py [--check-seed N]
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import reference_shim as rs  # noqa: E402
from oracle import ref as oref  # noqa: E402
import resize_edge_cases as rec  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main(seed=0):
    rs.install()
    import utils.blob as rb
    import utils.result_utils as ru
    cv2.ipp.setUseIPP(False)
    G = {"prep_cases": np.asarray(rec.PREP_CASES, np.int32), "fx_cases": np.asarray(rec.FX_CASES, np.float64)}
    for i, (h, w, ts, ms) in enumerate(rec.PREP_CASES):
        im = rec.prep_image(i, h, w, seed)
        blob, scale = rec.reference_prep(rb, im, ts, ms)
        mine, mscales = oref.prep_im_for_blob(im, target_sizes=[ts], max_size=ms)
        assert mscales[0] == scale and np.array_equal(oref.im_list_to_blob(mine), blob), (h, w, ts, ms)
        G["prep%d_blob" % i], G["prep%d_scale" % i] = blob, np.float64(scale)
        print("prep", (h, w, ts, ms), "->", blob.shape[2:], "scale", scale)
    for i, (h, w, fx) in enumerate(rec.FX_CASES):
        x = rec.fx_input(rec.prep_image(100 + i, h, w, seed))
        out = cv2.resize(x, None, None, fx=fx, fy=fx, interpolation=cv2.INTER_LINEAR)
        assert out.shape == (rec.cv_round(h * fx), rec.cv_round(w * fx), 3)
        assert np.array_equal(oref.resize_linear_f32_scale(x, fx), out), (h, w, fx)
        G["fx%d_out" % i] = np.ascontiguousarray(out)
        print("fx", (h, w, repr(fx)), "->", out.shape[:2])
    sets = rec.mask_sets(seed)
    G["mask_tags"] = np.array([s.tag for s in sets])
    for s in sets:
        pasted, strings = rec.reference_segm(ru, s)
        mp, ms_ = rec.oracle_segm(s)
        assert np.array_equal(mp, pasted) and ms_ == strings, s.tag
        enc = [x.encode() for x in strings]
        G[s.tag + "_digest"] = s.digest()
        G[s.tag + "_bits"] = np.packbits(pasted.reshape(s.D, -1), axis=1)
        G[s.tag + "_rle"] = np.frombuffer(b"".join(enc), np.uint8)
        G[s.tag + "_rle_off"] = np.concatenate([[0], np.cumsum([len(x) for x in enc])]).astype(np.int64)
        print(s.tag, "dets", s.D, "pixels set", int(pasted.sum()), "longest string", max(len(x) for x in enc))
    if seed:
        print("seed", seed, ": the oracle reproduces the reference")
        return
    path = os.path.join(OUT, "resize_edges_golden.npz")
    np.savez_compressed(path, **G)
    print("resize_edges_golden.npz", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main(int(sys.argv[sys.argv.index("--check-seed") + 1]) if "--check-seed" in sys.argv else 0)

"""The reference's own proposal-recall code with its compiled bbox_overlaps: oracle/build_cython_bbox.sh builds
lib/utils_cython/cython_bbox.pyx into oracle/_ref/, and load() imports the reference's utils.json_dataset_evaluator and
data.json_dataset from oracle/_ref/reflib.zip with that module in place of the stub reference_shim.install_compat registers.
The reference's pycocotools (oracle/cocoapi.py) is loaded first when it is built, so JsonDataset reads real annotation files."""
import glob
import importlib
import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")
_mods = None


def _so():
    hits = sorted(glob.glob(os.path.join(REF_DIR, "cython_bbox*.so")))
    return hits[0] if hits else None


def available():
    return _so() is not None and os.path.exists(os.path.join(REF_DIR, "reflib.zip"))


def build():
    import subprocess
    subprocess.check_call(["bash", os.path.join(_HERE, "build_cython_bbox.sh")], stdout=subprocess.DEVNULL)


def load():
    """-> (json_dataset_evaluator, json_dataset) modules of the reference; ImportError when the oracle is not built."""
    global _mods
    if _mods is not None:
        return _mods
    if not available():
        raise ImportError("reference cython_bbox / reflib.zip not built under %s (oracle/build_cython_bbox.sh, oracle/build_ref.sh)" % REF_DIR)
    from oracle import cocoapi, reference_shim
    if cocoapi.available():
        cocoapi.load()
    reference_shim.install_compat(stub_plotting=True)
    spec = importlib.util.spec_from_file_location("utils_cython.cython_bbox", _so())
    bb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bb)
    sys.modules["utils_cython.cython_bbox"] = bb
    zp = os.path.join(REF_DIR, "reflib.zip")
    if zp not in sys.path:
        sys.path.insert(0, zp)
    boxes = importlib.import_module("utils.boxes")
    boxes.bbox_overlaps = bb.bbox_overlaps          # boxes.py binds it at import time; an earlier import saw the stub
    jde = importlib.import_module("utils.json_dataset_evaluator")
    jd = importlib.import_module("data.json_dataset")
    _mods = (jde, jd)
    return _mods

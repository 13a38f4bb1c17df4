#!/usr/bin/env bash
# Builds the reference's lib/utils_cython/cython_bbox.pyx (bbox_overlaps) from where it lies under $REF (read-only) into
# oracle/_ref/ (git-ignored), the way build_ref.sh builds cython_nms: the source is copied to a temp dir and compiled there with
# Cython.  It needs no numpy-2 patch.  With it, the reference's own evaluate_box_proposals runs from oracle/_ref/reflib.zip with the
# real bbox_overlaps (oracle/cython_bbox.py).
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
SRC=$REF/lib/utils_cython/cython_bbox.pyx
if [ ! -f "$SRC" ]; then echo "build_cython_bbox: $SRC not present - using prebuilt $OUT"; exit 0; fi
if ! python -c "import Cython" 2>/dev/null; then echo "build_cython_bbox: Cython not importable - cython_bbox oracle not built"; exit 0; fi
mkdir -p "$OUT"
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
cp "$SRC" "$TMP/cython_bbox.pyx"
cat > "$TMP/setup.py" <<'PY'
from setuptools import setup, Extension
from Cython.Build import cythonize
import numpy as np
setup(ext_modules=cythonize([Extension("cython_bbox", ["cython_bbox.pyx"], include_dirs=[np.get_include()],
      extra_compile_args=["-O2", "-Wno-cpp"])], language_level=2, quiet=True))
PY
(cd "$TMP" && python setup.py -q build_ext --inplace >/dev/null 2>&1 && cp cython_bbox*.so "$OUT/")
ls "$OUT"/cython_bbox*.so

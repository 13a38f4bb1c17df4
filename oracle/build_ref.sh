#!/usr/bin/env bash
# Builds the REFERENCE's own sources for the hot path, from where they lie under
# $REF (read-only), into oracle/_ref/ (git-ignored).
# No reference source is copied into the repo: the Cython NMS needs a 2-token numpy-2
# patch (np.int_t -> np.intp_t, np.int -> np.intp; SURVEY.md 8c), which is applied by
# sed into a temp dir at build time.
#   _ref/libroialign_ref.so       <- lib/cppcuda_cffi/src/cpp/roi_align_cpu_loop.cpp   (CPU loop)
#   _ref/libroialign_ref_cuda.so  <- lib/cppcuda_cffi/src/cuda/roi_align_forward_cuda_kernel.cu
#                                     (the reference CUDA kernel, compiled unmodified for sm_90a:
#                                      the kernel to beat)
#   _ref/cython_nms*.so           <- lib/utils_cython/cython_nms.pyx (patched as above)
#   _ref/libroialign_bwd_ref.so   <- lib/cppcuda/roi_align_backward_cpu.cpp: the file is ATen-0.4 flavoured and does not compile against
#                                     torch 2.x, but its templates bilinear_interpolate_gradient / add / roi_align_backward_loop
#                                     (from the first "template" line to the "} // ROIAlignBackward" line) are plain C++: exactly those lines
#                                     are cut out by sed into a temp file and instantiated for float behind an extern "C" entry point
#   _ref/reflib.zip               <- the reference's pure-Python host modules (lib/utils, lib/data, lib/model), zipped unmodified:
#                                     importable through zipimport, so that tests/test_gpu_notebooks.py can run the reference's OWN
#                                     notebook cells (its collate_custom, to_cuda_variable, add_multilevel_rois_for_test ...) on the GPU
#                                     box, where /root/reference does not exist
#   _ref/notebook_cells.json      <- the code cells of the reference's eval_*.ipynb notebooks ({notebook: {cell index: source}})
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
if [ ! -d "$REF/lib" ]; then echo "build_ref: $REF not present (GPU box) - using prebuilt $OUT"; exit 0; fi
mkdir -p "$OUT"
g++ -O2 -fPIC -shared -o "$OUT/libroialign_ref.so" "$REF/lib/cppcuda_cffi/src/cpp/roi_align_cpu_loop.cpp"
if command -v nvcc >/dev/null; then
  nvcc -O3 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -shared \
       -o "$OUT/libroialign_ref_cuda.so" "$REF/lib/cppcuda_cffi/src/cuda/roi_align_forward_cuda_kernel.cu"
fi
TMPB=$(mktemp -d)
{ echo '#include <algorithm>'; echo '#include <cmath>'; echo 'namespace refbwd {';
  sed -n '/^template <typename T>/,/^} \/\/ ROIAlignBackward/p' "$REF/lib/cppcuda/roi_align_backward_cpu.cpp";
  echo '}';
  echo 'extern "C" void roi_align_backward_loop_f32(int nthreads, const float* top_diff, int num_rois, float spatial_scale, int channels, int height,';
  echo '    int width, int pooled_height, int pooled_width, int sampling_ratio, float* bottom_diff, const float* bottom_rois, int rois_cols) {';
  echo '  refbwd::roi_align_backward_loop<float>(nthreads, top_diff, num_rois, spatial_scale, channels, height, width, pooled_height, pooled_width,';
  echo '                                         sampling_ratio, bottom_diff, bottom_rois, rois_cols); }'; } > "$TMPB/bwd.cpp"
g++ -O2 -fPIC -shared -o "$OUT/libroialign_bwd_ref.so" "$TMPB/bwd.cpp"
rm -rf "$TMPB"
TMP=$(mktemp -d)
sed -e 's/np\.int_t/np.intp_t/g' -e 's/dtype=np\.int)/dtype=np.intp)/g' \
    "$REF/lib/utils_cython/cython_nms.pyx" > "$TMP/cython_nms.pyx"
cat > "$TMP/setup.py" <<'PY'
from setuptools import setup, Extension
from Cython.Build import cythonize
import numpy as np
setup(ext_modules=cythonize([Extension("cython_nms", ["cython_nms.pyx"], include_dirs=[np.get_include()],
      extra_compile_args=["-O2", "-Wno-cpp"])], language_level=2, quiet=True))
PY
(cd "$TMP" && python setup.py -q build_ext --inplace >/dev/null 2>&1 && cp cython_nms*.so "$OUT/")
rm -rf "$TMP"
python - "$REF" "$OUT" <<'PY'
import json, os, sys, zipfile
ref, out = sys.argv[1], sys.argv[2]
with zipfile.ZipFile(os.path.join(out, "reflib.zip"), "w", zipfile.ZIP_DEFLATED) as z:
    for pkg in ("utils", "data", "model"):
        d = os.path.join(ref, "lib", pkg)
        z.writestr(pkg + "/", "")          # explicit directory entry: zipimport then offers it as a namespace-package portion
        for f in sorted(os.listdir(d)):
            if f.endswith(".py"):
                z.write(os.path.join(d, f), pkg + "/" + f)
cells = {}
for nb in sorted(f for f in os.listdir(ref) if f.startswith("eval_") and f.endswith(".ipynb")):
    doc = json.load(open(os.path.join(ref, nb)))
    cells[nb] = {str(i): "".join(c["source"]) for i, c in enumerate(doc["cells"]) if c["cell_type"] == "code"}
json.dump(cells, open(os.path.join(out, "notebook_cells.json"), "w"))
PY
ls -la "$OUT"

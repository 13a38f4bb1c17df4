"""RoIAlign + NMS microbench (BASELINE.json configs[4]): 100k boxes x 256-ch 50x68 feature map on 1 H100,
achieved HBM GB/s vs the measured roofline, next to the reference's own CUDA kernel (compiled unmodified for
sm_90a into oracle/_ref/libroialign_ref_cuda.so) and the reference's CPU loop / Cython NMS on a bounded sample.

  python tests/bench_micro.py            -> one JSON line per measurement
"""
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from detectorch_b200 import ops  # noqa: E402
from oracle import ref  # noqa: E402

dev = torch.device("cuda:0")


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p)).get("hbm_gbs", 6650.0), "measured"
    return 6650.0, "fallback"


def synth_rois(n, seed=0, W=1088, H=800):
    """SURVEY.md 8d: centres U(0,W)xU(0,H), width log-U(16,600) px, aspect log-U(e^-0.7, e^0.7), clipped to the image."""
    rng = np.random.RandomState(seed)
    cx, cy = rng.uniform(0, W, n), rng.uniform(0, H, n)
    w = np.exp(rng.uniform(np.log(16), np.log(600), n))
    a = np.exp(rng.uniform(-0.7, 0.7, n))
    bw, bh = w * np.sqrt(a), w / np.sqrt(a)
    b = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, W - 1)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, H - 1)
    return b.astype(np.float32)


def time_cuda(fn, warm=3, reps=10, flush=None):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        if flush is not None:
            flush.zero_()               # > L2-sized write between timed iterations
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def roialign():
    hbm, which = peaks()
    R, C, H, W = 100000, 256, 50, 68
    g = torch.Generator().manual_seed(0)
    feat = torch.randn((1, C, H, W), generator=g).to(dev)
    rois = torch.from_numpy(np.hstack([np.zeros((R, 1), np.float32), synth_rois(R)])).to(dev)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    refso = os.path.join(ROOT, "oracle", "_ref", "libroialign_ref_cuda.so")
    for (p, sr) in ((7, 2), (14, 2)):
        out_bytes = R * C * p * p * 4
        alg_bytes = out_bytes + feat.numel() * 4 + rois.numel() * 4
        out = torch.empty((R, C, p, p), device=dev)
        res = {}
        res["exact"] = time_cuda(lambda: ops.roi_align_forward_nchw(feat, rois, p, p, 1 / 16., sr, out=out), flush=flush)
        exact_out = out[:2000].clone()
        res["fast"] = time_cuda(lambda: ops.roi_align_forward_nchw_fast(feat, rois, p, p, 1 / 16., sr, out=out), flush=flush)
        diff_fast = float((out[:2000] - exact_out).abs().max())
        diff_ref = None
        if os.path.exists(refso) and out.numel() < 2 ** 31:
            L = ctypes.CDLL(refso)
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

            def run_ref():
                L.launch_roi_align_forward_cuda(ctypes.c_int(out.numel()), ctypes.c_void_p(feat.data_ptr()), ctypes.c_void_p(rois.data_ptr()),
                                                ctypes.c_float(1 / 16.), C, H, W, p, p, sr, ctypes.c_void_p(out.data_ptr()), st)
            res["reference_cuda_kernel"] = time_cuda(run_ref, flush=flush)
            diff_ref = float((out[:2000] - exact_out).abs().max())
        # bounded CPU sample of the reference loop (single-threaded by construction)
        ncpu = 300
        t0 = time.perf_counter()
        ref.roi_align_forward(feat.cpu().numpy(), rois[:ncpu].cpu().numpy(), p, p, 1 / 16., sr)
        cpu_ms_per_roi = (time.perf_counter() - t0) * 1e3 / ncpu
        for k, ms in res.items():
            gbs = alg_bytes / (ms * 1e-3) / 1e9
            print(json.dumps({"bench": "roialign", "impl": k, "rois": R, "channels": C, "map": [H, W], "pooled": p, "sampling_ratio": sr, "ms": ms,
                              "rois_per_s": R / (ms * 1e-3), "algorithmic_bytes": alg_bytes, "achieved_gbs": gbs, "hbm_peak_gbs": hbm,
                              "peak_source": which, "frac": gbs / hbm, "max_abs_diff_fast_vs_exact": diff_fast, "max_abs_diff_ref_vs_exact": diff_ref,
                              "cpu_reference_loop_ms_per_roi": cpu_ms_per_roi}), flush=True)
        del out


def nms():
    for n in (1000, 6000, 20000, 100000):
        rng = np.random.RandomState(n)
        d = np.hstack([synth_rois(n, seed=n, W=1216), rng.permutation(n).astype(np.float32)[:, None] / n]).astype(np.float32)
        dd = torch.from_numpy(d).to(dev)
        ms = time_cuda(lambda: ops.nms(dd, 0.5), warm=1, reps=3)
        kept = int(ops.nms(dd, 0.5).numel())
        cpu_ms = None
        equal = None
        if n <= 20000:
            t0 = time.perf_counter()
            want = ref.nms(d, 0.5)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            equal = bool(np.array_equal(want, ops.nms(dd, 0.5).cpu().numpy()))
        print(json.dumps({"bench": "nms", "boxes": n, "thresh": 0.5, "ms": ms, "kept": kept, "pair_tests": n * (n - 1) // 2,
                          "cpu_reference_ms": cpu_ms, "kept_ids_equal_cpu": equal}), flush=True)


def segm():
    """SURVEY 8f rank 1: 100 detections of one 800x1216 image, 28x28 masks -> COCO RLE strings.  GPU: dt_segm_rle (device masks
    in, strings out, D2H of the strings included); CPU: the reference algorithm (cv2.resize when importable, else the numpy
    restatement) + the restated maskApi RLE, single thread as the reference runs it."""
    rng = np.random.RandomState(7)
    im_h, im_w, D, M = 800, 1216, 100, 28
    b = synth_rois(D, seed=3, W=im_w, H=im_h)
    yy, xx = np.mgrid[0:M, 0:M].astype(np.float32) / M
    masks = np.stack([np.clip(1 / (1 + np.exp(((xx - rng.uniform(.3, .7)) ** 2 + (yy - rng.uniform(.3, .7)) ** 2 - rng.uniform(.05, .2)) * 40))
                              + 0.1 * rng.randn(M, M), 0, 1) for _ in range(D)]).astype(np.float32)
    tm, tb = torch.from_numpy(masks).to(dev), torch.from_numpy(b).to(dev)
    ms = time_cuda(lambda: ops.segm_rle(tm, None, tb, im_h, im_w), warm=2, reps=5)
    ms_paste = time_cuda(lambda: ops.segm_paste(tm, None, tb, im_h, im_w), warm=2, reps=5)
    counts, strings = ops.segm_rle(tm, None, tb, im_h, im_w)
    exp = ref.expand_boxes(b, (M + 2.0) / M).astype(np.int32)
    try:
        import cv2
        cv2.ipp.setUseIPP(False)
        cv2.setNumThreads(1)
        resize, kind = (lambda m, w, h: cv2.resize(m, (w, h))), "cv2.resize (IPP off) + restated maskApi RLE"
    except Exception:
        resize, kind = ref.resize_linear_f32, "numpy restatement"
    t0 = time.perf_counter()
    same = True
    for d in range(D):
        padded = np.zeros((M + 2, M + 2), np.float32)
        padded[1:-1, 1:-1] = masks[d]
        w, h = max(exp[d, 2] - exp[d, 0] + 1, 1), max(exp[d, 3] - exp[d, 1] + 1, 1)
        m = (resize(padded, int(w), int(h)) > 0.5).astype(np.uint8)
        im = np.zeros((im_h, im_w), np.uint8)
        x0, x1, y0, y1 = max(exp[d, 0], 0), min(exp[d, 2] + 1, im_w), max(exp[d, 1], 0), min(exp[d, 3] + 1, im_h)
        im[y0:y1, x0:x1] = m[y0 - exp[d, 1]:y1 - exp[d, 1], x0 - exp[d, 0]:x1 - exp[d, 0]]
        s = ref.rle_to_string(ref.rle_encode(im))
        same = same and (s == strings[d])
    cpu_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"bench": "segm_rle", "dets": D, "image": [im_h, im_w], "mask": M, "gpu_ms_rle_incl_d2h": ms, "gpu_ms_paste_uint8": ms_paste,
                      "cpu_ms": cpu_ms, "cpu_kind": kind, "strings_equal_cpu": bool(same),
                      "string_bytes": int(sum(len(s) for s in strings)), "avoided_d2h_bytes": D * 81 * M * M * 4}), flush=True)


if __name__ == "__main__":
    print(json.dumps({"device": torch.cuda.get_device_name(0)}), flush=True)
    which = sys.argv[1:] or ["roialign", "nms", "segm"]
    if "roialign" in which:
        roialign()
    if "nms" in which:
        nms()
    if "segm" in which:
        segm()

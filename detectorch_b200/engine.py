"""Python handle on the fused C++/CUDA engine (include/detectorch_b200.h, dt_engine_*).
Torch only provides the two flat device buffers, the stream and zero-copy views of the named
engine tensors; every kernel is launched by the C++ side."""
import ctypes
import os
import weakref

import torch

from . import _lib

ARCH_BLOCKS = {"resnet50": (3, 4, 6, 3), "resnet101": (3, 4, 23, 3)}


def param_table(arch="resnet50", use_mask=True, num_classes=81, model="fpn", use_rpn=True):
    """{reference state_dict name: numel} the engine expects (no GPU needed)."""
    L = _lib.lib()
    _bind_engine_api(L)
    cfg = EngineConfig()
    cfg.arch_blocks = (ctypes.c_int * 4)(*ARCH_BLOCKS[arch])
    cfg.batch, cfg.height, cfg.width = 1, 64, 64
    cfg.pre_nms_top_n = cfg.post_nms_top_n = 1000
    cfg.num_classes, cfg.max_dets, cfg.det_cap, cfg.use_mask = num_classes, 100, 100, int(use_mask)
    cfg.model_type, cfg.use_rpn = (1 if model == "c4" else 0), int(use_rpn)
    h = L.dt_engine_create(ctypes.byref(cfg))
    out = {}
    buf = ctypes.create_string_buffer(256)
    n = ctypes.c_int64()
    for i in range(L.dt_engine_param_count(h)):
        L.dt_engine_param_info(h, i, buf, 256, ctypes.byref(n))
        out[buf.value.decode()] = n.value
    L.dt_engine_destroy(h)
    return out

# stage ids (dt_engine_run)
ST_TRUNK, ST_FPN, ST_RPN, ST_PROPOSALS, ST_COLLECT, ST_ROI_BOX, ST_BOX_HEAD, ST_DETECT, ST_MASK_ROIS, ST_MASK_ROI_FEAT, \
    ST_MASK_HEAD, ST_MASK_OUT = range(12)


class EngineConfig(ctypes.Structure):
    _fields_ = [("arch_blocks", ctypes.c_int * 4), ("batch", ctypes.c_int), ("height", ctypes.c_int), ("width", ctypes.c_int),
                ("pre_nms_top_n", ctypes.c_int), ("post_nms_top_n", ctypes.c_int), ("rpn_nms_thresh", ctypes.c_float),
                ("rpn_min_size", ctypes.c_float), ("num_classes", ctypes.c_int), ("score_thresh", ctypes.c_float),
                ("det_nms_thresh", ctypes.c_float), ("max_dets", ctypes.c_int), ("det_cap", ctypes.c_int),
                ("use_mask", ctypes.c_int), ("output_prob", ctypes.c_int), ("emit_full_masks", ctypes.c_int),
                ("passes", ctypes.c_int), ("precise_mask", ctypes.c_int), ("stem_im2col", ctypes.c_int), ("exact_roialign", ctypes.c_int), ("model_type", ctypes.c_int), ("use_rpn", ctypes.c_int),
                ("conv_kind", ctypes.c_int), ("plane_handover", ctypes.c_int)]


_DTYPES = {0: torch.float32, 1: torch.int32, 2: torch.uint8}


def _bind_engine_api(L):
    if getattr(L, "_engine_bound", False):
        return
    vp, ci, c64, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
    L.dt_engine_create.restype, L.dt_engine_create.argtypes = vp, [ctypes.POINTER(EngineConfig)]
    L.dt_engine_destroy.restype, L.dt_engine_destroy.argtypes = None, [vp]
    L.dt_engine_weight_bytes.restype, L.dt_engine_weight_bytes.argtypes = c64, [vp]
    L.dt_engine_workspace_bytes.restype, L.dt_engine_workspace_bytes.argtypes = c64, [vp]
    L.dt_engine_bind.restype, L.dt_engine_bind.argtypes = ci, [vp, vp, vp, vp]
    L.dt_engine_attach.restype, L.dt_engine_attach.argtypes = ci, [vp, vp, vp, vp]
    L.dt_engine_load_param.restype, L.dt_engine_load_param.argtypes = ci, [vp, ctypes.c_char_p, vp, c64, vp]
    L.dt_engine_finalize_weights.restype, L.dt_engine_finalize_weights.argtypes = ci, [vp, vp]
    L.dt_engine_buffer.restype = ci
    L.dt_engine_buffer.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(c64), ctypes.POINTER(ci), ctypes.POINTER(ci * 5), ctypes.POINTER(ci)]
    L.dt_engine_num_stages.restype, L.dt_engine_num_stages.argtypes = ci, []
    L.dt_engine_param_count.restype, L.dt_engine_param_count.argtypes = ci, [vp]
    L.dt_engine_param_info.restype, L.dt_engine_param_info.argtypes = ci, [vp, ci, ctypes.c_char_p, ci, ctypes.POINTER(c64)]
    L.dt_engine_set_original_size.restype, L.dt_engine_set_original_size.argtypes = ci, [vp, cf, cf]
    L.dt_engine_run.restype, L.dt_engine_run.argtypes = ci, [vp, vp, cf, ci, ci, vp]
    L.dt_engine_count_launches.restype, L.dt_engine_count_launches.argtypes = ci, [vp, ci, ci]
    L.dt_engine_profile.restype, L.dt_engine_profile.argtypes = ci, [vp, vp, cf, ci, ci, vp, vp, vp, vp, vp, ci]
    L._engine_bound = True


_live_engines = weakref.WeakSet()


def engine_owning(*tensors):
    """The live Engine whose workspace contains one of the given CUDA tensors (views of engine buffers returned by the mirror API), else None.
    This is how postprocess_output / mask_head find the engine that produced their inputs without any global "active engine" state."""
    for t in tensors:
        if isinstance(t, (list, tuple)):
            e = engine_owning(*t)
            if e is not None:
                return e
            continue
        if not torch.is_tensor(t) or not t.is_cuda or t.numel() == 0:
            continue
        p = t.data_ptr()
        for e in list(_live_engines):
            if e.device == t.device and e.owns(p):
                return e
    return None


def fold_bn_running_stats(sd, eps=1e-5):
    """The engine folds eval-mode BatchNorm as gamma / sqrt(1 + eps), beta -- the reference's situation (detector.py:231,301: the Detectron
    import never touches the running stats, so they stay at (0, 1)).  A state_dict with NON-trivial running_mean / running_var (a
    torchvision-pretrained trunk, a checkpoint trained with live BN) is re-expressed in that form here, so that the result equals what
    torch's eval BatchNorm computes: gamma' = gamma * sqrt(1 + eps) / sqrt(var + eps), beta' = beta - mean * gamma / sqrt(var + eps)."""
    out = dict(sd)
    for k, mean in sd.items():
        if not k.endswith(".running_mean"):
            continue
        pre = k[:-len(".running_mean")]
        var = sd.get(pre + ".running_var")
        if var is None or (pre + ".weight") not in sd or (pre + ".bias") not in sd:
            continue
        mean, var = mean.detach().double(), var.detach().double()
        if bool((mean == 0).all()) and bool((var == 1).all()):
            continue
        g, b = sd[pre + ".weight"].detach().double().to(mean.device), sd[pre + ".bias"].detach().double().to(mean.device)
        inv = 1.0 / torch.sqrt(var + eps)
        out[pre + ".weight"] = (g * inv * (1.0 + eps) ** 0.5).float()
        out[pre + ".bias"] = (b - mean * g * inv).float()
    return out


class Engine:
    def __init__(self, arch="resnet50", batch=1, height=800, width=1216, pre_nms_top_n=1000, post_nms_top_n=1000,
                 rpn_nms_thresh=0.7, rpn_min_size=0.0, num_classes=81, score_thresh=0.05, det_nms_thresh=0.5, max_dets=100,
                 det_cap=100, use_mask=True, output_prob=True, emit_full_masks=False, passes=3, precise_mask=True, stem_im2col=False, exact_roialign=False, model="fpn", use_rpn=True, conv_kind=None, device="cuda:0",
                 share_weights_with=None):
        if not torch.cuda.is_available():
            raise RuntimeError("detectorch_b200.Engine needs a CUDA device (no CPU fallback)")
        self.L = _lib.lib()
        _bind_engine_api(self.L)
        self.device = torch.device(device)
        cfg = EngineConfig()
        cfg.arch_blocks = (ctypes.c_int * 4)(*ARCH_BLOCKS[arch])
        cfg.batch, cfg.height, cfg.width = batch, height, width
        cfg.pre_nms_top_n, cfg.post_nms_top_n = pre_nms_top_n, post_nms_top_n
        cfg.rpn_nms_thresh, cfg.rpn_min_size = rpn_nms_thresh, rpn_min_size
        cfg.num_classes, cfg.score_thresh, cfg.det_nms_thresh = num_classes, score_thresh, det_nms_thresh
        cfg.max_dets, cfg.det_cap = max_dets, det_cap
        cfg.use_mask, cfg.output_prob, cfg.emit_full_masks, cfg.passes = int(use_mask), int(output_prob), int(emit_full_masks), passes
        cfg.precise_mask = int(precise_mask)          # 1/True = K-split mask convs, 2 = 64-wide tiles with 3 rotating accumulators, 0 = plain
        cfg.stem_im2col = int(stem_im2col)
        cfg.exact_roialign = int(exact_roialign)
        cfg.model_type = 1 if model == "c4" else 0
        cfg.use_rpn = int(use_rpn)
        if conv_kind is None:
            conv_kind = os.environ.get("DT_CONV_KIND", "f16")
        if conv_kind not in ("f16", "tf32"):
            raise ValueError("conv_kind must be 'f16' or 'tf32'")
        cfg.conv_kind = 0 if conv_kind == "f16" else 1
        cfg.plane_handover = int(os.environ.get("DT_PLANE_HANDOVER", "3"))     # 0 = fp32 hand-over, 1 = conv1 -> conv2 as fp16 planes, 2 = also conv2 -> conv3, 3 = also image -> stem; 4 = also pool -> first bottleneck (measured: no net gain, opt-in)
        self.cfg = cfg
        self.h = self.L.dt_engine_create(ctypes.byref(cfg))
        if not self.h:
            raise RuntimeError("dt_engine_create failed (see stderr)")
        self._views = {}
        self.weights_loaded = False
        with torch.cuda.device(self.device):
            self.workspace = torch.zeros((self.L.dt_engine_workspace_bytes(self.h),), dtype=torch.uint8, device=self.device)
            self._ws_lo = self.workspace.data_ptr()
            self._ws_hi = self._ws_lo + self.workspace.numel()
            if share_weights_with is not None:
                # packed weights do not depend on the input shape: engines of one model for different image sizes share one copy
                o = share_weights_with
                if self.model_key() != o.model_key() or not o.weights_loaded or o.device != self.device or \
                        self.L.dt_engine_weight_bytes(self.h) != o.weights.numel():
                    raise RuntimeError("share_weights_with: the other engine must hold loaded weights of the same model configuration on the same device")
                self.weights = o.weights
                _lib.check(self.L.dt_engine_attach(self.h, self.weights.data_ptr(), self.workspace.data_ptr(), self._stream()), "dt_engine_attach")
                self.weights_loaded = True
            else:
                self.weights = torch.empty((self.L.dt_engine_weight_bytes(self.h),), dtype=torch.uint8, device=self.device)
                _lib.check(self.L.dt_engine_bind(self.h, self.weights.data_ptr(), self.workspace.data_ptr(), self._stream()), "dt_engine_bind")
        _live_engines.add(self)

    def model_key(self):
        """What shapes the packed weight buffer (matrices, fp16 halves, and the per-conv-launch scale vectors, which are laid out in launch
        order): the model and the numerics mode -- not the image size, RoI / detection capacities or thresholds."""
        c = self.cfg
        return tuple(c.arch_blocks) + (c.num_classes, c.use_mask, c.model_type, c.use_rpn, c.conv_kind, c.precise_mask, c.passes, c.stem_im2col)

    def owns(self, ptr):
        return self._ws_lo <= ptr < self._ws_hi

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.L.dt_engine_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def load_state_dict(self, sd):
        """sd: {reference state_dict name: tensor}.  Names that are not hot-path parameters are ignored; BatchNorm running statistics other
        than (0, 1) are folded into the affine pair (fold_bn_running_stats)."""
        n = 0
        sd = fold_bn_running_stats({k: v for k, v in sd.items() if torch.is_tensor(v) and v.dtype.is_floating_point})
        staged = []                                                # keeps the device copies alive until the pack kernels ran
        with torch.cuda.device(self.device):
            for name, t in sd.items():
                if name.endswith((".running_mean", ".running_var")):
                    continue
                t = t.detach().to(self.device, torch.float32).contiguous()
                r = self.L.dt_engine_load_param(self.h, name.encode(), t.data_ptr(), t.numel(), self._stream())
                if r == 0:
                    raise RuntimeError("dt_engine_load_param(%s) failed" % name)
                n += (r == 1)
                staged.append(t)
            _lib.check(self.L.dt_engine_finalize_weights(self.h, self._stream()), "dt_engine_finalize_weights")
            torch.cuda.current_stream(self.device).synchronize()
        del staged
        self.weights_loaded = True
        return n

    def buffer(self, name):
        """Zero-copy torch view of a named engine tensor."""
        if name in self._views:
            return self._views[name]
        off, nd, dims, dt = ctypes.c_int64(), ctypes.c_int(), (ctypes.c_int * 5)(), ctypes.c_int()
        if self.L.dt_engine_buffer(self.h, name.encode(), ctypes.byref(off), ctypes.byref(nd), ctypes.byref(dims), ctypes.byref(dt)) != 1:
            raise KeyError(name)
        shape = [dims[i] for i in range(nd.value)]
        dtype = _DTYPES[dt.value]
        n = 1
        for s in shape:
            n *= s
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        v = self.workspace[off.value:off.value + nbytes].view(dtype).view(shape)
        self._views[name] = v
        return v

    def run(self, image=None, scaling_factor=1.0, first=0, last=None):
        if not self.weights_loaded:
            raise RuntimeError("Engine.run before load_state_dict")
        if last is None:
            last = ST_MASK_OUT if self.cfg.use_mask else ST_DETECT
        ptr = 0
        if image is not None:
            if not image.is_cuda or image.dtype != torch.float32 or not image.is_contiguous():
                raise RuntimeError("image must be a contiguous fp32 CUDA tensor [B,3,H,W]")
            if tuple(image.shape) != (self.cfg.batch, 3, self.cfg.height, self.cfg.width):
                raise RuntimeError("image shape %s does not match the engine (%d,3,%d,%d)" % (tuple(image.shape), self.cfg.batch, self.cfg.height, self.cfg.width))
            ptr = image.data_ptr()
        with torch.cuda.device(self.device):       # the C ABI launches on the current device: make it the engine's
            _lib.check(self.L.dt_engine_run(self.h, ptr, float(scaling_factor), int(first), int(last), self._stream()), "dt_engine_run")

    def check_range(self):
        """kind::f16 convs raise a device flag when an activation does not fit fp16 (|x| >= 65504).  Synchronises; raises if set."""
        f = self.buffer("range_flag")
        if int(f.item()) != 0:
            f.zero_()
            raise FloatingPointError("detectorch_b200: an activation exceeded the fp16 range of the kind::f16 convolution path; "
                                     "build the Engine with conv_kind='tf32' for this model / input")

    def set_original_size(self, h, w):
        self.L.dt_engine_set_original_size(self.h, float(h), float(w))

    def profile(self, image, scaling_factor=1.0, first=0, last=11):
        """One event-bracketed pass: list of (ms, algorithmic_flops, stage, block_n) per launch."""
        cap = 512
        ms = (ctypes.c_float * cap)(); fl = (ctypes.c_double * cap)(); st = (ctypes.c_int * cap)(); bn = (ctypes.c_int * cap)()
        with torch.cuda.device(self.device):
            n = self.L.dt_engine_profile(self.h, image.data_ptr(), float(scaling_factor), first, last, self._stream(), ms, fl, st, bn, cap)
        if n <= 0:
            raise RuntimeError("dt_engine_profile failed")
        return [(ms[i], fl[i], st[i], bn[i]) for i in range(n)]

    def count_launches(self, first=0, last=11):
        return self.L.dt_engine_count_launches(self.h, first, last)

"""Mirror of the image half of the reference lib/utils/blob.py (prep_im_for_blob :57-87, im_list_to_blob :27-55) on the device:
the uint8 image is uploaded once (a quarter of the fp32 bytes, and before the up-scaling), mean subtraction, OpenCV-exact
bilinear resize, zero padding to the FPN stride and the HWC->CHW transpose happen in one kernel (dt_prep_image)."""
import ctypes

import numpy as np
import torch

from .. import _lib

PIXEL_MEANS = [122.7717, 115.9465, 102.9801]


def im_scale_for(im_shape, target_size=800, max_size=1333):
    """The scale factor of prep_im_for_blob (blob.py:67-76) for one target size."""
    im_size_min, im_size_max = np.min(im_shape[0:2]), np.max(im_shape[0:2])
    im_scale = float(target_size) / float(im_size_min)
    if np.round(im_scale * im_size_max) > max_size:
        im_scale = float(max_size) / float(im_size_max)
    return im_scale


def blob_geometry(im_shape, target_size=800, max_size=1333, fpn_on=False, fpn_coarsest_stride=32):
    """-> (im_scale, resized height, resized width, blob height, blob width) of one image: the scale of prep_im_for_blob, the size
    cv2.resize(fx, fy) produces (cvRound), and with fpn_on the im_list_to_blob padding to a multiple of the coarsest FPN stride."""
    h, w = int(im_shape[0]), int(im_shape[1])
    s = im_scale_for((h, w), target_size, max_size)
    oh, ow = int(np.rint(h * s)), int(np.rint(w * s))
    bh, bw = oh, ow
    if fpn_on:
        stride = float(fpn_coarsest_stride)
        bh, bw = int(np.ceil(oh / stride) * stride), int(np.ceil(ow / stride) * stride)
    return s, oh, ow, bh, bw


def image_to_blob(im, pixel_means=PIXEL_MEANS, target_size=800, max_size=1333, fpn_on=False, fpn_coarsest_stride=32, device=None):
    """uint8 BGR image [H,W,3] (numpy or CUDA uint8 tensor) -> (blob CUDA fp32 [1,3,Hp,Wp], im_scale): exactly
    torch.FloatTensor(im_list_to_blob(prep_im_for_blob(im, ...)[0], fpn_on)) of the reference, without the host round trip."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    t = im if torch.is_tensor(im) else torch.from_numpy(np.ascontiguousarray(im))
    if t.dtype != torch.uint8 or t.dim() != 3 or t.size(2) != 3:
        raise TypeError("image_to_blob: expected a uint8 [H,W,3] image")
    t = t.to(dev).contiguous()
    h, w = int(t.size(0)), int(t.size(1))
    s, oh, ow, bh, bw = blob_geometry((h, w), target_size, max_size, fpn_on, fpn_coarsest_stride)
    blob = torch.empty((1, 3, bh, bw), dtype=torch.float32, device=dev)
    means = (ctypes.c_double * 3)(*[float(m) for m in pixel_means])
    ok = _lib.lib().dt_prep_image(ctypes.c_void_p(t.data_ptr()), h, w, ctypes.cast(means, ctypes.c_void_p), float(s), oh, ow,
                                  ctypes.c_void_p(blob.data_ptr()), bh, bw, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(ok, "dt_prep_image")
    return blob, s


def prep_im_for_blob(im, pixel_means=PIXEL_MEANS, target_sizes=[800], max_size=1333):
    """Same return structure as blob.py:57-87 (list of HWC float32 images, list of scales) but the images are CUDA tensors."""
    ims, scales = [], []
    for ts in target_sizes:
        blob, s = image_to_blob(im, pixel_means, ts, max_size, fpn_on=False)
        ims.append(blob[0].permute(1, 2, 0).contiguous())
        scales.append(s)
    return ims, scales


def im_list_to_blob(ims, fpn_on=False, fpn_coarsest_stride=32):
    """blob.py:27-55 for CUDA HWC tensors (as returned by prep_im_for_blob above): zero-pad to the common / stride-aligned shape,
    NHWC -> NCHW."""
    mh, mw = max(int(i.shape[0]) for i in ims), max(int(i.shape[1]) for i in ims)
    if fpn_on:
        stride = float(fpn_coarsest_stride)
        mh, mw = int(np.ceil(mh / stride) * stride), int(np.ceil(mw / stride) * stride)
    blob = torch.zeros((len(ims), mh, mw, 3), dtype=torch.float32, device=ims[0].device)
    for i, im in enumerate(ims):
        blob[i, :im.shape[0], :im.shape[1], :] = im
    return blob.permute(0, 3, 1, 2).contiguous()


def images_to_batch(ims, target_size=800, max_size=1333, canvas=None, pixel_means=PIXEL_MEANS, fpn_coarsest_stride=32, device=None):
    """Differently-sized uint8 BGR images [H,W,3] -> one padded batch for detector.detect(..., image_sizes, original_sizes):
    (blob CUDA fp32 [B,3,Hc,Wc], image_sizes int64 [B,2], scales float64 [B], original_sizes int64 [B,2]).
    Slot b holds image_to_blob(ims[b], fpn_on=True) in its top-left image_sizes[b] corner and zeros elsewhere.  canvas=None takes the
    largest per-image size of the batch; a fixed (Hc, Wc) (e.g. 800x1344 for landscape images, 1344x800 for portrait ones) lets one
    engine and one captured graph serve every batch."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    ts, geo = [], []
    for im in ims:
        t = im if torch.is_tensor(im) else torch.from_numpy(np.ascontiguousarray(im))
        if t.dtype != torch.uint8 or t.dim() != 3 or t.size(2) != 3:
            raise TypeError("images_to_batch: expected uint8 [H,W,3] images")
        t = t.to(dev).contiguous()
        h, w = int(t.size(0)), int(t.size(1))
        ts.append(t)
        geo.append((h, w) + blob_geometry((h, w), target_size, max_size, True, fpn_coarsest_stride))      # the blob image_to_blob(fpn_on=True) makes
    if not geo:
        raise ValueError("images_to_batch: no images")
    if canvas is None:
        hc, wc = max(g[5] for g in geo), max(g[6] for g in geo)
    else:
        hc, wc = int(canvas[0]), int(canvas[1])
        if hc % fpn_coarsest_stride or wc % fpn_coarsest_stride:
            raise ValueError("images_to_batch: the canvas must be a multiple of %d" % fpn_coarsest_stride)
        for g in geo:
            if g[5] > hc or g[6] > wc:
                raise ValueError("images_to_batch: a %dx%d image does not fit the %dx%d canvas" % (g[5], g[6], hc, wc))
    blob = torch.empty((len(ts), 3, hc, wc), dtype=torch.float32, device=dev)
    means = (ctypes.c_double * 3)(*[float(m) for m in pixel_means])
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for b, (t, (h, w, s, oh, ow, _, _)) in enumerate(zip(ts, geo)):
        # the kernel writes the whole [3, hc, wc] slot: the resized image, zeros around it
        ok = _lib.lib().dt_prep_image(ctypes.c_void_p(t.data_ptr()), h, w, ctypes.cast(means, ctypes.c_void_p), float(s), oh, ow,
                                      ctypes.c_void_p(blob[b].data_ptr()), hc, wc, stream)
        _lib.check(ok, "dt_prep_image")
    sizes = torch.tensor([[g[5], g[6]] for g in geo], dtype=torch.int64)
    scales = torch.tensor([g[2] for g in geo], dtype=torch.float64)
    orig = torch.tensor([[g[0], g[1]] for g in geo], dtype=torch.int64)
    return blob, sizes, scales, orig

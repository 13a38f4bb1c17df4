"""GPU tests of two-phase conv launches (RES_STAGED): phase 1's result stays in the staging area as phase 2's residual.  Each case
asserts that the one launch equals, bit for bit, the composition it replaces: phase 1 written to a buffer, then phase 2 with that
buffer as its residual.  Cases: the bottleneck downsample (stride 2, another Cin) and the mask-head K-split (the same input, filter taps
[0,5) then [5,9)), both kinds, 64- and 128-wide tiles, short and long K, several tiles per persistent CTA, boxes smaller than 128
pixels, per-image output masking and the fp16 range flag."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _phase(dev, g, x, cout, k, pad, stride, tap0=0, ntaps=0, w=None):
    cin = x.size(3)
    if w is None:
        w = (torch.randn((cout, k * k * cin), generator=g) * (1.0 / (k * k * cin) ** 0.5)).to(dev)
    scale = (1.0 + 0.25 * torch.randn(cout, generator=g)).to(dev)
    shift = (0.5 * torch.randn(cout, generator=g)).to(dev)
    return dict(x=x, w=w, scale=scale, shift=shift, k=k, pad=pad, stride=stride, tap0=tap0, ntaps=ntaps)


def _check(dev, phase1, phase2, kind, block_n, relu=True, im_info=None, im_stride=0):
    from detectorch_b200 import ops
    flag_sep = torch.zeros((1,), dtype=torch.int32, device=dev)
    flag_two = torch.zeros((1,), dtype=torch.int32, device=dev)
    kw = dict(kind=kind, force_block_n=block_n, im_info=im_info, im_stride=im_stride)
    res = ops.conv2d_nhwc_two_phase(phase1, relu=False, range_flag=flag_sep, kind=kind, force_block_n=block_n)
    want = ops.conv2d_nhwc_two_phase(phase2, residual=res, relu=relu, range_flag=flag_sep, **kw)
    got = ops.conv2d_nhwc_two_phase(phase2, phase1=phase1, relu=relu, range_flag=flag_two, **kw)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert int(flag_two.item()) == int(flag_sep.item())
    return got, int(flag_two.item())


def _downsample(dev, kind, block_n, N, H, W, cin1, cin2, cout, stride, seed=0, **kw):
    g = torch.Generator().manual_seed(seed)
    x1 = torch.randn((N, H, W, cin1), generator=g).to(dev)
    ho, wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    x2 = torch.relu(torch.randn((N, ho, wo, cin2), generator=g)).to(dev)
    return _check(dev, _phase(dev, g, x1, cout, 1, 0, stride), _phase(dev, g, x2, cout, 1, 0, 1), kind, block_n, **kw)


def _ksplit(dev, kind, block_n, N, H, W, cin, cout, seed=0, **kw):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, H, W, cin), generator=g).to(dev)
    p1 = _phase(dev, g, x, cout, 3, 1, 1, 0, 5)
    p2 = dict(p1, tap0=5, ntaps=4, scale=p1["scale"], shift=torch.zeros_like(p1["shift"]))
    return _check(dev, p1, p2, kind, block_n, **kw)


# [8, 80, 128] -> 40 x 64 at stride 2: 160 M-tiles, 2 or 4 N-tiles -- two to five tiles per persistent CTA
@pytest.mark.parametrize("kind", ["tf32", "f16"])
@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("cin1", [64, 256])
def test_two_phase_downsample(dev, kind, block_n, cin1):
    """The first bottleneck of a ResNet layer: a stride-2 1x1 downsample (K = 64 or 256) as phase 1 of conv3 (another Cin)."""
    _downsample(dev, kind, block_n, 8, 80, 128, cin1, 128, 256, 2)


@pytest.mark.parametrize("kind", ["tf32", "f16"])
@pytest.mark.parametrize("block_n", [64, 128])
def test_two_phase_mask_head_ksplit(dev, kind, block_n):
    """A mask-head conv (3x3, K = 2304) split into filter taps [0,5) and [5,9) over the same input, 64 RoIs of 14 x 14."""
    _ksplit(dev, kind, block_n, 64, 14, 14, 256, 256)


@pytest.mark.parametrize("kind", ["tf32", "f16"])
def test_two_phase_long_k_both_phases(dev, kind):
    """Two full 3x3 convolutions (K = 2304 each) over different inputs: 64-wide tiles with three rotating main accumulators in the
    tf32 kind, restarted at phase 2's first k-block."""
    g = torch.Generator().manual_seed(3)
    x1 = torch.randn((4, 20, 24, 256), generator=g).to(dev)
    x2 = torch.randn((4, 20, 24, 256), generator=g).to(dev)
    _check(dev, _phase(dev, g, x1, 128, 3, 1, 1), _phase(dev, g, x2, 128, 3, 1, 1), kind, 64)


@pytest.mark.parametrize("kind", ["tf32", "f16"])
@pytest.mark.parametrize("case", [
    (1, 14, 14, 512, 256, 1024, 2),        # 7 x 7 = 49-pixel boxes, like the C4 res5 block 0
    (3, 10, 9, 64, 32, 64, 2),             # 5 x 5 maps, 64 channels: one 64-wide N-tile
    (2, 5, 7, 32, 64, 128, 1)])            # 35-pixel box, stride 1
def test_two_phase_small_box(dev, kind, case):
    N, H, W, cin1, cin2, cout, stride = case
    _downsample(dev, kind, 0, N, H, W, cin1, cin2, cout, stride)


@pytest.mark.parametrize("kind", ["tf32", "f16"])
def test_two_phase_small_box_ksplit(dev, kind):
    _ksplit(dev, kind, 0, 1, 7, 7, 256, 256)


@pytest.mark.parametrize("kind", ["tf32", "f16"])
def test_two_phase_per_image_mask(dev, kind):
    """The MASK instantiation: a batch of differently-sized images on a padded canvas.  Output pixels outside each image are zero
    and the rest equal the composition."""
    info = torch.tensor([[256, 384, 1.0, 0, 0], [200, 301, 1.0, 0, 0], [96, 384, 1.0, 0, 0], [9, 17, 1.0, 0, 0]], device=dev)
    y, _ = _downsample(dev, kind, 0, 4, 64, 96, 128, 64, 256, 2, im_info=info, im_stride=8)
    assert y.shape == (4, 32, 48, 256)
    for n, (h, w) in enumerate([(32, 48), (25, 38), (12, 48), (2, 3)]):
        assert y[n, :h, :w].abs().sum() > 0
        assert not y[n, h:].any() and not y[n, :, w:].any()


def test_two_phase_range_flag_from_phase1(dev):
    """A phase-1 input that fp16 cannot hold raises the range flag, as the separate phase-1 launch does."""
    g = torch.Generator().manual_seed(9)
    x1 = torch.randn((2, 16, 16, 64), generator=g).to(dev)
    x1[1, 14, 6, 3] = 1.0e5
    x2 = torch.randn((2, 8, 8, 64), generator=g).to(dev)
    _, flag = _check(dev, _phase(dev, g, x1, 256, 1, 0, 2), _phase(dev, g, x2, 256, 1, 0, 1), "f16", 0)
    assert flag == 1


def test_two_phase_refuses_other_tile_shapes(dev):
    """Phases whose separate launches would use other tile shapes are refused: the result could not be the composition's."""
    from detectorch_b200 import ops
    g = torch.Generator().manual_seed(1)
    x1 = torch.randn((2, 8, 8, 1024), generator=g).to(dev)     # tf32, K = 1024: 64-wide tiles, three accumulators
    x2 = torch.randn((2, 8, 8, 512), generator=g).to(dev)      # tf32, K = 512: 128-wide tiles
    with pytest.raises(RuntimeError):
        ops.conv2d_nhwc_two_phase(_phase(dev, g, x2, 256, 1, 0, 1), phase1=_phase(dev, g, x1, 256, 1, 0, 1), kind="tf32")

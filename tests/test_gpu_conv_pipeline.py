"""GPU tests of the f16 conv main loop at the shapes where its pipeline bookkeeping changes: k-blocks per tile around the
pipeline depth (5 stages at 128-wide tiles, 6 at 64-wide), several tiles per persistent CTA (barrier phases wrap across tiles),
TMA boxes smaller than 128 pixels, and residual layers (the residual tile is loaded during the main loop)."""
import pytest
import torch

from test_gpu_ops import _conv_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


# [4, 40, 64, Cin] -> 10240 output pixels = 80 M-tiles; with 2 or 4 N-tiles every CTA runs 2-3 tiles
@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("cin,k,pad", [(32, 1, 0), (128, 1, 0), (160, 1, 0), (192, 1, 0), (224, 1, 0), (32, 3, 1)])
def test_conv_f16_kblocks_per_tile(dev, block_n, cin, k, pad):
    """1, 4, 5, 6, 7 and 9 k-blocks per tile (the last one, at 64-wide tiles, with three rotating main accumulators)."""
    assert _conv_case(dev, 4, 40, 64, cin, 256, k, pad, 1, kind="f16", force_block_n=block_n) < 1e-4


@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("cin,k,pad", [(160, 1, 0), (32, 3, 1), (224, 1, 0)])
def test_conv_f16_residual_several_tiles_per_cta(dev, block_n, cin, k, pad):
    assert _conv_case(dev, 4, 40, 64, cin, 256, k, pad, 1, res=True, relu=True, kind="f16", force_block_n=block_n) < 1e-4


@pytest.mark.parametrize("case", [
    (1, 7, 7, 256, 256, 3, 1, 1, False),      # 49-pixel box
    (1, 5, 5, 160, 128, 1, 0, 1, False),      # 25-pixel box
    (1, 7, 7, 128, 256, 1, 0, 1, True),       # 49-pixel box, residual
    (3, 9, 11, 64, 64, 3, 1, 1, True)])       # 99-pixel box, residual, 64-wide
def test_conv_f16_small_box(dev, case):
    *shape, res = case
    assert _conv_case(dev, *shape, res=res, relu=res, kind="f16") < 1e-4


def test_conv_f16_small_box_range_flag(dev):
    """Rows past a box smaller than 128 pixels hold whatever an earlier tile left in shared memory: they must not raise the range
    flag, while an out-of-range value inside the box must."""
    from detectorch_b200 import ops
    g = torch.Generator().manual_seed(5)
    w = (torch.randn((256, 128), generator=g) * 0.05).to(dev)
    one, zero = torch.ones(256, device=dev), torch.zeros(256, device=dev)
    flag = torch.zeros((1,), dtype=torch.int32, device=dev)
    # fill the A stages of every SM with values fp16 cannot hold (full 128-pixel boxes)
    big = torch.full((4, 40, 64, 128), 1.0e5, device=dev)
    ops.conv2d_nhwc(big, w, one, zero, 1, 1, 0, 1, kind="f16", range_flag=flag)
    torch.cuda.synchronize()
    assert int(flag.item()) == 1
    flag.zero_()
    x = torch.randn((1, 7, 7, 128), generator=g).to(dev)          # one 49-pixel box
    ops.conv2d_nhwc(x, w, one, zero, 1, 1, 0, 1, kind="f16", range_flag=flag)
    assert int(flag.item()) == 0
    x[0, 6, 6, 127] = 1.0e5                                        # last pixel of the box, last channel
    ops.conv2d_nhwc(x, w, one, zero, 1, 1, 0, 1, kind="f16", range_flag=flag)
    assert int(flag.item()) == 1

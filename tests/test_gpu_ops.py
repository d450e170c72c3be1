"""GPU parity of the operator boundary (upfirdn2d, fused_leaky_relu) through the C ABI:
CUDA path vs the CPU oracle and vs the committed reference-generated golden vectors."""
import os

import numpy as np
import pytest
import torch

from oracle import stylegan2_oracle as O
from tests.gpu_util import TOL_FP32

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture(scope="module")
def op():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import hairfastgan_b200.op as op
    return op


def test_upfirdn2d_golden_all_modes(op, golden_dir):
    g = np.load(os.path.join(golden_dir, "ops.npz"))
    x = torch.from_numpy(g["x"]).cuda()
    names = sorted(k[:-3] for k in g.files if k.endswith("__y"))
    for n in names:
        up, down, p0, p1 = (int(v) for v in g[n + "__cfg"])
        y = op.upfirdn2d(x, torch.from_numpy(g[n + "__k"]).cuda(), up=up, down=down, pad=(p0, p1))
        ref = torch.from_numpy(g[n + "__y"])
        assert y.shape == ref.shape, n
        err = float((y.cpu() - ref).abs().max())
        assert err < TOL_FP32, (n, err)


@pytest.mark.parametrize("shape,up,down,pad", [
    ((2, 8, 65, 65), 1, 1, (1, 1)),      # Blur after the up-conv: (2R+1)^2 -> (2R)^2, model.py:252-263
    ((2, 3, 64, 64), 2, 1, (2, 1)),      # RGB skip Upsample, model.py:35-53
    ((1, 4, 64, 64), 1, 2, (1, 1)),      # Downsample
    ((1, 2, 37, 53), 1, 1, (2, 1)),      # ragged sizes (tile tails, unaligned rows)
    ((1, 2, 37, 53), 2, 1, (2, 1)),
    ((3, 1, 5, 7), 3, 2, (2, 3)),        # general path
    ((1, 2, 4, 4), 1, 1, (-1, 1)),       # negative pad = crop
])
def test_upfirdn2d_vs_oracle(op, shape, up, down, pad):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(*shape, generator=g)
    k = torch.randn(4, 4, generator=g)
    y = op.upfirdn2d(x.cuda(), k.cuda(), up=up, down=down, pad=pad)
    ref = O.upfirdn2d_ref(x, k, up, down, pad)
    assert y.shape == ref.shape
    assert float((y.cpu() - ref).abs().max()) < TOL_FP32 * 4


@pytest.mark.parametrize("shape,up,down,pad", [
    # TMA bulk strips (full-width rows fetched with cp.async.bulk): up 1 = the blur after the up-conv
    ((2, 2, 131, 257), 1, 1, (1, 1)),    # rows only 4-byte aligned
    ((1, 4, 70, 129), 1, 1, (2, 1)),     # padding rows above, one padding column right
    ((1, 4, 200, 1025), 1, 1, (1, 1)),   # the 1024-wide case (4 columns per thread), several strips
    ((4, 1, 67, 1027), 1, 1, (0, 0)),    # no padding at all
    ((1, 4, 66, 300), 1, 1, (3, 3)),     # widest padding, 2 columns per thread
    ((1, 4, 9, 128), 1, 1, (0, 3)),      # a single short strip
    # down 2 (Downsample / ConvLayer blur)
    ((2, 2, 131, 257), 1, 2, (1, 1)),
    ((1, 4, 70, 1024), 1, 2, (1, 1)),
    ((1, 4, 66, 1039), 1, 2, (2, 3)),    # out_w = 521: 4 columns per thread
    ((1, 4, 67, 300), 1, 2, (0, 0)),
    ((1, 4, 9, 128), 1, 2, (3, 0)),
    # up 2 (RGB-skip Upsample), pad (2,1)
    ((2, 2, 37, 65), 2, 1, (2, 1)),
    ((1, 4, 70, 512), 2, 1, (2, 1)),
    ((1, 4, 35, 1024), 2, 1, (2, 1)),    # 4 columns per thread
    ((1, 4, 3, 129), 2, 1, (2, 1)),
    ((1, 4, 1, 64), 2, 1, (2, 1)),       # one input row
])
@pytest.mark.parametrize("separable", [True, False])
def test_upfirdn2d_bulk_paths_vs_oracle(op, shape, up, down, pad, separable):
    g = torch.Generator().manual_seed(8)
    x = torch.randn(*shape, generator=g)
    k = O.make_kernel([1, 3, 3, 1]) * (up ** 2) if separable else torch.randn(4, 4, generator=g)
    ref = O.upfirdn2d_ref(x, k, up, down, pad)
    y = op.upfirdn2d(x.cuda(), k.cuda(), up=up, down=down, pad=pad)
    assert y.shape == ref.shape
    assert float((y.cpu() - ref).abs().max()) < TOL_FP32 * 4
    # the same call on a 4-byte-offset view takes the general kernel instead: both paths must agree
    buf = torch.empty(x.numel() + 1, device="cuda")
    xv = buf[1:].view(shape)
    xv.copy_(x)
    y2 = op.upfirdn2d(xv, k.cuda(), up=up, down=down, pad=pad)
    assert float((y2 - y).abs().max()) < 1e-5


def test_upfirdn2d_blur_full_size_both_paths(op):
    """The north_star blur shape [B*C, 1025, 1025] -> 1024^2 (model.py:252-263) at full size: TMA bulk path vs the
    general kernel on an unaligned view of the same data, plus the DC gain of the normalised FIR in the interior."""
    k = (O.make_kernel([1, 3, 3, 1]) * 4).cuda()
    x = torch.randn(1, 8, 1025, 1025, device="cuda")
    y = op.upfirdn2d(x, k / 4, up=1, down=1, pad=(1, 1))
    assert y.shape == (1, 8, 1024, 1024)
    buf = torch.empty(x.numel() + 1, device="cuda")
    xv = buf[1:].view(x.shape)
    xv.copy_(x)
    y2 = op.upfirdn2d(xv, k / 4, up=1, down=1, pad=(1, 1))
    assert float((y2 - y).abs().max()) < 1e-5
    ones = torch.ones(1, 4, 1025, 1025, device="cuda")
    y1 = op.upfirdn2d(ones, k / 4, up=1, down=1, pad=(1, 1))
    assert float((y1[:, :, 2:-2, 2:-2] - 1).abs().max()) < 1e-6


def test_upfirdn2d_other_kernel_sizes(op):
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 3, 12, 10, generator=g)
    for kh, kw in [(1, 1), (2, 2), (3, 3), (5, 3), (6, 6)]:
        k = torch.randn(kh, kw, generator=g)
        y = op.upfirdn2d(x.cuda(), k.cuda(), up=2, down=1, pad=(kh // 2, kw // 2))
        ref = O.upfirdn2d_ref(x, k, 2, 1, (kh // 2, kw // 2)) if kh == kw else None
        if ref is not None:
            assert float((y.cpu() - ref).abs().max()) < TOL_FP32 * 4


def test_upfirdn2d_full_size_properties(op):
    """1024^2 RGB upsample at full size: linearity + DC gain (size-independent properties)."""
    k = (O.make_kernel([1, 3, 3, 1]) * 4).cuda()
    a = torch.randn(1, 3, 512, 512, device="cuda")
    b = torch.randn(1, 3, 512, 512, device="cuda")
    ya, yb = op.upfirdn2d(a, k, up=2, pad=(2, 1)), op.upfirdn2d(b, k, up=2, pad=(2, 1))
    yab = op.upfirdn2d(a + 2 * b, k, up=2, pad=(2, 1))
    assert yab.shape == (1, 3, 1024, 1024)
    assert float((yab - (ya + 2 * yb)).abs().max()) < 1e-4
    ones = torch.ones(1, 1, 512, 512, device="cuda")
    y1 = op.upfirdn2d(ones, k, up=2, pad=(2, 1))
    assert float((y1[:, :, 2:-2, 2:-2] - 1).abs().max()) < 1e-6      # interior: unit DC gain


def test_fused_leaky_relu(op, golden_dir):
    g = np.load(os.path.join(golden_dir, "ops.npz"))
    y = op.fused_leaky_relu(torch.from_numpy(g["lrelu_x"]).cuda(), torch.from_numpy(g["lrelu_b"]).cuda())
    assert float((y.cpu() - torch.from_numpy(g["lrelu_y"])).abs().max()) < 1e-6
    y = op.fused_leaky_relu(torch.from_numpy(g["lrelu2d_x"]).cuda(), torch.from_numpy(g["lrelu_b"]).cuda())
    assert float((y.cpu() - torch.from_numpy(g["lrelu2d_y"])).abs().max()) < 1e-6
    # module form, vectorised (HW % 4 == 0) and scalar (odd HW) paths, non-default slope/scale
    m = op.FusedLeakyReLU(6, negative_slope=0.1, scale=1.5).cuda()
    m.bias.data.normal_()
    for hw in [(8, 8), (5, 7)]:
        x = torch.randn(2, 6, *hw, device="cuda")
        ref = O.fused_leaky_relu_ref(x.cpu(), m.bias.data.cpu(), 0.1, 1.5)
        assert float((m(x).cpu() - ref).abs().max()) < 1e-6
    # empty input
    assert op.fused_leaky_relu(torch.empty(0, 6, 4, 4, device="cuda"), m.bias.data).shape == (0, 6, 4, 4)


def test_cpu_tensor_is_rejected(op):
    with pytest.raises(RuntimeError):
        op.upfirdn2d(torch.randn(1, 1, 4, 4), torch.ones(2, 2))
    with pytest.raises(RuntimeError):
        op.fused_leaky_relu(torch.randn(1, 4, 2, 2), torch.zeros(4))

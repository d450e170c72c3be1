"""GPU parity of both mainloops of the wgmma convolution against the oracle: the column-shift path (one
(8 + 2) x 16 activation box per channel chunk and column shift; stride-1 3x3 layers on 16-pixel-wide tiles of one
sample) and the per-tap path that the narrower, strided and 1x1 layers keep.  Which path a shape takes is decided
from the shape alone (see tests/test_conv_plan_halo_cpu.py)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import stylegan2_oracle as O
from tests.gpu_util import TOL_RGB, TOL_SINGLE, dtype_name, enc_dtype_name, rel_err

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

TOL_CONV = {"bf16": 4e-2, "fp16": 6e-3}     # one encoder conv incl. 16-bit rounding of its input and output


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


# (Cin, Cout, H, W, up, batch): column-shift path unless marked
STYLED = [
    (64, 64, 16, 16, False, 3),      # two tile rows per sample: halo rows come from the neighbouring tile
    (128, 128, 24, 32, False, 2),    # odd tile-row count, two tile columns, image edges on all sides
    (32, 32, 32, 32, False, 2),      # 32-channel chunks (SWIZZLE_64B)
    (64, 64, 16, 16, True, 3),       # polyphase up-conv
    (256, 128, 32, 16, True, 2),
    (64, 64, 8, 8, False, 3),        # 8-pixel-wide tile, two samples per tile: per-tap path
]


@pytest.mark.parametrize("cin,cout,h,w,up,batch", STYLED)
def test_styled_conv_vs_oracle(dev, cin, cout, h, w, up, batch):
    import hairfastgan_b200.model as M
    torch.manual_seed(cin + h + w)
    m = M.StyledConv(cin, cout, 3, 512, upsample=up)
    m.noise.weight.data.normal_(0, 0.3)
    m.activate.bias.data.normal_(0, 0.3)
    m.conv.modulation.bias.data.add_(0.1 * torch.randn(cin))
    g = torch.Generator().manual_seed(h * w)
    x = torch.randn(batch, cin, h, w, generator=g)
    st = torch.randn(batch, 512, generator=g)
    ho, wo = (2 * h, 2 * w) if up else (h, w)
    nz = torch.randn(batch, 1, ho, wo, generator=g)
    ref = O.styled_conv_ref(x, st, dict(m.state_dict()), "", nz, up)
    y = m.to(dev)(x.to(dev), st.to(dev), noise=nz.to(dev))
    assert y.shape == ref.shape
    e, _ = rel_err(y, ref)
    assert e < TOL_SINGLE[dtype_name()], e


def test_generator_fused_torgb_vs_oracle(dev):
    """Generator(64): the 16^2..64^2 layers run the column-shift path with the fused ToRGB partial sums and noise."""
    import hairfastgan_b200.model as M
    params = O.synth_generator_params(size=64, seed=5)
    gen = M.Generator(64, 512, 8)
    gen.load_state_dict(params, strict=True)
    gen = gen.to(dev).eval()
    lat = torch.randn(3, gen.n_latent, 512, generator=torch.Generator().manual_seed(6))
    noise = O.synth_noise(64, batch=3, seed=7)
    img, _ = gen([lat.to(dev)], input_is_latent=True, noise=[n.to(dev) for n in noise])
    ref, _ = O.generator_ref(params, lat, noise)
    e, _ = rel_err(img, ref)
    assert e < TOL_RGB[dtype_name()], e


# (Cin, Cout, H, W, stride, groups, act, residual, post, y16b): column-shift path unless stride 2 / W < 16
ENC = [
    (64, 64, 32, 32, 1, 1, 1, True, False, False),     # PReLU + residual
    (64, 64, 16, 48, 1, 1, 3, True, True, True),       # activation after the residual, second 16-bit output
    (32, 64, 32, 16, 1, 1, 2, False, False, True),     # 32-channel chunks
    (128, 128, 16, 16, 1, 2, 1, False, False, False),  # grouped N tiles
    (64, 128, 32, 32, 2, 1, 1, False, False, False),   # stride 2: per-tap path
    (64, 64, 8, 8, 1, 1, 1, True, False, False),       # 8-pixel-wide tile: per-tap path
]


@pytest.mark.parametrize("cin,cout,h,w,stride,groups,act,residual,post,y16b", ENC)
def test_encoder_conv_variants(dev, cin, cout, h, w, stride, groups, act, residual, post, y16b):
    import hairfastgan_b200.nn16 as N
    g = torch.Generator().manual_seed(cin + cout + h + w)
    x = torch.randn(2, cin, h, w, generator=g)
    wt = torch.randn(cout, cin // groups, 3, 3, generator=g) / (3 * (cin // groups) ** 0.5)
    osc, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.3
    slope = torch.rand(cout, generator=g) * 0.5
    s2, b2 = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.3
    a = F.conv2d(x, wt, None, stride, 1, 1, groups) * osc.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    res = torch.randn_like(a) if residual else None

    def act_fn(v):
        if act == 1:
            return torch.where(v > 0, v, v * slope.view(1, -1, 1, 1))
        return F.leaky_relu(v, 0.01) if act == 2 else F.relu(v)

    if residual and post:
        ref = act_fn(a + res)
    else:
        ref = act_fn(a) + (res if residual else 0)
    pc = N.PackedConv2d(wt.to(dev), osc.to(dev), stride=stride, groups=groups)
    y16, yb, y32 = pc(N.to_nhwc16(x.to(dev)), shift=shift.to(dev), act=act,
                      slope=slope.to(dev) if act == 1 else None, slope0=0.01,
                      residual16=N.to_nhwc16(res.to(dev)) if residual else None, want_y32=True,
                      y16b_affine=(s2.to(dev), b2.to(dev)) if y16b else None, act_after_residual=post)
    tol = TOL_CONV[enc_dtype_name()]
    assert rel_err(y32, ref)[0] < tol
    assert rel_err(N.to_nchw32(y16), ref)[0] < tol * 1.5
    if y16b:
        refb = ref * s2.view(1, -1, 1, 1) + b2.view(1, -1, 1, 1)
        assert rel_err(N.to_nchw32(yb), refb)[0] < tol * 1.5

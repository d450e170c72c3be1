"""Exact-arithmetic tests of the wgmma convolution (csrc/hf_conv_tc.cu).

The kernel multiplies 16-bit operands and accumulates in fp32.  With small integer activations and weights every
product and every partial sum is an integer below 2^24, exact in fp32 in any summation order, so the raw output must
equal a float64 reference BIT FOR BIT: a dropped, duplicated or misplaced tap, channel chunk, halo row, sample or
N tile changes integers and no tolerance can absorb it.  The cases (tests/conv_exact_cases.py) reach every
(K chunk, N tile, mainloop) kernel variant; each asserts through the plan query that it runs the variant it names.

A second tier keeps the integer accumulators and checks the fp32 epilogue arithmetic (shift, activations, residual,
second output, demodulation, noise) against float64 at a few fp32 ulps, 16-bit outputs at one ulp of their type.

The fused ToRGB partial sums are not covered here: they exist only inside hf_generator_forward, where the conv
inputs are the 16-bit rounded activations of the previous layer, never integers; tests/test_gpu_conv_halo.py::
test_generator_fused_torgb_vs_oracle keeps checking them against the oracle."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import stylegan2_oracle as O
from tests import conv_exact_cases as T
from tests.gpu_util import dtype_name

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

_SMS_ASSUMED = 132                       # the table is only enumerated with this count; cases rebuild it per device
ENC_NAMES = [c.name for c in T.encoder_cases(_SMS_ASSUMED)]
GEN_NAMES = [c.name for c in T.generator_cases(_SMS_ASSUMED)]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def sms(dev):
    from hairfastgan_b200 import _lib
    _lib.use_device(dev.index)
    n = _lib.lib().hf_sm_count()
    assert n > 0
    return n


@pytest.fixture()
def dt(hf_dtype):
    """(library dtype code, torch dtype) of this module run."""
    from hairfastgan_b200 import _lib
    return (_lib.HF_F16, torch.float16) if dtype_name() == "fp16" else (_lib.HF_BF16, torch.bfloat16)


# ------------------------------------------------------------------------------------------------ operands
def ints(g, shape, lo, hi, zero_frac=0.2):
    """Seeded integers in [lo, hi] as float64, a fraction of them forced to zero."""
    v = torch.randint(lo, hi + 1, shape, generator=g).double()
    return v * (torch.rand(shape, generator=g) >= zero_frac)


def nhwc16(x, tdt, dev, c_pad=None):
    """[B,C,H,W] integer-valued float64 -> the 16-bit NHWC device tensor the kernel reads (zero channel padding)."""
    if c_pad is not None and c_pad > x.shape[1]:
        x = F.pad(x, (0, 0, 0, 0, 0, c_pad - x.shape[1]))
    y = x.permute(0, 2, 3, 1).contiguous().to(tdt).to(dev)
    assert torch.equal(y.cpu().double().permute(0, 3, 1, 2), x)          # the operands are exact in 16 bits
    return y


def nchw64(y16):
    return y16.cpu().double().permute(0, 3, 1, 2)


def first_mismatch(got, ref, what):
    bad = (got != ref).nonzero()
    if bad.numel() == 0:
        return ""
    b, o, y, x = [int(v) for v in bad[0]]
    return (f"{what}: {bad.shape[0]} of {ref.numel()} values differ; first at sample {b} channel {o} y {y} x {x}: "
            f"got {float(got[b, o, y, x])!r}, expected {float(ref[b, o, y, x])!r}")


def assert_equal(got, ref, what):
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.equal(got, ref), first_mismatch(got, ref, what)


def enc_operands(c, seed):
    g = torch.Generator().manual_seed(seed)
    x = ints(g, (c.batch, c.cin, c.h, c.w), -3, 3)
    if c.hot_last_row:        # what the first row of the next sample (and the zero fill below the image) must not see
        x[:, :, -1, :] = torch.randint(40, 61, (c.batch, c.cin, c.w), generator=g).double()
    w = ints(g, (c.cout, c.cin // c.groups, c.k, c.k), -2, 2)
    assert 9 * (c.cin // c.groups) * 60 * 2 < 2 ** 24
    ref = F.conv2d(x, w, None, c.stride, c.k // 2, 1, c.groups)
    return x, w, ref


def run_enc(c, x, w, dt, dev, out_scale=None, **kw):
    import hairfastgan_b200.nn16 as N
    pc = N.PackedConv2d(w.float().to(dev), None if out_scale is None else out_scale.float().to(dev), stride=c.stride,
                        groups=c.groups, cin_pad=c.cin_pad, dtype=dt[0])
    return pc(nhwc16(x, dt[1], dev, c.cin_pad), **kw)


# ------------------------------------------------------------------------------------------------ encoder form, exact
@pytest.mark.parametrize("name", ENC_NAMES)
def test_encoder_conv_bit_exact(dev, sms, dt, name):
    from hairfastgan_b200 import _lib
    c = {k.name: k for k in T.encoder_cases(sms)}[name]
    T.check_claim(c, T.encoder_plan(_lib, c, dt[0]), sms)
    x, w, ref = enc_operands(c, seed=len(name) * 131 + c.cin + c.h)
    ref16 = ref.float().to(dt[1]).double()                 # round-to-nearest-even of the 16-bit store
    if c.y32_only:
        y16, yb, y32 = run_enc(c, x, w, dt, dev, want_y16=False, want_y32=True)
        assert y16 is None and yb is None
        assert_equal(y32.cpu().double(), ref, "y32")
        return
    # the 16-bit output alone (epilogue variant without residual / second output / fp32 store)
    y16, _, _ = run_enc(c, x, w, dt, dev)
    assert_equal(nchw64(y16), ref16, "y16")
    # every output at once, still exact: integer residual, power-of-two second scale, integer second shift
    g = torch.Generator().manual_seed(c.cout + c.w)
    res = ints(g, tuple(ref.shape), -8, 8)
    s2 = torch.tensor([0.5, 1.0, 2.0]).double()[torch.randint(0, 3, (c.cout,), generator=g)]
    b2 = ints(g, (c.cout,), -4, 4)
    y16, yb, y32 = run_enc(c, x, w, dt, dev, residual16=nhwc16(res, dt[1], dev), want_y32=True,
                           y16b_affine=(s2.to(dev), b2.to(dev)))
    v = ref + res
    vb = v * s2.view(1, -1, 1, 1) + b2.view(1, -1, 1, 1)
    assert_equal(y32.cpu().double(), v, "y32 with residual")
    assert_equal(nchw64(y16), v.float().to(dt[1]).double(), "y16 with residual")
    assert_equal(nchw64(yb), vb.float().to(dt[1]).double(), "y16b")


def test_encoder_residual_and_second_output_alone_bit_exact(dev, sms, dt):
    """The two 16-bit-only epilogue variants (residual without y16b, y16b without residual) on both mainloops."""
    cases = {k.name: k for k in T.encoder_cases(sms)}
    for name in ("shift_kc64_n64_h24_w48", "tap_kc64_n32_4x4_b5"):
        c = cases[name]
        x, w, ref = enc_operands(c, seed=77)
        g = torch.Generator().manual_seed(78)
        res = ints(g, tuple(ref.shape), -8, 8)
        s2 = torch.tensor([0.5, 1.0, 2.0]).double()[torch.randint(0, 3, (c.cout,), generator=g)]
        b2 = ints(g, (c.cout,), -4, 4)
        y16, yb, _ = run_enc(c, x, w, dt, dev, residual16=nhwc16(res, dt[1], dev))
        assert yb is None
        assert_equal(nchw64(y16), (ref + res).float().to(dt[1]).double(), name + " y16 = conv + residual")
        y16, yb, _ = run_enc(c, x, w, dt, dev, y16b_affine=(s2.to(dev), b2.to(dev)))
        vb = ref * s2.view(1, -1, 1, 1) + b2.view(1, -1, 1, 1)
        assert_equal(nchw64(y16), ref.float().to(dt[1]).double(), name + " y16")
        assert_equal(nchw64(yb), vb.float().to(dt[1]).double(), name + " y16b")


# ------------------------------------------------------------------------------------------------ impulse probes
# (cin, cout, H, W, mainloop, [(y, x)]): one sample per probe position and channel
IMPULSE = [
    (128, 32, 16, 32, T.SHIFT, [(0, 0), (0, 31), (15, 0), (15, 31), (7, 15), (7, 16), (8, 15), (8, 16)]),
    (128, 32, 8, 8, T.TAP, [(0, 0), (0, 7), (7, 0), (7, 7), (3, 4)]),
]


@pytest.mark.parametrize("cin,cout,h,w,loop,positions", IMPULSE)
def test_impulse_response_is_the_flipped_footprint(dev, sms, dt, cin, cout, h, w, loop, positions):
    """One non-zero input element per sample against weights whose nine taps are 1..9 (sign by channel parity): the
    output is the flipped 3x3 footprint around the impulse, clipped at the image edge, and nothing else.  Positions:
    the image corners and both sides of the tile seams (x = 15 | 16, y = 7 | 8); channels: first and last of a
    64-channel K chunk."""
    from hairfastgan_b200 import _lib
    probes = [(y, x, ch) for (y, x) in positions for ch in (0, 63, 64, 127)]
    c = T.Enc("impulse", cin, cout, h, w, len(probes), (64, 32, loop))
    T.check_claim(c, T.encoder_plan(_lib, c, dt[0]), sms)
    xin = torch.zeros(len(probes), cin, h, w, dtype=torch.float64)
    for b, (y, x, ch) in enumerate(probes):
        xin[b, ch, y, x] = 1.0
    taps = torch.arange(1, 10, dtype=torch.float64).view(1, 1, 3, 3)
    sign = 1.0 - 2.0 * ((torch.arange(cout).view(-1, 1) + torch.arange(cin).view(1, -1)) % 2).double()
    wgt = taps * sign.view(cout, cin, 1, 1)
    ref = F.conv2d(xin, wgt, None, 1, 1)
    _, _, y32 = run_enc(c, xin, wgt, dt, dev, want_y16=False, want_y32=True)
    got = y32.cpu().double()
    bad = (got != ref).nonzero()
    if bad.numel():
        b, o, oy, ox = [int(v) for v in bad[0]]
        y, x, ch = probes[b]
        dy, dx = y - oy + 1, x - ox + 1             # the tap that carries the impulse to this output pixel
        tap = f"tap (dy={dy}, dx={dx})" if 0 <= dy < 3 and 0 <= dx < 3 else "outside the 3x3 footprint"
        pytest.fail(f"impulse at y={y} x={x} channel {ch}: output channel {o} pixel y={oy} x={ox} ({tap}) is "
                    f"{float(got[b, o, oy, ox])}, expected {float(ref[b, o, oy, ox])}; {bad.shape[0]} values differ")


# ------------------------------------------------------------------------------------------------ determinism
def test_two_calls_give_identical_outputs(dev, sms, dt):
    cases = {k.name: k for k in T.encoder_cases(sms)}
    for name in ("persist_n128_two_n_tiles", "tap_kc64_n128_8x8_fill"):
        c = cases[name]
        import hairfastgan_b200.nn16 as N
        g = torch.Generator().manual_seed(5)
        x = torch.randn(c.batch, c.h, c.w, c.cin, generator=g).to(dt[1]).to(dev)
        w = torch.randn(c.cout, c.cin, 3, 3, generator=g) / (3 * c.cin ** 0.5)
        shift = torch.randn(c.cout, generator=g).to(dev)
        pc = N.PackedConv2d(w.to(dev), None, dtype=dt[0])
        a = pc(x, shift=shift, act=2, slope0=0.01, want_y32=True)
        b = pc(x, shift=shift, act=2, slope0=0.01, want_y32=True)
        assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]), name


# ------------------------------------------------------------------------------------------------ encoder form, fp32 epilogue
def ulp16(ref, tdt):
    """Spacing of the 16-bit type at |ref| (float64 tensor)."""
    mant, emin = (10, -14) if tdt == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin)))
    return torch.pow(torch.tensor(2.0, dtype=torch.float64), e - mant)


def assert_close_fp32(got, ref, mag, what, extra=None):
    """|got - ref| <= 4e-6 * mag + 1e-6 (+ extra), mag = the largest magnitude among the terms that were added to
    form ref (>= |ref|): fp32 rounding is relative to the operands, not to a cancelled sum."""
    tol = 4e-6 * torch.maximum(mag, ref.abs()) + 1e-6 + (0 if extra is None else extra)
    err = (got - ref).abs()
    over = (err > tol).nonzero()
    if over.numel():
        i = tuple(int(v) for v in over[0])
        pytest.fail(f"{what}: {over.shape[0]} values out of bound; first at {i}: got {float(got[i])!r}, expected "
                    f"{float(ref[i])!r}, bound {float(tol[i]):.3g}")


# (case name, act, residual, act after residual, y16b, power-of-two out_scale)
EPILOGUES = [
    ("shift_kc64_n64_h24_w48", 1, True, False, True, True),      # PReLU, then + residual; second output; folded scale
    ("shift_kc32_n128_fill", 2, True, True, True, False),        # LeakyReLU after the residual add
    ("shift_groups2_n32", 3, False, False, True, True),          # ReLU
    ("tap_kc64_n32_4x4_b5", 1, True, True, False, True),
    ("tap_kc64_n64_stride2_fill", 2, True, False, True, False),
    ("tap_1x1_stride2", 3, True, True, True, False),
    ("tap_kc32_n128_1x1_fill", 0, False, False, True, True),     # shift alone
]


@pytest.mark.parametrize("name,act,residual,post,y16b,scaled", EPILOGUES)
def test_encoder_epilogue_fp32_arithmetic(dev, sms, dt, name, act, residual, post, y16b, scaled):
    c = {k.name: k for k in T.encoder_cases(sms)}[name]
    x, w, acc = enc_operands(c, seed=act * 17 + c.cout)
    g = torch.Generator().manual_seed(act + 3)
    col = lambda t: t.view(1, -1, 1, 1)
    osc = torch.pow(2.0, torch.randint(-2, 3, (c.cout,), generator=g).double()) if scaled else None
    shift = torch.randn(c.cout, generator=g).float().double() * 3
    slope = torch.rand(c.cout, generator=g).float().double() * 0.5
    s2 = (torch.rand(c.cout, generator=g).float() + 0.5).double()
    b2 = torch.randn(c.cout, generator=g).float().double()
    res = (torch.randn(tuple(acc.shape), generator=g) * 8).to(dt[1]).double() if residual else None
    slope0 = float(torch.tensor(0.01, dtype=torch.float32))

    def act_fn(v):
        if act == 0:
            return v
        neg = col(slope) if act == 1 else (slope0 if act == 2 else 0.0)
        return torch.where(v > 0, v, v * neg)

    a = (acc * col(osc) if scaled else acc) + col(shift)
    mag = torch.maximum(a.abs(), (acc * col(osc) if scaled else acc).abs())
    if residual:
        v = act_fn(a + res) if post else act_fn(a) + res
        mag = torch.maximum(mag, res.abs())
    else:
        v = act_fn(a)
    vb = v * col(s2) + col(b2)
    kw = dict(shift=shift.float().to(dev), act=act, slope=slope.float().to(dev) if act == 1 else None, slope0=slope0,
              residual16=nhwc16_raw(res, dt[1], dev) if residual else None, act_after_residual=post,
              y16b_affine=(s2.float().to(dev), b2.float().to(dev)) if y16b else None)
    for want_y32 in (True, False):          # the all-outputs epilogue variant, then the 16-bit-only one
        y16, yb, y32 = run_enc(c, x, w, dt, dev, out_scale=osc, want_y32=want_y32, **kw)
        if want_y32:
            assert_close_fp32(y32.cpu().double(), v, mag, f"{name} y32")
        assert_close_fp32(nchw64(y16), v, mag, f"{name} y16 (y32 {want_y32})", extra=ulp16(v, dt[1]))
        if y16b:
            magb = torch.maximum(mag * col(s2), col(b2).abs().expand_as(v))
            assert_close_fp32(nchw64(yb), vb, magb, f"{name} y16b (y32 {want_y32})", extra=ulp16(vb, dt[1]))


def nhwc16_raw(x, tdt, dev):
    """[B,C,H,W] float64 values already representable in the 16-bit type -> NHWC device tensor."""
    return x.permute(0, 2, 3, 1).contiguous().to(tdt).to(dev)


# ------------------------------------------------------------------------------------------------ generator form
def make_modconv(c, seed, demodulate, dev):
    """ModulatedConv2d whose packed 16-bit weights are the integers m: hf_conv_pack multiplies by 1/sqrt(Cin*9), so it
    is handed m*sqrt(Cin*9) and the 16-bit rounding snaps the product back to m.  modulation.weight = 0 makes the style
    scale the bias, a power of two, so x*s is exact in 16 bits."""
    import hairfastgan_b200.model as M
    g = torch.Generator().manual_seed(seed)
    m = M.ModulatedConv2d(c.cin, c.cout, 3, 512, demodulate=demodulate, upsample=bool(c.up))
    wi = ints(g, (c.cout, c.cin, 3, 3), -2, 2)
    m.weight.data = (wi * math.sqrt(c.cin * 9)).float().view(1, c.cout, c.cin, 3, 3)
    m.modulation.weight.data.zero_()
    s = torch.tensor([0.5, 1.0, 2.0]).double()[torch.randint(0, 3, (c.cin,), generator=g)]
    m.modulation.bias.data = s.float()
    x = ints(g, (c.batch, c.cin, c.h, c.w), -3, 3)
    style = torch.randn(c.batch, 512, generator=g)
    return m.to(dev), wi, s, x, style


def modconv_acc(c, m, wi, s, x):
    """float64 accumulator of the modulated conv without demodulation: integers (plain) or multiples of 1/32 (up)."""
    xs = x * s.view(1, -1, 1, 1)
    if not c.up:
        return F.conv2d(xs, wi, None, 1, 1)
    out = F.conv_transpose2d(xs, wi.transpose(0, 1).contiguous(), None, 2, 0)           # model.py:260
    return O.upfirdn2d_ref(out, m.blur.kernel.detach().cpu().double(), pad=(1, 1))       # Blur(pad=(1, 1)), model.py:263


@pytest.mark.parametrize("name", GEN_NAMES)
def test_modulated_conv_bit_exact(dev, sms, dt, name):
    """demodulate = 0, no noise, no activation: y is the accumulator.  The polyphase taps of the up-conv are sums of
    m * {1, 3, 9} / 16 with numerators below 2^6, exact in both 16-bit types, so the up-conv is exact as well."""
    from hairfastgan_b200 import _lib
    c = {k.name: k for k in T.generator_cases(sms)}[name]
    T.check_claim(c, T.generator_plan(_lib, c, dt[0]), sms)
    m, wi, s, x, style = make_modconv(c, len(name) * 7 + c.h, False, dev)
    ref = modconv_acc(c, m, wi, s, x)
    y = m._run(x.float().to(dev), style.to(dev), dtype=dt[0])
    if not c.up:        # the packed operand really is the integer tensor: wpk[o][tap * Cin + c]
        _, blob = m._packed.get(m, dt[0])
        wpk = blob[: c.cout * 9 * c.cin * 2].view(dt[1]).view(c.cout, 9, c.cin).cpu().double()
        assert torch.equal(wpk, wi.permute(0, 2, 3, 1).reshape(c.cout, 9, c.cin)), "packed weights are not integers"
    assert_equal(y.cpu().double(), ref, "y")


@pytest.mark.parametrize("name,noise_batch", [("plain_shift_kc64_n64_fill", 1), ("plain_tap_kc64_8x8", 0),
                                              ("up_shift_kc64", 0), ("up_tap_kc32_4x4", 1)])
def test_styled_conv_epilogue_fp32_arithmetic(dev, sms, dt, name, noise_batch):
    """Demodulation, noise (shared, noise_batch = 1, or per sample), bias + LeakyReLU * sqrt(2) on exact accumulators."""
    c = {k.name: k for k in T.generator_cases(sms)}[name]
    m, wi, s, x, style = make_modconv(c, 11 + c.cout, True, dev)
    acc = modconv_acc(c, m, wi, s, x)
    g = torch.Generator().manual_seed(12)
    nb = noise_batch or c.batch
    noise = torch.randn(nb, 1, acc.shape[2], acc.shape[3], generator=g)
    nw = torch.tensor([0.7])
    bias = torch.randn(c.cout, generator=g)
    d = torch.rsqrt((wi.pow(2).sum((2, 3)) @ s.pow(2)) + 1e-8).view(1, -1, 1, 1)     # same s for every sample
    pre = acc * d + nw.double() * noise.double() + bias.double().view(1, -1, 1, 1)
    ref = torch.where(pre > 0, pre, pre * float(torch.tensor(0.2, dtype=torch.float32))) * math.sqrt(2.0)
    mag = math.sqrt(2.0) * torch.maximum((acc * d).abs(), (nw.double() * noise.double()).abs().expand_as(pre))
    mag = torch.maximum(mag, math.sqrt(2.0) * bias.double().abs().view(1, -1, 1, 1).expand_as(pre))
    y = m._run(x.float().to(dev), style.to(dev), noise=noise.to(dev), noise_weight=nw.to(dev), act_bias=bias.to(dev),
               act=1, dtype=dt[0])
    assert_close_fp32(y.cpu().double(), ref, mag, name)
    # demodulation alone, no tail
    y = m._run(x.float().to(dev), style.to(dev), dtype=dt[0])
    assert_close_fp32(y.cpu().double(), acc * d, (acc * d).abs(), name + " demodulated")

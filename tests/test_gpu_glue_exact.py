"""Exact-arithmetic tests of the SIMT glue kernels around the wgmma convolution (csrc/hf_enc_ops.cu, csrc/hf_seg_ops.cu).

Operands are small integers or dyadic values (power-of-two fractions), so every fp32 intermediate of these kernels is
exact.  The reference is float64 torch on the CPU, rounded ONCE to the output type; `r16` asserts that the float64
value is exact in fp32 first, so the float64 -> fp32 -> 16-bit conversion cannot round twice.  The kernel output must
then equal the reference bit for bit: a misplaced tap, edge row, channel or sample changes an integer, and no tolerance
absorbs it.  Where a kernel rounds in a way exact inputs cannot avoid (1/HW when HW is not a power of two, rsqrtf,
__expf in the sigmoids, bilinear weights whose ratio is not dyadic) the test states a bound of the form
"1 ulp of the output type + k * 2^-24 * sum|terms|" beside the operation and explains k there.

Each case names the dispatch path it takes, derived from the host-side condition of its entry point: vec8 / scalar
(C % 8, 16-byte alignment, bin count), the split count S of the shared channel reduction, the row / scalar bilinear
kernels, the static / opt-in shared memory of the fused arg-max."""
import pytest
import torch
import torch.nn.functional as F

from tests.gpu_util import dtype_name

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

EPS = 2.0 ** -24                        # unit roundoff of fp32


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hairfastgan_b200 import _lib
    _lib.use_device(0)
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def sms(dev):
    from hairfastgan_b200 import _lib
    n = _lib.lib().hf_sm_count()
    assert n > 0
    return n


@pytest.fixture()
def dt(hf_dtype):
    """(library dtype code, torch dtype) of this module run."""
    from hairfastgan_b200 import _lib
    return (_lib.HF_F16, torch.float16) if dtype_name() == "fp16" else (_lib.HF_BF16, torch.bfloat16)


@pytest.fixture(scope="module")
def N(dev):
    import hairfastgan_b200.nn16 as N
    return N


# ------------------------------------------------------------------------------------------------ operands, checks
def ints(g, shape, lo, hi):
    """Seeded integers in [lo, hi] as float64."""
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def pick(g, shape, values):
    """Seeded draws from a list of (dyadic) values as float64."""
    v = torch.tensor(values, dtype=torch.float64)
    return v[torch.randint(0, len(values), shape, generator=g)]


def to16(x, tdt, dev):
    """[B,C,H,W] float64, exact in the 16-bit type -> the NHWC device tensor the kernels read."""
    y = x.permute(0, 2, 3, 1).contiguous().to(tdt).to(dev)
    assert torch.equal(y.cpu().double().permute(0, 3, 1, 2), x), "operand not exact in 16 bits"
    return y


def nchw64(y16):
    return y16.cpu().double().permute(0, 3, 1, 2)


def r16(ref, tdt):
    """float64 reference rounded once to the 16-bit type; it must be exact in fp32 (no double rounding)."""
    f = ref.float()
    assert torch.equal(f.double(), ref), "reference not exact in fp32: the bit-exact comparison would be invalid"
    return f.to(tdt).double()


def ulp16(ref, tdt):
    """Spacing of the 16-bit type at |ref| (float64 tensor)."""
    mant, emin = (10, -14) if tdt == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin)))
    return torch.pow(torch.tensor(2.0, dtype=torch.float64), e - mant)


def assert_equal(got, ref, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    bad = (got != ref) & ~(torch.isnan(got) & torch.isnan(ref))
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail(f"{what}: {int(bad.sum())} of {ref.numel()} values differ; first at {i}: got {float(got[i])!r}, "
                    f"expected {float(ref[i])!r}")


def assert_within(got, ref, bound, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    over = (got - ref).abs() > bound
    if over.any():
        i = tuple(int(v) for v in over.nonzero()[0])
        pytest.fail(f"{what}: {int(over.sum())} of {ref.numel()} values out of bound; first at {i}: got "
                    f"{float(got[i])!r}, expected {float(ref[i])!r}, bound {float(bound[i]):.3g}")


# ------------------------------------------------------------------------------------------------ NCHW fp32 <-> NHWC 16-bit
def _pads(c):
    """Cpad of C itself when even (the entry point rejects an odd Cpad), the next multiple of 2, of 8 and of 32."""
    return sorted({p for p in (c if c % 2 == 0 else None, c + c % 2, -(-c // 8) * 8, -(-c // 32) * 32) if p})


LAYOUT = [(c, p) for c in (3, 8, 19, 70, 130) for p in _pads(c)]
LAYOUT_IDS = [f"c{c}_cpad{p}" + ("_padded" if p > c else "") + ("_ctail" if c % 64 else "") for c, p in LAYOUT]
HW_SHAPES = [(1, 1), (3, 11), (1, 64 * 17 + 5)]          # HW = 1, 33, 1093: a single pixel and two 32-pixel tails


@pytest.mark.parametrize("c,cpad", LAYOUT, ids=LAYOUT_IDS)
def test_nchw_nhwc16_layout_bit_exact(N, dev, dt, c, cpad):
    """y = x * scale[c] + shift[c] in the first C channels, +0.0 (all bits clear) in the padding; the inverse
    conversion is exact, and the round trip through fp32 is the identity on 16-bit data."""
    g = torch.Generator().manual_seed(c * 1000 + cpad)
    for h, w in HW_SHAPES:
        x = ints(g, (2, c, h, w), -40, 40) / 4
        sc = pick(g, (c,), [0.5, 1.0, 2.0, -1.0, 0.25])
        sh = ints(g, (c,), -8, 8) / 2
        for mode in ("scale", "shift", "both"):
            s = sc if mode != "shift" else None
            t = sh if mode != "scale" else None
            ref = x * (1.0 if s is None else s.view(1, -1, 1, 1)) + (0.0 if t is None else t.view(1, -1, 1, 1))
            y = N.to_nhwc16(x.float().to(dev), None if s is None else s.float().to(dev),
                            None if t is None else t.float().to(dev), c_pad=cpad, dtype=dt[0])
            assert y.shape == (2, h, w, cpad)
            what = f"{h}x{w} {mode}"
            assert_equal(nchw64(y)[:, :c], r16(ref, dt[1]), what)
            assert not y[..., c:].view(torch.int16).any(), f"{what}: padding channels are not +0.0"
        v = torch.randn(2, h, w, cpad, generator=g).to(dt[1]).to(dev)
        f = N.to_nchw32(v, dtype=dt[0])
        assert_equal(f.cpu().double(), v.cpu().double().permute(0, 3, 1, 2), f"{h}x{w} nhwc16_to_nchw")
        back = N.to_nhwc16(f, dtype=dt[0])
        assert torch.equal(back.view(torch.int16), v.view(torch.int16)), f"{h}x{w}: round trip is not the identity"


# ------------------------------------------------------------------------------------------------ split channel reduction
def expected_splits(sms, b, hw, c):
    """channel_reduce_splits: about 4 CTAs per SM, at least 64 pixels per split, at most 64 splits."""
    ctas = b * -(-c // 64)
    s = -(-4 * sms // ctas)
    s = min(s, max(1, hw // 64))
    return max(1, min(s, 64))


# (name, B, H, W, C, Cr / Cout): the name states S on the 132 SMs of an H100 SXM; the test checks the class on any count
REDUCE = [
    ("s1_c520", 4, 8, 8, 520, 13),
    ("s1_c8_hw35", 3, 5, 7, 8, 3),
    ("mid_c72", 2, 32, 32, 72, 5),
    ("mid_c520_hw561", 1, 33, 17, 520, 13),
    ("cap64_c8", 1, 64, 64, 8, 3),
    ("cap64_c72", 2, 64, 128, 72, 5),
    ("cap64_c8_hw4355_tail", 1, 67, 65, 8, 3),
]


def mean_error(m, hw):
    """fp32 sum * (1/HW): the sum of integers is exact; 1/HW and the product round once each unless HW is 2^k."""
    return torch.zeros_like(m) if hw & (hw - 1) == 0 else 3 * EPS * m.abs()


def matvec(w, v, ev, depth):
    """v @ w.T in float64, and the bound of its fp32 evaluation from inputs v (error ev): the propagated input error
    plus one roundoff of sum|terms| per partial-sum level (depth = the longest chain of fp32 additions)."""
    return v @ w.T, ev @ w.abs().T + depth * EPS * (v.abs() @ w.abs().T)


def sigmoid_error(t, et):
    """1 / (1 + __expf(-t)): __expf is within 2 + 1.173|t| ulps (2^-23 each), then one rounding each for 1 + e and
    the IEEE division; sigmoid' <= 1/4 carries the error of t."""
    s = torch.sigmoid(t)
    return et / 4 + (8 + 3 * t.abs()) * EPS * s


@pytest.mark.parametrize("name,b,h,w,c,cr", REDUCE, ids=[r[0] for r in REDUCE])
def test_channel_reduction_mean_se_gate_pooled_fc(N, dev, sms, dt, name, b, h, w, c, cr):
    from hairfastgan_b200 import _lib
    hw = h * w
    s = expected_splits(sms, b, hw, c)
    assert _lib.lib().hf_channel_reduce_workspace_bytes(b, hw, c) == b * s * c * 4
    if name.startswith("s1"):
        assert s == 1
    elif name.startswith("mid"):
        assert 1 < s < 64
    else:
        assert s == 64
    g = torch.Generator().manual_seed(hw + c)
    base = ints(g, (b, c, 1, 1), -3, 3)
    x = base + ints(g, (b, c, h, w), -2, 2)                 # per-channel offsets: the means are spread out
    x16 = to16(x, dt[1], dev)
    m = x.sum((2, 3)) / hw
    em = mean_error(m, hw)
    got = N.channel_mean(x16, dtype=dt[0]).cpu().double()
    if hw & (hw - 1) == 0:
        assert_equal(got, m.float().double(), "channel mean")          # exact sum, exact 1/HW
    else:
        assert_within(got, m, em, "channel mean")
    depth = c // 32 + 6                                       # per-lane fmaf chain + 5 shuffle levels
    # SE gate: sigmoid(W2 . relu(W1 . mean)), Cr not a multiple of 8
    w1 = pick(g, (cr, c), [-0.5, -0.25, 0.0, 0.25, 0.5])
    w2 = pick(g, (c, cr), [-1.0, -0.5, 0.0, 0.5, 1.0])
    hid, eh = matvec(w1, m, em, depth)
    hid = hid.clamp_min(0)                                    # relu is 1-Lipschitz: eh still bounds its error
    t, et = matvec(w2, hid, eh, cr + 1)
    got = N.se_gate(x16, w1.float().to(dev), w2.float().to(dev), dtype=dt[0]).cpu().double()
    assert_within(got, torch.sigmoid(t), sigmoid_error(t, et), "se_gate")
    # pooled 1x1 conv: act(W . mean * scale + shift), Cout not a multiple of 8, scale / shift each null or set
    wf = pick(g, (cr, c), [-1.0, -0.5, 0.0, 0.5, 1.0])
    scale = pick(g, (cr,), [0.5, 1.0, 2.0])
    shift = ints(g, (cr,), -8, 8) / 4
    t, et = matvec(wf, m, em, depth)
    for sc in (None, scale):
        for shf in (None, shift):
            v = t * (1.0 if sc is None else sc) + (0.0 if shf is None else shf)
            ev = et * (1.0 if sc is None else sc) + EPS * v.abs()          # fmaf: one rounding
            for act in (0, 1, 2):
                got = N.pooled_fc(x16, wf.float().to(dev), None if sc is None else sc.float().to(dev),
                                  None if shf is None else shf.float().to(dev), act=act, dtype=dt[0]).cpu().double()
                what = f"pooled_fc act {act} scale {sc is not None} shift {shf is not None}"
                if act == 2:
                    assert_within(got, torch.sigmoid(v), sigmoid_error(v, ev), what)
                else:
                    assert_within(got, v.clamp_min(0) if act == 1 else v, ev, what)


# ------------------------------------------------------------------------------------------------ instance norm
@pytest.mark.parametrize("b,h,w,c", [(3, 8, 8, 8), (2, 4, 16, 72), (4, 1, 1, 72), (2, 1, 1, 8)],
                         ids=["c8_hw64", "c72_hw64", "c72_hw1_zero_var", "c8_hw1_zero_var"])
def test_instance_norm_lrelu_bounded(N, dev, dt, b, h, w, c):
    """(x - mean) * rsqrtf(var + 1e-5), LeakyReLU.  HW is a power of two, so the mean and every x - mean are
    exact; the variance sum rounds (k <= HW + 64 levels, all terms positive, so relative to var), var + eps and
    rsqrtf (2 ulps) round, then the product and the slope: 8 + var_levels / 2 roundoffs of |y|, plus 1 ulp of the
    16-bit store.  HW = 1 has zero variance: the output is exactly 0.  Every sample has its own statistics."""
    g = torch.Generator().manual_seed(b * c + h)
    x = ints(g, (b, c, 1, 1), -20, 20) + ints(g, (b, 1, 1, 1), 1, 3) * ints(g, (b, c, h, w), -6, 6)
    x16 = to16(x, dt[1], dev)
    hw = h * w
    m = x.mean((2, 3), keepdim=True)
    var = (x - m).pow(2).mean((2, 3), keepdim=True)
    eps32 = float(torch.tensor(1e-5, dtype=torch.float32))
    t = (x - m) / torch.sqrt(var + eps32)
    for slope in (0.0, 0.2, 1.0):
        s32 = float(torch.tensor(slope, dtype=torch.float32))
        ref = torch.where(t > 0, t, t * s32)
        got = nchw64(N.instance_norm_lrelu(x16, slope=slope, dtype=dt[0]))
        if hw == 1:
            assert_equal(got, torch.zeros_like(ref), f"slope {slope}: zero variance")
            continue
        assert_within(got, ref, ulp16(ref, dt[1]) + (8 + (hw + 64) / 2) * EPS * ref.abs(), f"slope {slope}")


# ------------------------------------------------------------------------------------------------ reflection padding
@pytest.mark.parametrize("b,h,w,c", [(2, 2, 2, 8), (1, 3, 5, 16), (2, 6, 2, 8)], ids=["h2_w2", "h3_w5", "h6_w2"])
def test_reflect_pad1_bit_exact(N, dev, dt, b, h, w, c):
    x = ints(torch.Generator().manual_seed(h * w), (b, c, h, w), -100, 100)
    got = nchw64(N.reflect_pad1(to16(x, dt[1], dev), dtype=dt[0]))
    assert_equal(got, F.pad(x, (1, 1, 1, 1), mode="reflect"), "reflect_pad1")


# ------------------------------------------------------------------------------------------------ SE scale + shortcut add
SCALE_ADD = [(c, s) for c in (16, 72, 2, 6, 10) for s in (1, 2)]


@pytest.mark.parametrize("c,stride", SCALE_ADD,
                         ids=[f"{'vec8' if c % 8 == 0 else 'scalar'}_c{c}_stride{s}" for c, s in SCALE_ADD])
def test_scale_add_bit_exact(N, dev, dt, c, stride):
    """out = res * se[b,c] + shortcut[b, y*s, x*s, c]; y16 = out, y16b = out * s2[c] + b2[c] (fmaf), every operand
    null or set, either output alone or both."""
    b, h, w = 2, 3, 5
    g = torch.Generator().manual_seed(c * 10 + stride)
    res = ints(g, (b, c, h, w), -8, 8)
    se = pick(g, (b, c), [-1.0, 0.25, 0.5, 1.0, 2.0])
    sc = ints(g, (b, c, h * stride, w * stride), -8, 8)
    s2 = pick(g, (c,), [-1.0, 0.5, 1.0, 2.0])
    b2 = ints(g, (c,), -8, 8) / 2
    res16, sc16 = to16(res, dt[1], dev), to16(sc, dt[1], dev)
    col = lambda v: v.view(1, c, 1, 1)
    for use_se in (False, True):
        for use_sc in (False, True):
            out = res * (se.view(b, c, 1, 1) if use_se else 1.0) + (sc[:, :, ::stride, ::stride] if use_sc else 0.0)
            kw = dict(se=se.float().to(dev) if use_se else None, shortcut16=sc16 if use_sc else None,
                      shortcut_stride=stride, dtype=dt[0])
            what = f"se {use_se} shortcut {use_sc}"
            y, yb = N.scale_add(res16, **kw)
            assert yb is None
            assert_equal(nchw64(y), r16(out, dt[1]), what + " y16 only")
            for a, d in ((None, None), (s2, None), (None, b2), (s2, b2)):
                ref_b = out * (1.0 if a is None else col(a)) + (0.0 if d is None else col(d))
                aff = (None if a is None else a.float().to(dev), None if d is None else d.float().to(dev))
                for want_y16 in (False, True):
                    y, yb = N.scale_add(res16, y16b_affine=aff, want_y16=want_y16, **kw)
                    w_ = f"{what} s2 {a is not None} b2 {d is not None} y16 {want_y16}"
                    assert_equal(nchw64(yb), r16(ref_b, dt[1]), w_ + " y16b")
                    if want_y16:
                        assert_equal(nchw64(y), r16(out, dt[1]), w_ + " y16")
                    else:
                        assert y is None


# ------------------------------------------------------------------------------------------------ FPN upsample + add
# (name, h, w, H, W, C, dyadic): align_corners ratios (h-1)/(H-1) and (w-1)/(W-1)
UPSAMPLE_ADD = [
    ("vec8_dyadic_5to9_5to17", 5, 5, 9, 17, 16, True),
    ("scalar_dyadic_5to9_5to17", 5, 5, 9, 17, 6, True),
    ("vec8_same_size", 6, 7, 6, 7, 8, True),
    ("scalar_same_size", 6, 7, 6, 7, 2, True),
    ("vec8_h1_ry0", 1, 5, 4, 9, 16, True),
    ("scalar_H1_ry0", 3, 5, 1, 9, 10, True),
    ("vec8_nondyadic_7to16", 7, 7, 16, 16, 8, False),
    ("vec8_nondyadic_13to32_7to16", 13, 7, 32, 16, 72, False),
    ("scalar_nondyadic_13to32_7to16", 13, 7, 32, 16, 6, False),
]


@pytest.mark.parametrize("name,h,w,H,W,c,dyadic", UPSAMPLE_ADD, ids=[u[0] for u in UPSAMPLE_ADD])
def test_upsample_add(N, dev, dt, name, h, w, H, W, c, dyadic):
    """bilinear(x, (H, W), align_corners=True) + y.  Dyadic ratios: exact weights, bit-exact.  Otherwise the fp32
    ratio and source coordinate round (|d fy| <= 2^-23 (h-1), the value moves by at most 2 max|x| per unit of fy),
    and the blend rounds eight times: 1 ulp + 2^-24 (4 max|x| (h + w) + 8 (max|x| + |y|))."""
    b = 2
    g = torch.Generator().manual_seed(h * 100 + W + c)
    x = ints(g, (b, c, h, w), -8, 8)
    y = ints(g, (b, c, H, W), -8, 8)
    got = nchw64(N.upsample_add(to16(x, dt[1], dev), to16(y, dt[1], dev), dtype=dt[0]))
    ref = F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True) + y
    if dyadic:
        assert_equal(got, r16(ref, dt[1]), name)
    else:
        mx = x.abs().amax()
        bound = ulp16(ref, dt[1]) + EPS * (4 * mx * (h + w) + 8 * (mx + y.abs()))
        assert_within(got, ref, bound, name)


# ------------------------------------------------------------------------------------------------ adaptive average pooling
# (name, B, H, W, C, oh, ow)
AVGPOOL = [
    ("vec8_overlap_7to3_10to4", 2, 7, 10, 16, 3, 4),
    ("vec8_up_2to3_5to2", 2, 2, 5, 8, 3, 2),
    ("vec8_c72_16x12_to_3x3", 2, 16, 12, 72, 3, 3),
    ("scalar_c6_overlap_7to3_10to4", 2, 7, 10, 6, 3, 4),
    ("scalar_c10_up_2to3_3to5", 1, 2, 3, 10, 3, 5),
    ("scalar_c8_bins_over_65535", 1, 5, 7, 8, 257, 256),
]


@pytest.mark.parametrize("name,b,h,w,c,oh,ow", AVGPOOL, ids=[a[0] for a in AVGPOOL])
def test_adaptive_avgpool_bit_exact(N, dev, dt, name, b, h, w, c, oh, ow):
    """The window sum of integers is exact and the division by its size is IEEE, so the fp32 output is the correctly
    rounded mean; float64 cannot round it twice (a quotient by n < 2^28 never lies within 2^-53 of an fp32 tie)."""
    assert ("scalar" in name) == (c % 8 != 0 or oh * ow > 65535)
    x = ints(torch.Generator().manual_seed(h * w + c + oh), (b, c, h, w), -50, 50)
    got = N.adaptive_avgpool(to16(x, dt[1], dev), oh, ow, dtype=dt[0]).cpu().double()
    assert_equal(got, F.adaptive_avg_pool2d(x, (oh, ow)).float().double(), name)


# ------------------------------------------------------------------------------------------------ BiSeNet max pooling
@pytest.mark.parametrize("c", [8, 72], ids=["c8", "c72"])
@pytest.mark.parametrize("h", [1, 2, 3, 7, 64, 65], ids=lambda v: f"h{v}")
def test_maxpool3x3s2_bit_exact(N, dev, dt, h, c):
    g = torch.Generator().manual_seed(h * 7 + c)
    for w in (1, 2, 3, 7, 64, 65):
        x = ints(g, (2, c, h, w), -100, 100)
        got = nchw64(N.maxpool3x3s2(to16(x, dt[1], dev), dtype=dt[0]))
        assert_equal(got, F.max_pool2d(x, 3, 2, 1), f"{h}x{w}")


def test_maxpool3x3s2_extremes_neg_inf_and_lowest(N, dev, dt):
    """A plane of -inf, a plane of the lowest finite value of the type (bf16: -3.39e38, below any finite fp32 seed
    such as -3.0e38) and a plane mixing both come out unchanged: the padding is skipped, never compared."""
    g = torch.Generator().manual_seed(9)
    x = ints(g, (2, 16, 7, 6), -100, 100)
    lowest = float(torch.finfo(dt[1]).min)
    x[:, 0] = float("-inf")
    x[:, 1] = lowest
    x[:, 2] = torch.where(ints(g, (2, 7, 6), 0, 1) > 0, lowest, float("-inf"))
    got = nchw64(N.maxpool3x3s2(to16(x, dt[1], dev), dtype=dt[0]))
    ref = F.max_pool2d(x, 3, 2, 1)
    assert (ref[:, 1] == lowest).all() and (ref[:, 0] == float("-inf")).all()
    assert_equal(got, ref, "maxpool extremes")


# ------------------------------------------------------------------------------------------------ gated add + nearest upsample
@pytest.mark.parametrize("up", [1, 2], ids=["up1", "up2"])
@pytest.mark.parametrize("b,h,w,c", [(2, 3, 5, 16), (3, 1, 1, 72)], ids=["h3_w5", "h1_w1"])
def test_gate_add_up_bit_exact(N, dev, dt, b, h, w, c, up):
    """nearest_up(x * gate[b,c] + addvec[b,c] + addt): every operand null or set; all null with up = 2 is the plain
    nearest 2x upsample of SEAN and the shape adaptor."""
    g = torch.Generator().manual_seed(h * c + up)
    x = ints(g, (b, c, h, w), -8, 8)
    gate = pick(g, (b, c), [-1.0, 0.25, 0.5, 1.0, 2.0])
    addv = ints(g, (b, c), -8, 8) / 2
    addt = ints(g, (b, c, h, w), -8, 8)
    x16, t16 = to16(x, dt[1], dev), to16(addt, dt[1], dev)
    for ug in (False, True):
        for ua in (False, True):
            for ut in (False, True):
                v = x * (gate.view(b, c, 1, 1) if ug else 1.0) + (addv.view(b, c, 1, 1) if ua else 0.0)
                v = v + (addt if ut else 0.0)
                ref = v.repeat_interleave(up, 2).repeat_interleave(up, 3)
                got = nchw64(N.gate_add_up(x16, gate=gate.float().to(dev) if ug else None,
                                           addvec=addv.float().to(dev) if ua else None, addt16=t16 if ut else None,
                                           up=up, dtype=dt[0]))
                assert_equal(got, r16(ref, dt[1]), f"gate {ug} addvec {ua} addt {ut}")


# ------------------------------------------------------------------------------------------------ fused RGB stems
def exact_bn(g, dev):
    """Eval BatchNorm with eps = 0, running_var = 1 and a dyadic weight: the folded scale is the weight itself and
    the shift an integer."""
    bn = torch.nn.BatchNorm2d(64, eps=0.0).eval()
    bn.weight.data = pick(g, (64,), [-1.0, 0.5, 1.0, 2.0]).float()
    bn.bias.data = ints(g, (64,), -16, 16).float()
    bn.running_mean.copy_(ints(g, (64,), -4, 4).float())
    bn.running_var.fill_(1.0)
    scale = bn.weight.data.double()
    shift = bn.bias.data.double() - bn.running_mean.double() * scale
    return bn.to(dev), scale, shift


STEM_SIZES = [(1, 1, 1), (1, 7, 7), (2, 15, 33), (2, 17, 65), (3, 9, 12), (3, 12, 9)]
STEM_IDS = ["1x1", "7x7", "15x33", "17x65", "odd9x12", "12xodd9"]


@pytest.mark.parametrize("b,h,w", STEM_SIZES + [(None, 17, 65)], ids=STEM_IDS + ["17x65_tiles_over_2x_sms"])
def test_stem7x7s2_bit_exact(N, dev, sms, dt, b, h, w):
    """Conv 7x7 / 2 / pad 3 + BatchNorm + ReLU on integer images and integer weights: the 147-tap accumulator is an
    integer below 2^11, so a dropped or misplaced tap, channel or padding column changes the output."""
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    per_image = -(-wo // 32) * -(-ho // 8)
    if b is None:                                   # more 8x32 tiles than the persistent grid of 2 CTAs per SM
        b = -(-2 * sms // per_image) + 3
        assert b * per_image > 2 * sms
    g = torch.Generator().manual_seed(h * w + b)
    x = ints(g, (b, 3, h, w), -3, 3)
    wt = ints(g, (64, 3, 7, 7), -2, 2)
    bn, scale, shift = exact_bn(g, dev)
    stem = N.PackedStem7x7(wt.float().to(dev), bn, dtype=dt[0])
    got = nchw64(stem(x.float().to(dev)))
    ref = F.relu(F.conv2d(x, wt * scale.view(-1, 1, 1, 1), None, 2, 3) + shift.view(1, -1, 1, 1))
    assert_equal(got, r16(ref, dt[1]), f"stem7x7s2 B={b} {h}x{w}")


@pytest.mark.parametrize("b,h,w", STEM_SIZES + [(None, 17, 65)], ids=STEM_IDS + ["17x65_tiles_over_2x_sms"])
def test_stem3x3_bit_exact(N, dev, sms, dt, b, h, w):
    """Conv 3x3 / 1 / pad 1 + BatchNorm + PReLU (dyadic slopes), and the second output y16b = y * s2 + b2 (dyadic),
    computed from the fp32 value, not from the rounded y16."""
    per_image = -(-w // 32) * -(-h // 8)
    if b is None:
        b = -(-2 * sms // per_image) + 2
        assert b * per_image > 2 * sms
    g = torch.Generator().manual_seed(h * w + b + 1)
    x = ints(g, (b, 3, h, w), -3, 3)
    wt = ints(g, (64, 3, 3, 3), -2, 2)
    bn, scale, shift = exact_bn(g, dev)
    slope = pick(g, (64,), [0.0, 0.25, 0.5, 1.0, -0.5])
    s2 = pick(g, (64,), [-1.0, 0.5, 1.0, 2.0])
    b2 = ints(g, (64,), -8, 8) / 2
    stem = N.PackedStem3x3(wt.float().to(dev), bn, slope.float().to(dev), dtype=dt[0])
    t = F.conv2d(x, wt * scale.view(-1, 1, 1, 1), None, 1, 1) + shift.view(1, -1, 1, 1)
    t = torch.where(t > 0, t, t * slope.view(1, -1, 1, 1))
    tb = t * s2.view(1, -1, 1, 1) + b2.view(1, -1, 1, 1)
    y, yb = stem(x.float().to(dev))
    assert yb is None
    assert_equal(nchw64(y), r16(t, dt[1]), "y16 alone")
    y, yb = stem(x.float().to(dev), y16b_affine=(s2.float().to(dev), b2.float().to(dev)))
    assert_equal(nchw64(y), r16(t, dt[1]), "y16")
    assert_equal(nchw64(yb), r16(tb, dt[1]), "y16b")


# ------------------------------------------------------------------------------------------------ bilinear logit upsampling
def bilinear_into(y, x, c, H, W):
    from hairfastgan_b200 import _lib
    b, cin, h, w = x.shape
    _lib.check(_lib.lib().hf_bilinear_upsample_nchw_f32(x.data_ptr(), y.data_ptr(), b, c, cin, h, w, H, W,
                                                        _lib.stream_ptr()), "hf_bilinear_upsample_nchw_f32")
    return y


def unaligned_out(shape, dev):
    """An output tensor 4 bytes into a buffer of numel + 1 floats: never 16-byte aligned, so the scalar kernel runs."""
    n = 1
    for s in shape:
        n *= s
    return torch.empty(n + 1, device=dev)[1:].view(shape)


# (name, B, Cin, C, h, w, H, W, dyadic).  Row kernel: W % 4 == 0, y 16-byte aligned and w <= 8192; else scalar.
BILINEAR = [
    ("row_dyadic_rows_5to9_cols_12to12", 2, 32, 19, 5, 12, 9, 12, True),
    ("row_dyadic_down_9to3_13to4", 2, 8, 8, 9, 13, 3, 4, True),
    ("scalar_wtail_dyadic_5to9_9to33", 2, 32, 19, 5, 9, 9, 33, True),
    ("scalar_w_over_8192_dyadic", 1, 2, 2, 3, 8196, 5, 8196, True),
    ("row_H1", 1, 4, 3, 6, 15, 1, 8, True),
    ("scalar_W1", 1, 4, 3, 6, 7, 5, 1, True),
    ("row_src_1x1", 2, 3, 3, 1, 1, 4, 8, True),
    ("row_nondyadic_8x12_to_64x96", 2, 32, 19, 8, 12, 64, 96, False),
    ("scalar_wtail_nondyadic_7x10_to_30x45", 1, 19, 19, 7, 10, 30, 45, False),
]


@pytest.mark.parametrize("name,b,cin,c,h,w,H,W,dyadic", BILINEAR, ids=[v[0] for v in BILINEAR])
def test_bilinear_upsample_nchw(dev, name, b, cin, c, h, w, H, W, dyadic):
    """The first C of Cin planes, align_corners=True.  The row kernel and the scalar kernel (forced by an unaligned
    output view) are bit-equal on random data.  Dyadic ratios on integer data are bit-exact against float64; other
    ratios are within 2^-24 max|x| (4 (h + w) + 8): the rounded fp32 coordinate (|d fy| <= 2^-23 (h-1), slope
    <= 2 max|x|) and the six roundings of the three lerps."""
    assert name.startswith("row") == (W % 4 == 0 and w <= 8192)
    g = torch.Generator().manual_seed(h * w + H + W)
    xr = torch.randn(b, cin, h, w, generator=g).to(dev)
    y_dispatch = bilinear_into(torch.empty(b, c, H, W, device=dev), xr, c, H, W)
    y_scalar = bilinear_into(unaligned_out((b, c, H, W), dev), xr, c, H, W)
    assert torch.equal(y_dispatch, y_scalar), "row and scalar kernels differ"
    x = ints(g, (b, cin, h, w), -8, 8)
    got = bilinear_into(torch.empty(b, c, H, W, device=dev), x.float().to(dev), c, H, W).cpu().double()
    ref = F.interpolate(x[:, :c], size=(H, W), mode="bilinear", align_corners=True)
    if dyadic:
        assert_equal(got, ref.float().double(), name)
    else:
        assert_within(got, ref, EPS * x.abs().amax() * (4 * (h + w) + 8) + torch.zeros_like(ref), name)


# (name, B, Cin, C, h, w, H, W): shared memory C * w * 4 bytes, opt-in above 48 KB
ARGMAX = [
    ("smem_static_19x12", 2, 32, 19, 8, 12, 64, 96),
    ("smem_over_48k_19x700", 1, 19, 19, 3, 700, 5, 1400),
]


@pytest.mark.parametrize("name,b,cin,c,h,w,H,W", ARGMAX, ids=[a[0] for a in ARGMAX])
def test_bilinear_argmax_matches_upsampled_logits(N, dev, name, b, cin, c, h, w, H, W):
    """labels == argmax(dim=1) of the kernel's own upsampled logits, on random logits and on integer logits with
    duplicated planes (exact ties, which take the first index like torch.argmax)."""
    assert (c * w * 4 > 48 * 1024) == ("over_48k" in name)
    g = torch.Generator().manual_seed(w + c)
    for kind in ("random", "ties"):
        if kind == "random":
            x = torch.randn(b, cin, h, w, generator=g)
        else:
            x = ints(g, (b, cin, h, w), -2, 2).float()
            x[:, 3] = ints(g, (b, h, w), -2, 4).float()          # often the maximum, always tied with plane 7
            x[:, 7] = x[:, 3]
            x[:, c - 1] = x[:, 0]
        logits = N.bilinear_upsample_nchw(x.to(dev), c, H, W).cpu()
        labels = N.bilinear_argmax_nchw(x.to(dev), c, H, W).cpu()
        ref = logits.argmax(dim=1)
        if kind == "ties":
            top = logits.amax(dim=1, keepdim=True)
            assert ((logits == top).sum(1) > 1).float().mean() > 0.05, "the tie data has too few ties"
        assert_equal(labels, ref, f"{name} {kind}")


def test_bilinear_argmax_rejects_over_200k_smem_without_launch(dev):
    """19 classes x 2700 source columns need 205 KB of shared memory: an error, and the labels stay untouched."""
    from hairfastgan_b200 import _lib
    b, c, h, w, H, W = 1, 19, 2, 2700, 3, 16
    x = torch.zeros(b, c, h, w, device=dev)
    labels = torch.full((b, H, W), -7, dtype=torch.int64, device=dev)
    rc = _lib.lib().hf_bilinear_argmax_nchw_f32(x.data_ptr(), labels.data_ptr(), b, c, c, h, w, H, W,
                                                _lib.stream_ptr())
    assert rc != 0 and b"do not fit in shared memory" in _lib.lib().hf_last_error()
    torch.cuda.synchronize()
    assert (labels == -7).all()

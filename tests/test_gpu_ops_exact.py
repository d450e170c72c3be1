"""Exact-arithmetic tests of the StyleGAN2 operator boundary (csrc/hf_ops.cu: hf_upfirdn2d_f32, hf_bias_act_f32) and of
the stage glue (csrc/hf_glue_ops.cu: BicubicDownSample, DilateErosion, the Alignment mask algebra and the F-space blend
chain), called through the C ABI.

Operands are small integers and dyadic values (multiples of a power of two), so every fp32 intermediate of these
kernels is exact.  The references are float64 torch on the CPU (tests/ops_exact_cases.py), rounded once to fp32 after
asserting that the float64 value is exact in fp32; the kernel output must then equal them bit for bit, so a flipped,
transposed or shifted tap, a wrong pad, a leaked plane or a stale pipeline stage changes an integer that no tolerance
absorbs.  bias_act is one IEEE add and two multiplies per element, so a float32 CPU restatement is bit-exact on any
values, signed zeros, infinities and NaN included.  Where a kernel rounds in a way exact inputs cannot avoid, the test
states a bound beside the operation.

Each case id starts with the dispatch path it takes, from the Python restatement of its entry point's host condition
in tests/ops_exact_cases.py; tests/test_ops_exact_cases_cpu.py checks without a device that the tables reach every
path.  All kernels here are fp32, so the module runs once, not once per 16-bit operand type."""
import pytest
import torch
import torch.nn.functional as F

from tests import ops_exact_cases as T

pytestmark = pytest.mark.gpu
HF_DTYPES = ["default"]
torch.set_grad_enabled(False)

EPS = 2.0 ** -24                        # unit roundoff of fp32


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hairfastgan_b200 import _lib
    _lib.use_device(0)
    return _lib


@pytest.fixture(scope="module")
def sms(L):
    n = L.lib().hf_sm_count()
    assert n > 0
    return n


# ------------------------------------------------------------------------------------------------ operands, checks
def ints(g, shape, lo, hi):
    """Seeded integers in [lo, hi] as float64."""
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def pick(g, shape, values):
    """Seeded draws from a list of (dyadic) values as float64."""
    v = torch.tensor(values, dtype=torch.float64)
    return v[torch.randint(0, len(values), shape, generator=g)]


def exact32(ref, what="reference"):
    """float64 -> fp32, asserting there is nothing to round (so the comparison below is bit for bit)."""
    f = ref.float()
    assert torch.equal(f.double(), ref), f"{what} not exact in fp32: the bit-exact comparison would be invalid"
    return f


def assert_equal(got, ref, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    bad = (got != ref) & ~(torch.isnan(got) & torch.isnan(ref))
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail(f"{what}: {int(bad.sum())} of {ref.numel()} values differ; first at {i}: got {float(got[i])!r}, "
                    f"expected {float(ref[i])!r}")


def assert_bits(got, ref, what):
    """fp32 bit patterns equal (so the sign of zero counts); any NaN matches any NaN."""
    assert got.dtype == ref.dtype == torch.float32 and got.shape == ref.shape, what
    bad = (got.view(torch.int32) != ref.view(torch.int32)) & ~(torch.isnan(got) & torch.isnan(ref))
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail(f"{what}: {int(bad.sum())} of {ref.numel()} values differ in their bits; first at {i}: got "
                    f"{float(got[i])!r}, expected {float(ref[i])!r}")


def assert_within(got, ref, bound, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    over = (got - ref).abs() > bound
    if over.any():
        i = tuple(int(v) for v in over.nonzero()[0])
        pytest.fail(f"{what}: {int(over.sum())} of {ref.numel()} values out of bound; first at {i}: got "
                    f"{float(got[i])!r}, expected {float(ref[i])!r}, bound {float(bound[i]):.3g}")


def at_offset(t, off, dev):
    """A contiguous device copy of t that starts `off` bytes into a fresh allocation (the caching allocator hands
    out 512-byte aligned blocks, so its alignment is exactly that of `off`)."""
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=dev)
    v = buf[off // t.element_size():off // t.element_size() + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == off % 16
    return v


def nan_like(shape, off, dev):
    return at_offset(torch.full(shape, float("nan")), off, dev)


# ------------------------------------------------------------------------------------------------ upfirdn2d
def up_operands(u):
    g = torch.Generator().manual_seed(T.seed(u.name))
    x = ints(g, (u.planes, u.in_h, u.in_w), -8, 8)
    if u.impulses:                       # plane 0: impulses at the corners and inside pin the taps' orientation
        x[0] = 0
        for (i, j), v in zip(((0, 0), (0, u.in_w - 1), (u.in_h - 1, 0), (u.in_h - 1, u.in_w - 1),
                              (u.in_h // 2, u.in_w // 3)), (1, -2, 3, -4, 5)):
            x[0, i, j] = v
    return x, T.upfirdn_taps(u)


def run_upfirdn(L, x, k, u, x_off, y_off, dev):
    xd = at_offset(x.float(), x_off, dev)
    kd = k.float().to(dev)
    out_h, out_w = T.upfirdn_out(u)
    y = nan_like((u.planes, out_h, out_w), y_off, dev)
    L.check(L.lib().hf_upfirdn2d_f32(xd.data_ptr(), y.data_ptr(), kd.data_ptr(), u.planes, u.in_h, u.in_w, u.kh, u.kw,
                                     u.up_x, u.up_y, u.down_x, u.down_y, u.px0, u.px1, u.py0, u.py1, L.stream_ptr()),
            "hf_upfirdn2d_f32")
    return y.cpu()


def up_ref(x, k, u):
    return T.upfirdn_ref(x, k, u.up_x, u.up_y, u.down_x, u.down_y, u.px0, u.px1, u.py0, u.py1)


def check_upfirdn_exact(L, u, dev):
    """The dispatched kernel and, for a bulk case, the general kernel on a 4-byte-offset copy of the same input: both
    equal the float64 reference bit for bit (and so each other)."""
    x, k = up_operands(u)
    path = T.upfirdn_path(u)
    ref = exact32(up_ref(x, k, u))
    assert_equal(run_upfirdn(L, x, k, u, u.x_off, u.y_off, dev), ref, f"{path} {u}")
    if path != "general":
        moved = u._replace(x_off=4)
        assert T.upfirdn_path(moved) == "general"
        assert_equal(run_upfirdn(L, x, k, moved, 4, u.y_off, dev), ref, f"general on the offset copy of {u}")


@pytest.mark.parametrize("u", T.UPFIRDN_EXACT, ids=T.upfirdn_id)
def test_upfirdn2d_bit_exact(L, u):
    check_upfirdn_exact(L, u, torch.device("cuda", 0))


@pytest.mark.parametrize("down,fir", [(d, f) for d in (1, 2) for f in ("sep", "gen")],
                         ids=[f"bulk_d{d}_nc2_{f}-pads_0to3_each_side" for d in (1, 2) for f in ("sep", "gen")])
def test_upfirdn2d_every_pad_each_side(L, down, fir):
    """All 256 (px0, px1, py0, py1) in 0..3, x and y pads independent (the Python wrapper ties them), through the
    C ABI: the padding columns go through the edge fix-up, padding rows are never fetched."""
    dev = torch.device("cuda", 0)
    for px0 in range(4):
        for px1 in range(4):
            for py0 in range(4):
                for py1 in range(4):
                    u = T.Up(f"pads_{down}_{px0}{px1}{py0}{py1}", 4, 10, 67, down_x=down, down_y=down, px0=px0,
                             px1=px1, py0=py0, py1=py1, fir=fir)
                    assert T.upfirdn_path(u) == f"bulk_d{down}_nc2_{fir}"
                    check_upfirdn_exact(L, u, dev)


@pytest.mark.parametrize("u", T.UPFIRDN_BOUNDED, ids=T.upfirdn_id)
def test_upfirdn2d_separable_loop_bounded(L, u):
    """Two FIRs the separable loop runs although it cannot be exact.

    sep3: u[3] = 3, so ky[a] = u[3-a] / 3 rounds (relative 2^-24).  Per output the loop adds four products h * ky[a]
    (h exact: x and row 0 of the taps are exact) with FFMAs: one rounding of ky plus four of the running sum, each at
    most 2^-24 of sum |x k| -- bound 5 * 2^-24 * sum |x| |k|.  The general kernel on the offset copy is exact.

    near: one tap is 2^-21 (4.8e-7) relative off the rank-1 product of row 0 and column 0, inside the kernel's 1e-6
    separability test.  The separable loop then computes the rank-1 kernel exactly (asserted bit for bit), which is
    within 2^-21 |x k| <= 1e-6 * sum |x| |k| of the true FIR (DESIGN.md section 4.2).  The general kernel computes the
    true FIR; with the perturbed tap its products round (16 FFMAs): bound 16 * 2^-24 * sum |x| |k|."""
    dev = torch.device("cuda", 0)
    x, k = up_operands(u)
    ref = up_ref(x, k, u)
    absref = up_ref(x.abs(), k.abs(), u)
    bulk = run_upfirdn(L, x, k, u, 0, 0, dev).double()
    general = run_upfirdn(L, x, k, u._replace(x_off=4), 4, 0, dev).double()
    if u.fir == "sep3":
        assert_within(bulk, ref, 5 * EPS * absref, f"separable loop, {u.name}")
        assert_equal(general, exact32(ref).double(), f"general kernel, {u.name}")
    else:
        assert_equal(bulk, exact32(up_ref(x, T.rank1_part(k), u)).double(), f"separable loop = rank-1 FIR, {u.name}")
        assert_within(bulk, ref, 1e-6 * absref, f"separable loop vs the true FIR, {u.name}")
        assert_within(general, ref, 16 * EPS * absref, f"general kernel, {u.name}")


# ------------------------------------------------------------------------------------------------ bias_act
SPECIALS = [0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-45, -1e-45, 3.4e38]


def bias_act_operands(c):
    n, size_b, step_b = T.bias_act_dims(c)
    g = torch.Generator().manual_seed(T.seed(c.name))
    x = (torch.randn(n, generator=g) * 4).float()
    b = (torch.randn(max(size_b, 1), generator=g) * 2).float()[:size_b]
    if size_b:
        b[0] = -0.0
        if size_b > 2:
            b[1] = 0.0
    sp = torch.tensor(SPECIALS * 4, dtype=torch.float32)
    pos = torch.randperm(n, generator=g)[:min(n, sp.numel())]
    x[pos] = sp[:pos.numel()]
    if size_b:                       # exact cancellations x = -b: +0 after the add
        rows = torch.randperm(n, generator=g)[:min(n, 16)]
        x[rows] = -b[(rows // step_b) % size_b]
    return x.view(c.shape), b


def bias_act_ref(x, b, c):
    """The reference's fused_bias_act_kernel.cu:25-46 in float32: x + b (when there is a bias), leaky relu as
    (t > 0) ? t : t * alpha, then * scale -- one IEEE operation each."""
    n, size_b, step_b = T.bias_act_dims(c)
    t = x.reshape(-1, step_b)
    if size_b:
        t = t + b[torch.arange(t.shape[0]) % size_b].view(-1, 1)
    alpha, scale = torch.tensor(c.alpha, dtype=torch.float32), torch.tensor(c.scale, dtype=torch.float32)
    if c.act == 3:
        t = torch.where(t > 0, t, t * alpha)
    return (t * scale).view(c.shape)


@pytest.mark.parametrize("c", T.BIAS_ACT, ids=T.bias_act_id)
def test_bias_act_bit_exact(L, sms, c):
    dev = torch.device("cuda", 0)
    n, size_b, step_b = T.bias_act_dims(c)
    x, b = bias_act_operands(c)
    assert T.bias_act_id(c, sms) == T.bias_act_id(c), "the path class differs on this device's SM count"
    xd = at_offset(x, c.x_off, dev)
    y = nan_like(c.shape, c.y_off, dev)
    bd = b.to(dev) if size_b else None
    L.check(L.lib().hf_bias_act_f32(xd.data_ptr(), None if bd is None else bd.data_ptr(), y.data_ptr(), n, size_b,
                                    step_b, c.act, c.alpha, c.scale, L.stream_ptr()), "hf_bias_act_f32")
    assert_bits(y.cpu(), bias_act_ref(x, b, c), c.name)


# ------------------------------------------------------------------------------------------------ BicubicDownSample
def bicubic_call(L, x, k, f, clip_round, dev):
    p, h, w = x.shape
    xd, kd = x.float().to(dev), k.float().to(dev)
    y = torch.full((p, h // f, w // f), float("nan"), device=dev)
    L.check(L.lib().hf_bicubic_downsample_f32(xd.data_ptr(), kd.data_ptr(), y.data_ptr(), p, h, w, f, int(clip_round),
                                              L.stream_ptr()), "hf_bicubic_downsample_f32")
    return y.cpu()


def bicubic_shapes(f):
    """(planes, H, W): partial tiles in both axes (Ho % 8, Wo % 64 != 0, two tile columns), and the smallest image
    the reflect padding allows (3f - 3f // 2 + 1; top and bottom pads differ for odd f)."""
    small = 3 * f - 3 * f // 2 + 1
    return [(3, 11 * f + f // 2, 70 * f + (f - 1)), (2, small, small + 1)]


@pytest.mark.parametrize("f", range(1, 9), ids=lambda f: f"f{f}")
def test_bicubic_downsample_bit_exact(L, f):
    """Integer images and taps that are multiples of 1/64 (distinct, of both signs): every sum is exact."""
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(f)
    k = ints(g, (4 * f,), -16, 16) / 64
    for shape in bicubic_shapes(f):
        x = ints(g, shape, -8, 8)
        ref = exact32(T.bicubic_ref(x, k, f, False))
        assert_equal(bicubic_call(L, x, k, f, False, dev), ref, f"f{f} {shape}")


@pytest.mark.parametrize("f", range(1, 9), ids=lambda f: f"f{f}")
def test_bicubic_downsample_clip_round_bit_exact(L, f):
    """clip_round: taps that are multiples of 1/2 make about half the values land exactly on k + 1/2, for even and odd
    k, which rintf rounds to even; values fall below 0 and above 255 in both passes, and the second pass reads the
    clamped, rounded first pass."""
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(100 + f)
    k = pick(g, (4 * f,), [-0.5, 0.0, 0.5])
    k[1:3] = torch.tensor([0.5, -0.5])
    k[0] += 1 - k.sum()                                 # unit gain: the values spread on both sides of 0 .. 255
    for shape in bicubic_shapes(f):
        x = ints(g, shape, -30, 285)
        keep = []
        ref = exact32(T.bicubic_ref(x, k, f, True, keep))
        if shape[0] == 3:                             # the large image covers every rounding and clamping case
            for i, v in enumerate(keep):
                frac = v - v.floor()
                ties = v[frac == 0.5].floor()
                assert (ties % 2 == 0).any() and (ties % 2 == 1).any(), f"pass {i}: no ties of both parities"
                assert (v < -0.5).any() and (v > 255.5).any(), f"pass {i}: nothing to clamp"
        assert_equal(bicubic_call(L, x, k, f, True, dev), ref, f"f{f} {shape}")


@pytest.mark.parametrize("f", [2, 4], ids=["f2", "f4"])
def test_bicubic_downsample_module_bounded(L, f):
    """BicubicDownSample(f).k on data in [-1, 1] against float64 with the same fp32 taps.  Each pass is a chain of 4f
    FFMAs, each rounding by at most 2^-24 of the sum of |terms|; the second pass also carries the first pass's error
    through sum |k|: bound 8 f * 2^-24 * (sum |k|)^2 * max|x|.  The module's nhwc and byte_output forms equal the
    direct call bit for bit."""
    import hairfastgan_b200.bicubic as B
    dev = torch.device("cuda", 0)
    m = B.BicubicDownSample(factor=f)
    k = m.k.double()
    g = torch.Generator().manual_seed(f)
    x = (torch.rand(6, 67 * f + 1, 131 * f + 3, generator=g) * 2 - 1).double()
    got = bicubic_call(L, x, k, f, False, dev)
    s1 = float(k.abs().sum())
    ref = T.bicubic_ref(x, k, f, False)
    assert_within(got.double(), ref, torch.full_like(ref, 8 * f * EPS * s1 * s1), f"BicubicDownSample({f}).k")
    xm = x.float().view(2, 3, *x.shape[1:]).to(dev)
    assert_equal(m(xm).cpu().view(got.shape), got, "module, NCHW")
    nhwc = m(xm.permute(0, 2, 3, 1).contiguous(), nhwc=True)
    assert_equal(nhwc.permute(0, 3, 1, 2).cpu().reshape(got.shape), got, "module, nhwc=True")
    img = (x * 140 + 127).round()                      # the swap() form: 0..255 images, clamp-round, bytes on the host
    direct = bicubic_call(L, img, k, f, True, dev)
    byte = m(img.float().view(2, 3, *x.shape[1:]).to(dev), clip_round=True, byte_output=True)
    assert byte.dtype == torch.uint8 and not byte.is_cuda
    assert_equal(byte.view(got.shape), direct.to(torch.uint8), "module, byte_output=True")


# ------------------------------------------------------------------------------------------------ DilateErosion
def dilate_erode_ref(m, iterations):
    """image_utils.py:42-55 on 0/1 masks: each round sums the 3x3 cross with zero padding; dilation keeps sum > 0,
    erosion keeps sum == 5; the two masks advance separately."""
    cross = torch.tensor([[0, 1, 0], [1, 1, 1], [0, 1, 0]], dtype=torch.float64).view(1, 1, 3, 3)
    d, e = m.clone(), m.clone()
    for _ in range(iterations):
        d = (F.conv2d(d[:, None], cross, padding=1)[:, 0] > 0).double()
        e = (F.conv2d(e[:, None], cross, padding=1)[:, 0] == 5).double()
    return d, e


DILATE = [(3, 17, 23), (2, 1, 9), (2, 9, 1), (1, 1, 1), (4, 6, 40), (3, 512, 400)]


@pytest.mark.parametrize("planes,h,w", DILATE, ids=[f"{p}x{h}x{w}" for p, h, w in DILATE])
def test_dilate_erode_bit_exact(L, sms, planes, h, w):
    """Iterations 0, 1, 2, 3 (the first ping-pong buffer is read, then written again) and 5.  Every plane has set
    pixels on its first and last row and column next to clear ones, so a neighbour read across a plane boundary
    changes the dilation or the erosion.  3 x 512 x 400 needs a second grid-stride iteration."""
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(planes * h * w)
    m = (torch.rand(planes, h, w, generator=g) < 0.55).double()
    if h > 2 and w > 2:
        m[:, 0, ::3] = 1
        m[:, -1, 1::3] = 1
        m[:, 2::3, 0] = 1
        m[:, ::4, -1] = 1
        m[1::2, 0, 1::3] = 0
        m[::2, -1, ::3] = 0
    if planes * h * w > 4 * h * w * 3:
        assert planes * h * w > T.grid_threads(sms), "one grid covers the tensor: no grid-stride iteration"
    # the mask and the workspace are followed by a guard plane of ones: a read past the last row of the last plane
    # sets pixels of the dilation instead of going unnoticed
    md = torch.ones(planes + 1, h, w, device=dev)[:planes]
    md.copy_(m.float())
    for it in (0, 1, 2, 3, 5):
        d = torch.full_like(md, float("nan"))
        e = torch.full_like(md, float("nan"))
        ws = torch.full((4 * md.numel(),), float("nan"), device=dev)
        ws = torch.cat([ws, torch.ones(h * w, device=dev)])
        L.check(L.lib().hf_dilate_erode_f32(md.data_ptr(), d.data_ptr(), e.data_ptr(), ws.data_ptr(), planes, h, w, it,
                                            L.stream_ptr()), "hf_dilate_erode_f32")
        rd, re = dilate_erode_ref(m, it)
        assert_equal(d.cpu().double(), rd, f"dilate, {it} iterations")
        assert_equal(e.cpu().double(), re, f"erode, {it} iterations")


@pytest.mark.parametrize("n", [1, 256, 1000, 65543], ids=["n1", "n256", "n1000", "n65543"])
def test_align_masks_bit_exact(L, n):
    """[1 - (1 - hm1)(1 - hmx), hmx, hm2 * hmx] on 0/1 masks and on multiples of 1/8: every product is exact."""
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(n)
    for values in ([0.0, 1.0], [0.0, 0.125, 0.25, 0.5, 0.75, 1.0]):
        a, b, x = (pick(g, (n,), values) for _ in range(3))
        out = torch.full((3, n), float("nan"), device=dev)
        ad, bd, xd = a.float().to(dev), b.float().to(dev), x.float().to(dev)
        L.check(L.lib().hf_align_masks_f32(ad.data_ptr(), bd.data_ptr(), xd.data_ptr(), out.data_ptr(), n,
                                           L.stream_ptr()), "hf_align_masks_f32")
        ref = exact32(torch.stack([1 - (1 - a) * (1 - x), x, b * x]))
        assert_equal(out.cpu(), ref, f"values {values}")


# ------------------------------------------------------------------------------------------------ F-space blend
SCALES = [(1.0, -1.0), (0.0, 0.5), (0.5, 1.0), (-1.0, 2.0)]          # (scale_a, scale_b) of stages 0..3


def fspace_operands(c):
    g = torch.Generator().manual_seed(T.seed(c.name))
    first = ints(g, (c.C, c.Ho, c.Wo), -4, 4)
    srcs = [ints(g, (c.C, c.Ho, c.Wo), -4, 4) for _ in range(c.stages)]
    if c.mask == "int":
        masks = [ints(g, (c.Hm, c.Wm), 0, 3) for _ in range(c.stages)]
    else:
        masks = [pick(g, (c.Hm, c.Wm), [0.0, 0.25, 0.5, 0.75, 1.0]) for _ in range(c.stages)]
    return first, srcs, masks


def fspace_ref(first, srcs, masks, ho, wo, scales, mode="exact"):
    """w_s = scale_a + scale_b * bicubic(mask_s); F = src_s + w_s (F - src_s).

    exact: float64, and every weight, product and stage result must be exact in fp32, so no rounding or contraction
    of the kernel can matter.  ffma: the weights must be exact in fp32, the products need not be; each stage is then
    evaluated as the kernel's SASS does, d = fl(F - src) and one rounding of src + w d (FFMA), with that sum formed
    exactly in float64 (TwoSum asserts it) before its single rounding.  float64: no assertion (the bounded case)."""
    f = first
    for s, (src, m) in enumerate(zip(srcs, masks)):
        a, b = scales[s]
        w = a + b * T.bicubic_interp_ref(m, ho, wo)
        if mode == "ffma":
            d = (exact32(f, f"stage {s} input") - exact32(src, "source")).double()
            p = exact32(w, f"stage {s} weight").double() * d           # exact: two 24-bit significands
            t = p + src
            bv = t - p
            assert torch.equal((p - (t - bv)) + (src - bv), torch.zeros_like(t)), "FFMA sum not exact in float64"
            f = t.float().double()
            continue
        prod = w * (f - src)
        f = src + prod
        if mode == "exact":
            for v, what in ((w, "weight"), (prod, "product"), (f, "stage result")):
                exact32(v, f"stage {s} {what}")
    return f


def fspace_call(L, first, srcs, masks, scales, offs, dev):
    """hf_fspace_blend_f32 with first, each src and out starting `offs` bytes into their allocations."""
    n = len(srcs)
    C_, ho, wo = first.shape
    hm, wm = masks[0].shape
    import ctypes as C
    fd = at_offset(first.float(), offs, dev)
    sd = [at_offset(s.float(), offs, dev) for s in srcs]
    md = [m.float().to(dev) for m in masks]
    out = nan_like(first.shape, offs, dev)
    sp, mp = (C.c_void_p * n)(*[s.data_ptr() for s in sd]), (C.c_void_p * n)(*[m.data_ptr() for m in md])
    sa, sb = (C.c_float * n)(*[scales[i][0] for i in range(n)]), (C.c_float * n)(*[scales[i][1] for i in range(n)])
    L.check(L.lib().hf_fspace_blend_f32(fd.data_ptr(), sp, mp, sa, sb, out.data_ptr(), n, C_, ho, wo, hm, wm,
                                        L.stream_ptr()), "hf_fspace_blend_f32")
    return out.cpu()


@pytest.mark.parametrize("c", T.FSPACE, ids=T.fspace_id)
def test_fspace_blend_bit_exact(L, c):
    """Down by 8, 4 and 2 (t = 1/2), up by 2 (t = 1/4, 3/4; negative source index at the top and left, clamped taps),
    the same size (t = 0), non-square ratios, 1 to 4 stages with distinct masks and scales, C not a multiple of 16 or
    4.  Chains of several stages with fine weights outgrow fp32 and are compared with the FFMA evaluation.  Unaligned cases: first, every src and out 4 bytes into their buffers take the scalar loop and must equal the
    aligned call bit for bit."""
    dev = torch.device("cuda", 0)
    first, srcs, masks = fspace_operands(c)
    ref = exact32(fspace_ref(first, srcs, masks, c.Ho, c.Wo, SCALES, c.ref))
    got = fspace_call(L, first, srcs, masks, SCALES, 0 if c.aligned else 4, dev)
    assert_equal(got, ref, c.name)
    if not c.aligned:
        assert_bits(got, fspace_call(L, first, srcs, masks, SCALES, 0, dev), "unaligned vs aligned call")


def test_fspace_blend_nondyadic_ratio_bounded(L):
    """50 x 70 -> 20 x 12 (ratios 2.5, 35/6), 2 stages.  The fp32 source coordinate (oy + 0.5) * fl(Hm / Ho) - 0.5
    is off by at most 2^-23 (Hm + 1); the cubic weights' slopes are below 2 per tap, so the interpolated mask moves by
    at most 16 * 2^-23 (Hm + 1) max|m|, plus 16 roundings of 2^-24 * sum |w m| (sum |w| <= 1.5 per axis, so 2.25 max|m|)
    in the two weighted sums.  The weight error times |scale_b| multiplies |F - src|, and the two FFMAs of each stage
    round once each: with max|F|, max|src| <= 4 (|w| <= 3) the bound below covers two stages."""
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(7)
    C_, ho, wo, hm, wm = 3, 20, 12, 50, 70
    first = ints(g, (C_, ho, wo), -4, 4)
    srcs = [ints(g, (C_, ho, wo), -4, 4) for _ in range(2)]
    masks = [ints(g, (hm, wm), 0, 1) for _ in range(2)]
    ref = fspace_ref(first, srcs, masks, ho, wo, SCALES, "float64")
    m_err = 16 * 2.0 ** -23 * (max(hm, wm) + 1) + 16 * EPS * 2.25
    stage = 2 * m_err * 8 + 2 * EPS * 16                   # |scale_b| <= 2, |F - src| <= 8, |F| <= 16 after stage 0
    bound = torch.full_like(ref, 4 * stage)                # stage 1 carries stage 0's error times |w| <= 3
    assert_within(fspace_call(L, first, srcs, masks, SCALES, 0, dev).double(), ref, bound, "non-dyadic ratio")

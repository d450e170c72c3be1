"""Exact-arithmetic tests of the generator chain (csrc/hf_generator.cu) and the code it runs between the MMAs: the
style affine, the demodulation table and the NCHW -> NHWC pre-pass (csrc/hf_ops.cu), the generator epilogue of the
wgmma convolution with its 16-bit handoff and fused ToRGB partial sums (csrc/hf_conv_tc.cu), and rgb_combine.

Operands are small integers or dyadic values; the reference is float64 torch written here.

a. Standalone ToRGB (hf_torgb_forward) is checked BIT FOR BIT.  The ToRGB weights are snapped: w1 is the fp32 value
   for which fl(w1 * fl(1/sqrt(cin))) is a small integer m (found by an fp32 search below), so with integer x, dyadic
   styles, bias and skip and the [1,3,3,1] upsample kernel (multiples of 1/16) every fp32 intermediate is exact.  The
   style affine is observed through an impulse probe: pixel p of x is 1 in channel c(p) only, so
   y[b,j,p] = fl(bias_j + fl(m[j,c(p)] * s[b,c(p)])) with s = fl(dot * fl(1/sqrt(D)) + mod_bias).  The dot products
   are integers, so s is ONE rounding of an exact value and float64 reproduces it, also for D = 512 where the weight
   scale 2^-4.5 is not dyadic.

b. The generator chain (Generator._run -> hf_generator_forward) is checked link by link.  Every conv output a' (after
   demodulation, noise, bias and the scaled LeakyReLU) is observed through return_features.  The input of the next
   conv is rebuilt from the observed a' exactly as the epilogue builds it (an fp32 multiply by the next conv's style,
   then round-to-nearest-even to 16 bits), and its float64 accumulator is exact: the test asserts, per output, that
   the sum of |terms| stays below 2^24 times the smallest bit among them.  Three things keep that true along the chain:
   integer conv weights (snapped like the ToRGB weights, so the demodulation sums are exact too), two (channel, tap)
   pairs per output channel, and positive inputs, styles, noise and biases on the channels that feed the next conv,
   with biases that grow with depth like the activations do (nothing cancels, so no activation is orders of magnitude
   below its neighbours).  A quarter of the channels have a negative bias and reach the negative side of the
   LeakyReLU; they feed the ToRGB and nothing else.  The demodulation loop for Cin > 512 is reached with
   channel_multiplier 4 (1024 channels at 64^2), the pre-pass channel tail (C = 32) by an FSE feature insertion
   before the last conv of a 512^2, channel_multiplier 1 generator.
   What is left, a' = lrelu(acc * fl(d * sqrt2) + fl(fl(sqrt2 * nw) * noise) + fl(bias * sqrt2)), is bounded by
   10 * 2^-24 * (|acc d sqrt2| + |sqrt2 nw noise| + |sqrt2 bias|) (derivation at `check_conv`): about 2^-20 relative,
   while one 16-bit ulp in one handed-off activation moves an output by 2^-8 (bf16) or 2^-11 (fp16) of a term; a test
   below perturbs one element by one ulp and asserts that the check fails.  The fused ToRGB and rgb_combine are checked
   against float64 from the observed a' with a bound that names the fp32 summation length (N-tile partials).
   Every range also runs without return_features, which switches the epilogue variants; out_rgb and out_feature must
   be bit-identical between the two runs, which ties the observed chain to the production one.

Case ids name the dispatch paths: the affine path (D512 register path / generic) and the B % 4 tail, the demodulation
path (register path for Cin <= 512, strided loop above), the rgb_combine kernel (vec4 / scalar), skip or not, in place
or not, the epilogue variants (rgb_partial | out_nchw << 1 | xhat_out << 2) with and without return_features, and the
number of N-tile partials of every fused ToRGB, for a 132-SM H100."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from tests.gpu_util import dtype_name

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

U = 2.0 ** -24                                              # unit roundoff of fp32
SQRT2 = math.sqrt(2.0)
EPS_DEMOD = float(torch.tensor(1e-8, dtype=torch.float32))  # the 1e-8f of demod_kernel
SLOPE = float(torch.tensor(0.2, dtype=torch.float32))       # the 0.2f of the epilogue's LeakyReLU
SMS_NAMED = 132                                             # the N-tile counts in the case ids are for 132 SMs


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


# ------------------------------------------------------------------------------------------------ operands
def pick(g, shape, values):
    """Seeded draws from a list of (dyadic) values as float64."""
    v = torch.tensor(values, dtype=torch.float64)
    return v[torch.randint(0, len(values), shape, generator=g)]


def f32(x):
    """One round-to-nearest-even of a float64 tensor to fp32, back in float64."""
    return x.float().double()


def inv_sqrt_f32(n):
    """fl(1 / fl(sqrt(n))): the scale the library computes as 1.0f / sqrtf((float)n) (IEEE division and sqrt)."""
    return torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(torch.tensor(float(n), dtype=torch.float32))


def snap(m, scale):
    """The fp32 w nearest to m / scale with fl(w * scale) == m exactly (m a small integer, scale an fp32 scalar)."""
    w = torch.tensor(float(m), dtype=torch.float32) / scale
    cands, up, dn = [w], w, w
    for _ in range(16):
        up, dn = torch.nextafter(up, torch.tensor(math.inf)), torch.nextafter(dn, torch.tensor(-math.inf))
        cands += [up, dn]
    for c in cands:
        if float(c * scale) == float(m):
            return float(c)
    raise AssertionError(f"no fp32 w with fl(w * {float(scale)!r}) == {m}")


def snapped(mi, scale):
    """Integer-valued float64 tensor -> fp32 weights whose scaled fp32 value is that integer."""
    w = torch.zeros(mi.shape, dtype=torch.float32)
    for v in mi.unique().tolist():
        if v != 0:
            w[mi == v] = math.copysign(snap(abs(v), scale), v)
    return w


def up2(x, k):
    """Upsample (model.py:35-53) = upfirdn2d(x, k, up=2, pad=(2, 1)) in float64: zero insertion, pad, flipped k."""
    B, Cc, h, w = x.shape
    u = x.new_zeros(B * Cc, 1, 2 * h, 2 * w)
    u[:, :, ::2, ::2] = x.reshape(B * Cc, 1, h, w)
    u = F.pad(u, (2, 1, 2, 1))
    return F.conv2d(u, torch.flip(k, (0, 1)).view(1, 1, 4, 4)).view(B, Cc, 2 * h, 2 * w)


def blur_up_conv(x, w, blur):
    """The up-conv accumulator in float64: stride-2 transposed conv (model.py:260), then Blur(pad=(1, 1))."""
    out = F.conv_transpose2d(x, w.transpose(0, 1).contiguous(), None, 2, 0)
    B, Cc, h, ww = out.shape
    o = F.conv2d(F.pad(out.reshape(B * Cc, 1, h, ww), (1, 1, 1, 1)), torch.flip(blur, (0, 1)).view(1, 1, 4, 4))
    return o.view(B, Cc, h - 1, ww - 1)


def lsb16(x, tdt):
    """Weight of the last mantissa bit of each (16-bit representable) value; +inf where the value is zero."""
    mant, emin = (10, -24) if tdt == torch.float16 else (7, -133)
    _, e = torch.frexp(x)
    lsb = torch.pow(2.0, (e - 1 - mant).double()).clamp_min(2.0 ** emin)
    return torch.where(x == 0, torch.full_like(x, math.inf), lsb)


def first_bad(got, ref, bound, what):
    bad = ((got - ref).abs() > bound).nonzero()
    if bad.numel() == 0:
        return ""
    i = tuple(int(v) for v in bad[0])
    return (f"{what}: {bad.shape[0]} of {ref.numel()} values out of bound; first at {i}: got {float(got[i])!r}, "
            f"expected {float(ref[i])!r}, bound {float(bound[i]):.3g}")


def plan(cin, cout, res, batch, up, dtype):
    """(n_tile, number of N tiles) of the conv launch, from the library's plan query."""
    from hairfastgan_b200 import _lib
    d = _lib.hf_conv_desc(cin, cout, 3, up, dtype)
    out = (C.c_int * 12)()
    _lib.check(_lib.lib().hf_conv_plan_query(C.byref(d), batch, res, res, out), "hf_conv_plan_query")
    return out[1], out[2]


def n_tiles_named(cout, res, batch, sms=SMS_NAMED):
    """conv_plan's N-tile choice for a plain 3x3 conv (the largest tile that still fills the GPU)."""
    tw = min(res, 16)
    th = min(res, 128 // tw)
    tb = 128 // (tw * th)
    m_tiles = (res // tw) * (res // th) * -(-batch // tb)
    nt = 0
    for cand in (128, 64, 32):
        if cout % cand or tb * cand > 512:
            continue
        nt = cand
        if m_tiles * (cout // cand) >= sms:
            break
    return cout // nt


# ================================================================================================ a. standalone ToRGB
def make_torgb(g, cin, D, dev, mw_range):
    """ToRGB with snapped integer weights m in {-3..3} \\ {0}, integer modulation weights, dyadic biases.  Not every
    integer has a snapped weight (at cin = 32 and 512 no fp32 w gives fl(w * fl(1/sqrt(cin))) == 3); those are left
    out."""
    import hairfastgan_b200.model as M
    tr = M.ToRGB(cin, D)
    ms = []
    for v in (1, 2, 3):
        try:
            snap(v, inv_sqrt_f32(cin))
            ms += [v, -v]
        except AssertionError:
            pass
    m = pick(g, (3, cin), ms)
    tr.conv.weight.data = snapped(m, inv_sqrt_f32(cin)).view(1, 3, cin, 1, 1)
    mw = torch.randint(-mw_range, mw_range + 1, (cin, D), generator=g).double()
    mb = pick(g, (cin,), [-1.0, 0.5, 1.0, 1.25])
    bias = pick(g, (3,), [-0.5, 0.0, 0.25])
    tr.conv.modulation.weight.data, tr.conv.modulation.bias.data = mw.float(), mb.float()
    tr.bias.data = bias.float().view(1, 3, 1, 1)
    return tr.to(dev), m.to(dev), mw.to(dev), mb.to(dev), bias.to(dev)


def affine_ref(style, mw, mb, D):
    """s = fmaf(dot, fl(1/sqrt(D)), mod_bias): the dot product is an integer, so this is one rounding of an exact
    value, which float64 computes exactly before the single rounding to fp32."""
    dot = style @ mw.T
    assert torch.equal(dot, dot.round()) and float(dot.abs().max()) < 2 ** 24
    return f32(dot * float(inv_sqrt_f32(D)) + mb)


def torgb_raw(tr, x, style, skip, y_offset):
    """hf_torgb_forward into a y that starts `y_offset` floats into a NaN-filled buffer (offset 1: not 16-byte
    aligned, so rgb_combine takes its scalar kernel).  Returns (y, buffer)."""
    from hairfastgan_b200 import _lib
    B, cin, H, W = x.shape
    n = B * 3 * H * W
    buf = torch.full((n + 8,), math.nan, device=x.device)
    y = buf[y_offset:y_offset + n].view(B, 3, H, W)
    ws = torch.empty(B * cin, device=x.device)
    upk = tr.upsample.kernel.contiguous()
    _lib.check(_lib.lib().hf_torgb_forward(
        x.data_ptr(), style.data_ptr(), style.stride(0), style.shape[1], tr.conv.weight.data_ptr(),
        tr.conv.modulation.weight.data_ptr(), tr.conv.modulation.bias.data_ptr(), tr.bias.data_ptr(),
        upk.data_ptr() if skip is not None else None, skip.data_ptr() if skip is not None else None, y.data_ptr(),
        B, cin, H, W, ws.data_ptr(), _lib.stream_ptr()), "hf_torgb_forward")
    torch.cuda.synchronize()
    return y, buf


# (D, cin, H, W, B): the D = 512 register path (four samples per pass, B % 4 tail clamped) and the generic path
AFFINE = [(512, 64, 8, 8, b) for b in (1, 3, 4, 5, 6)] + [(512, 512, 16, 32, 5), (16, 64, 8, 8, 5), (64, 96, 8, 12, 3),
                                                        (64, 64, 8, 8, 6)]


def affine_id(p):
    D, cin, H, W, B = p
    path = "affineD512" if D == 512 else f"affineGenericD{D}"
    return f"{path}-B{B}tail{B % 4}-cin{cin}-vec4_inplace_noskip"


@pytest.mark.parametrize("D,cin,H,W,B", AFFINE, ids=[affine_id(p) for p in AFFINE])
def test_torgb_affine_impulse_bit_exact(dev, dt, D, cin, H, W, B):
    """Every style scale s[b, c] of every sample, observed one pixel per channel through the ToRGB."""
    g = torch.Generator().manual_seed(D + cin + 7 * B)
    tr, m, mw, mb, bias = make_torgb(g, cin, D, dev, 3)
    style = torch.randint(-3, 4, (B, D), generator=g).double().to(dev)      # a different row per sample
    c_of_p = torch.arange(H * W) % cin
    x = torch.zeros(B, cin, H * W, dtype=torch.float64)
    x[:, c_of_p, torch.arange(H * W)] = 1.0
    x = x.view(B, cin, H, W).to(dev)
    s = affine_ref(style, mw, mb, D)                                        # [B, cin]
    wsc = f32(m[None] * s[:, None, :])                                      # fl(m * s): [B, 3, cin]
    ref = f32(bias.view(1, 3, 1) + wsc[:, :, c_of_p.to(dev)]).view(B, 3, H, W)
    y = tr(x.float(), style.float())
    got = y.double()
    assert torch.equal(got, ref), first_bad(got, ref, torch.zeros_like(ref), "ToRGB impulse (affine)")


def edge_impulse_skip(g, B, h2, w2, dev):
    """Sample b: one impulse per RGB plane at the b-th of the half-resolution image's corners and edge midpoints."""
    pos = [(0, 0), (0, w2 - 1), (h2 - 1, 0), (h2 - 1, w2 - 1), (0, w2 // 2), (h2 - 1, w2 // 2), (h2 // 2, 0),
           (h2 // 2, w2 - 1)]
    sk = torch.zeros(B, 3, h2, w2, dtype=torch.float64)
    for b in range(B):
        y, x = pos[b % len(pos)]
        sk[b, :, y, x] = pick(g, (3,), [-4.0, -2.0, -1.0, 1.0, 2.0, 4.0])
    return sk.to(dev)


# (name, cin, H, W, skip, y offset in floats)
TORGB = [
    ("vec4_inplace_skip_W8", 64, 8, 8, True, 0),
    ("vec4_inplace_noskip_W8", 64, 8, 8, False, 0),
    ("vec4_inplace_skip_cin512_W16", 512, 8, 16, True, 0),
    ("scalar_W%4=2_inplace_skip_W10", 64, 6, 10, True, 0),
    ("scalar_W%4=2_inplace_noskip_W10", 64, 6, 10, False, 0),
    ("scalar_yoffset4B_inplace_skip_W8", 64, 8, 8, True, 1),
    ("scalar_yoffset4B_inplace_noskip_W8", 64, 8, 8, False, 1),
]


@pytest.mark.parametrize("name,cin,H,W,with_skip,y_off", TORGB, ids=[t[0] for t in TORGB])
def test_torgb_bit_exact(dev, dt, name, cin, H, W, with_skip, y_off):
    """Integer x, snapped integer weights, dyadic styles (generic affine, D = 16: fl(1/4) is exact), bias and skip:
    every product and partial sum is a multiple of 1/64 below 2^18, so y equals the float64 reference bit for bit.
    rgb_combine runs in place (the ToRGB partial is y itself).  The scalar kernel must give the vec4 kernel's bits."""
    D, B = 16, 8 if with_skip else 5
    g = torch.Generator().manual_seed(cin + H * W + with_skip)
    tr, m, mw, mb, bias = make_torgb(g, cin, D, dev, 1)
    style = torch.randint(-1, 2, (B, D), generator=g).double().to(dev)
    x = (torch.randint(-2, 3, (B, cin, H, W), generator=g) * (torch.rand(B, cin, H, W, generator=g) < 0.5)).double()
    x = x.to(dev)
    skip = edge_impulse_skip(g, B, H // 2, W // 2, dev) if with_skip else None
    if skip is not None:                          # plus a dyadic background on the last sample
        skip[-1] += pick(g, (3, H // 2, W // 2), [-0.75, -0.25, 0.0, 0.5, 1.0]).to(dev)
    s = affine_ref(style, mw, mb, D)
    wsc = m[None] * s[:, None, :]
    assert torch.equal(f32(wsc), wsc)
    ref = torch.einsum("bchw,bjc->bjhw", x, wsc) + bias.view(1, 3, 1, 1)
    if skip is not None:
        ref = ref + up2(skip, tr.upsample.kernel.double())
    assert torch.equal(f32(ref), ref), "the reference must be exact in fp32"
    y, buf = torgb_raw(tr, x.float(), style.float(), None if skip is None else skip.float(), y_off)
    n = y.numel()
    assert torch.isnan(buf[:y_off]).all() and torch.isnan(buf[y_off + n:]).all(), "wrote outside y"
    assert torch.equal(y.double(), ref), first_bad(y.double(), ref, torch.zeros_like(ref), name)
    if y_off:            # the same operands on the vec4 kernel: the same bits
        y4, _ = torgb_raw(tr, x.float(), style.float(), None if skip is None else skip.float(), 0)
        assert torch.equal(y4, y), "vec4 and scalar rgb_combine differ"
    else:                # the module path is this entry point
        ym = tr(x.float(), style.float(), None if skip is None else skip.float())
        assert torch.equal(ym, y)


def test_misaligned_style_rows_are_rejected_before_any_launch(dev, dt):
    """The affine reads style rows and modulation weights with float4 loads; a contiguous fp32 view that starts 4
    bytes into an allocation is refused by the library before it launches anything."""
    import hairfastgan_b200.model as M
    buf = torch.zeros(4096, device=dev)
    tr = M.ToRGB(64, 16).to(dev)
    x = torch.zeros(2, 64, 4, 4, device=dev)
    st = buf[1:33].view(2, 16)
    assert st.is_contiguous() and st.data_ptr() % 16 == 4
    with pytest.raises(RuntimeError, match="style and mod_weight must be 16-byte aligned"):
        tr(x, st)
    tr.conv.modulation.weight.data = buf[1:1 + 64 * 16].view(64, 16)
    with pytest.raises(RuntimeError, match="style and mod_weight must be 16-byte aligned"):
        tr(x, torch.zeros(2, 16, device=dev))
    gen = M.Generator(8, 64, 1).to(dev)
    gen.compute_dtype = dt[0]
    lat = buf[1:1 + 2 * gen.n_latent * 64].view(2, gen.n_latent, 64)
    with pytest.raises(RuntimeError, match="latent must be 16-byte aligned"):
        gen._run(lat, None, False)


# ================================================================================================ b. generator chain
# config name -> (size, style_dim, channel_multiplier, batch)
CONFIGS = {
    "g8_D64_cm2": (8, 64, 2, 3),
    "g16_D512_cm2": (16, 512, 2, 5),
    "g32_D64_cm1": (32, 64, 1, 2),
    "g64_D64_cm1": (64, 64, 1, 2),
    "g64_D512_cm4": (64, 512, 4, 1),        # 1024 channels at 64^2: the demodulation loop for Cin > 512
    "g512_D64_cm1": (512, 64, 1, 1),        # 32 channels at 512^2: the pre-pass channel tail (C % 64 == 32)
}


def channels(res, cm):
    return {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * cm, 128: 128 * cm, 256: 64 * cm, 512: 32 * cm}[res]


def layers_run(n, start, end):
    """Mirror of the layer loop of Generator.forward (model.py:534-557)."""
    run = [start == 0] + [False] * n
    if end != 0:
        for k in range(1, n + 1):
            if k < start:
                continue
            if k > end and k != start:
                break
            run[k] = True
    return [k for k in range(n + 1) if run[k]]


def convs_of(k):
    return [0] if k == 0 else [2 * k - 1, 2 * k]


def conv_shape(i, cm):
    """(cin, cout, res_in, res_out, up) of styled conv i."""
    if i == 0:
        return 512, 512, 4, 4, 0
    k = (i + 1) // 2
    r = 4 << k
    up = i & 1
    return channels(r // 2 if up else r, cm), channels(r, cm), r // 2 if up else r, r, up


def variants(n, layers, early, features):
    """Epilogue variant bits (rgb_partial | out_nchw << 1 | xhat_out << 2) of the executed convs."""
    v = set()
    last = layers[-1]
    for k in layers:
        more = k < last
        for i in convs_of(k):
            rgb = i == 0 or i % 2 == 0
            xout = (not rgb) or more
            nchw = features or (rgb and not more and early)
            v.add((1 if rgb else 0) | (2 if nchw else 0) | (4 if xout else 0))
    return "".join(str(x) for x in sorted(v))


# (config, start, end, feature_in index or None); single layers, the full range, an early exit
RANGES = []
for _name, (_size, _D, _cm, _B) in CONFIGS.items():
    _n = int(math.log2(_size)) - 2
    if _name == "g64_D512_cm4":
        RANGES.append((_name, 4, 4, None))
    elif _name == "g512_D64_cm1":
        RANGES.append((_name, 7, 7, 14))
    else:
        RANGES += [(_name, k, k, None) for k in range(1, _n + 1)]
        RANGES += [(_name, 0, 8, None), (_name, 0, _n - 1, None)]


def case_id(c):
    name, start, end, feat = c
    size, D, cm, B = CONFIGS[name]
    n = int(math.log2(size)) - 2
    layers = layers_run(n, start, end)
    early = layers[-1] < n
    nb = 1 if RANGES.index(c) % 2 == 0 else B
    rng = "full" if (start == 0 and not early) else (f"single{start}" if start == end and start else f"early0to{end}")
    affine = ("affineD512" if D == 512 else "affineGeneric") + f"_B{B}tail{B % 4}"
    cins = [conv_shape(i, cm)[0] for k in layers for i in convs_of(k)]
    demod = "demodGt512" if max(cins) > 512 else "demodLe512"
    nts = ".".join(str(n_tiles_named(channels(4 << k, cm), 4 << k, B)) for k in layers)
    fin = f"-featurein{feat}_prepassC{conv_shape(feat, cm)[0]}" if feat else ""
    return (f"{name}-{rng}-B{B}-noisebatch{nb}-{affine}-{demod}-epi{variants(n, layers, early, True)}"
            f"_vs_epi{variants(n, layers, early, False)}-rgbCombineVec4-ntiles{nts}{fin}")


class Chain:
    """A generator of one config with the float64 operands it was built from (on the device)."""

    def __init__(self, name, dt, dev):
        import hairfastgan_b200.model as M
        size, D, cm, B = CONFIGS[name]
        self.size, self.D, self.cm, self.B, self.tdt = size, D, cm, B, dt[1]
        self.n = int(math.log2(size)) - 2
        g = torch.Generator().manual_seed(size + D + cm)
        gen = M.Generator(size, D, 1, channel_multiplier=cm)
        gen.compute_dtype = dt[0]
        c4 = channels(4, cm)
        const = torch.randint(1, 4, (1, c4, 4, 4), generator=g).double()
        gen.input.input.data = const.float()
        self.const = const.to(dev)
        self.conv, self.rgb = [], []
        live_in = torch.ones(c4, dtype=torch.bool)
        for i, sc in enumerate(gen._styled()):
            cin, cout, _, _, up = conv_shape(i, cm)
            if i > 0:                                        # conv i reads the output of conv i - 1
                live_in = self.conv[i - 1]["live"].cpu()
            # two (input channel, tap) pairs per output channel, integer weights 1 or 2, only from channels that feed
            # forward (live); a repeated pair adds up (3 or 4)
            idx = live_in.nonzero().flatten()
            cc = idx[torch.randint(0, len(idx), (cout, 2), generator=g)]
            tt = torch.randint(0, 9, (cout, 2), generator=g)
            oo = torch.arange(cout).view(-1, 1).expand(cout, 2)
            w = torch.zeros(cout, cin, 9, dtype=torch.float64)
            w.index_put_((oo.reshape(-1), cc.reshape(-1), tt.reshape(-1)),
                         torch.randint(1, 3, (cout * 2,), generator=g).double(), accumulate=True)
            w = w.view(cout, cin, 3, 3)
            sc.conv.weight.data = snapped(w, inv_sqrt_f32(cin * 9)).view(1, cout, cin, 3, 3)
            mw, mb = self._modulation(g, cin)
            sc.conv.modulation.weight.data, sc.conv.modulation.bias.data = mw.float(), mb.float()
            # the activations grow about 2x per conv; so do the biases, which keeps the ratio of an activation that
            # sees no input (at the image border, where the two taps of its channel read the zero padding) to its
            # neighbours, and so the range of the next accumulator, bounded along the chain
            live = torch.rand(cout, generator=g) >= 0.25
            bias = torch.where(live, pick(g, (cout,), [0.5, 0.75, 1.0]), pick(g, (cout,), [-1.0, -2.0, -3.0]))
            bias = bias * 2.0 ** min(i, 8)
            nw = float(pick(g, (1,), [0.25, 0.5]))
            sc.activate.bias.data, sc.noise.weight.data = bias.float(), torch.tensor([nw])
            self.conv.append(dict(w=w.to(dev), pairs=cc.to(dev), wsq=w.pow(2).sum((2, 3)).to(dev), mw=mw.to(dev), mb=mb.to(dev),
                                  bias=bias.to(dev), nw=nw, live=live.to(dev), up=up,
                                  blur=sc.conv.blur.kernel.double().to(dev) if up else None))
        for k, tr in enumerate(gen._rgbs()):
            cin = channels(4 << k, cm)
            m = pick(g, (3, cin), [-2.0, -1.0, 1.0, 2.0])
            tr.conv.weight.data = snapped(m, inv_sqrt_f32(cin)).view(1, 3, cin, 1, 1)
            mw, mb = self._modulation(g, cin)
            tr.conv.modulation.weight.data, tr.conv.modulation.bias.data = mw.float(), mb.float()
            bias = pick(g, (3,), [-0.5, 0.0, 0.25])
            tr.bias.data = bias.float().view(1, 3, 1, 1)
            self.rgb.append(dict(m=m.to(dev), mw=mw.to(dev), mb=mb.to(dev), bias=bias.to(dev),
                                 upk=tr.upsample.kernel.double().to(dev) if k else None))
        self.gen = gen.to(dev).eval()

    def _modulation(self, g, cin):
        """Positive dyadic style scales.  D = 64: sparse {-1, 0, 1} weights, so s = dot / 8 + 2 in [1, 3], a
        multiple of 1/8.  D = 512: the weight scale fl(2^-4.5) is not dyadic, so the weights are zero and s is the
        bias (the register path is checked bit for bit by the ToRGB impulse tests)."""
        if self.D == 512:
            return torch.zeros(cin, self.D, dtype=torch.float64), pick(g, (cin,), [1.0, 1.5, 2.0])
        mw = torch.zeros(cin, self.D, dtype=torch.float64)
        mw[:, :8] = pick(g, (cin, 8), [-1.0, 0.0, 1.0])     # |dot| <= 8: s stays in [1, 3]
        return mw, torch.full((cin,), 2.0, dtype=torch.float64)

    def style(self, tbl, lat_row):
        s = affine_ref(lat_row, tbl["mw"], tbl["mb"], self.D)
        assert (s > 0).all()
        return s


_CHAINS = {}


def chain(name, dt, dev):
    key = (name, dt[0])
    if key not in _CHAINS:
        _CHAINS.clear()                       # one generator at a time (the 512^2 one holds ~100 MB of weights)
        _CHAINS[key] = Chain(name, dt, dev)
    return _CHAINS[key]


def handoff(a, s, tdt):
    """What the epilogue (and the pre-pass) writes for the next conv: fl(a * s) in fp32, then RNE to 16 bits."""
    return (a.float() * s.float()[:, :, None, None]).to(tdt).double()


def accumulate(cv, x16):
    with torch.backends.cudnn.flags(enabled=False):          # plain float64 GEMMs, no transform-based algorithms
        if cv["up"]:
            return blur_up_conv(x16, cv["w"], cv["blur"])
        return F.conv2d(x16, cv["w"], None, 1, 1)


def assert_exact_accumulator(cv, x16, tdt, what):
    """Precondition of the link check: the fp32 accumulator of the wgmma kernel is exact, in any summation order.
    Every product of output (b, o, y, x) is a multiple of q = (smallest 16-bit bit among the inputs of its 3x3 window
    in the two channels output channel o reads) * (weight bit: 1, or 1/16 for the blurred up-conv taps); if the sum of
    |products| stays below 2^24 q, every partial sum is exact."""
    lsb = -F.max_pool2d(-lsb16(x16, tdt), 3, 1, 1)                    # per channel, over the 3x3 window
    q = torch.minimum(lsb[:, cv["pairs"][:, 0]], lsb[:, cv["pairs"][:, 1]])   # the two input channels of output o
    with torch.backends.cudnn.flags(enabled=False):
        if cv["up"]:
            S = blur_up_conv(x16.abs(), cv["w"].abs(), cv["blur"])
            q = q.repeat_interleave(2, 2).repeat_interleave(2, 3) / 16
        else:
            S = F.conv2d(x16.abs(), cv["w"].abs(), None, 1, 1)
    ok = (S < 2.0 ** 24 * q).all()
    assert ok, f"{what}: the float64 accumulator is not exact in fp32; the operands must be changed"


def check_conv(cv, acc, s, noise, a_obs):
    """Violations of the bound on the epilogue's a' = lrelu(acc * d' + c') for one conv; returns (count, message).

    d' = fl(rsqrtf(fl(sum s^2 wsq + 1e-8f)) * fl(sqrt2)): the sum is exact (dyadic s, integer wsq), the +1e-8f
    rounding moves d by u/2, rsqrtf by at most 2 ulp = 4u, fl(sqrt2) and the product by u each: d' = d sqrt2 (1 + 7u).
    c' = fl(fl(fl(fl(sqrt2) * nw) * noise) + fl(bias * fl(sqrt2))): 3u on the noise term, 2u on the bias term, u on
    their sum.  The fmaf rounds once (u), the LeakyReLU fl(0.2f * a) once more (u / 5) and is 1-Lipschitz, so a sign
    flip near zero costs no more.  Total <= 8.2u (|acc d sqrt2| + |sqrt2 nw noise| + |sqrt2 bias|); the bound
    takes 10u, u = 2^-24."""
    d = torch.rsqrt(s.pow(2) @ cv["wsq"].T + EPS_DEMOD)                   # [B, cout]
    t_acc = acc * (d * SQRT2)[:, :, None, None]
    t_noise = SQRT2 * cv["nw"] * noise
    t_bias = SQRT2 * cv["bias"].view(1, -1, 1, 1)
    pre = t_acc + t_noise + t_bias
    ref = torch.where(pre > 0, pre, pre * SLOPE)
    bound = 10 * U * (t_acc.abs() + t_noise.abs() + t_bias.abs())
    bad = int(((a_obs - ref).abs() > bound).sum())
    return bad, first_bad(a_obs, ref, bound, "a'")


def positive_on_read_channels(g, cv, shape):
    """Integers 1..3 on the input channels conv `cv` reads, zero on the others (a quarter to a half of them).  A zero
    among the read inputs would let an activation stay at the noise + bias floor while its neighbours grow layer after
    layer, and stretch the range of the next accumulator beyond what fp32 holds exactly."""
    read = torch.zeros(shape[1], dtype=torch.bool)
    read[cv["pairs"].flatten().cpu()] = True
    return (torch.randint(1, 4, shape, generator=g) * read.view(1, -1, 1, 1)).double().to(cv["w"].device)


def run_case(ch, start, end, feat, nb, seed):
    B, dev = ch.B, ch.const.device
    g = torch.Generator().manual_seed(seed)
    layers = layers_run(ch.n, start, end)
    lat = pick(g, (B, ch.gen.n_latent, ch.D), [-1.0, 0.0, 0.0, 1.0]).to(dev)
    noise = [None] * ch.gen.num_layers
    for k in layers:
        for i in convs_of(k):
            r = conv_shape(i, ch.cm)[3]
            noise[i] = pick(g, (nb, 1, r, r), [0.0, 0.25, 0.5, 0.75, 1.0]).to(dev)
    layer_in = skip = None
    if start > 0:
        r_in = 4 << (start - 1)
        c_in = channels(r_in, ch.cm)
        layer_in = positive_on_read_channels(g, ch.conv[2 * start - 1], (B, c_in, r_in, r_in))
        skip = pick(g, (B, 3, r_in, r_in), [-2.0, -1.25, -0.5, 0.0, 0.25, 1.0, 1.75]).to(dev)
    features_in = None
    if feat is not None:
        cin, _, r, _, _ = conv_shape(feat, ch.cm)
        features_in = [None] * ch.gen.num_layers
        features_in[feat] = positive_on_read_channels(g, ch.conv[feat], (B, cin, r, r))

    def call(return_features):
        fin = None if features_in is None else [None if f is None else f.float() for f in features_in]
        out = ch.gen._run(lat.float(), noise, False, None if layer_in is None else layer_in.float(),
                          None if skip is None else skip.float(), start, end, fin, 1.0, return_features)
        torch.cuda.synchronize()
        return out
    return layers, lat, noise, layer_in, skip, features_in, call


@pytest.mark.parametrize("c", RANGES, ids=[case_id(c) for c in RANGES])
def test_generator_chain_link_by_link(dev, sms, dt, c):
    name, start, end, feat = c
    ch = chain(name, dt, dev)
    B, tdt = ch.B, dt[1]
    nb = 1 if RANGES.index(c) % 2 == 0 else B
    layers, lat, noise, layer_in, skip, features_in, call = run_case(ch, start, end, feat, nb, 100 + RANGES.index(c))
    early, out_feat, out_rgb, outs = call(True)
    assert early == (layers[-1] < ch.n)
    # ---- every conv, from the observed output of the one before
    executed = [i for k in layers for i in convs_of(k)]
    for i in executed:
        cv = ch.conv[i]
        s = ch.style(cv, lat[:, i])
        if i == 0:
            x16 = handoff(ch.const.expand(B, -1, -1, -1), s, tdt)          # the broadcast constant input
        elif features_in is not None and features_in[i] is not None:
            x16 = handoff(features_in[i], s, tdt)                          # FSE insert_feature (alpha = 1)
        elif i == executed[0]:
            x16 = handoff(layer_in, s, tdt)                                # layer_in of start_layer
        else:
            x16 = handoff(outs[i].double(), s, tdt)                        # the 16-bit handoff of conv i - 1
        what = f"conv {i} ({'up' if cv['up'] else 'plain'}, {x16.shape[1]}->{cv['w'].shape[0]} at {x16.shape[2]}^2)"
        assert_exact_accumulator(cv, x16, tdt, what)
        acc = accumulate(cv, x16)
        bad, msg = check_conv(cv, acc, s, noise[i].double(), outs[i + 1].double())
        assert bad == 0, f"{what}: {msg}"
    # ---- fused ToRGB partials + rgb_combine, layer by layer from the observed features
    prev = skip
    err = None if skip is None else torch.zeros_like(skip)
    for k in layers:
        ic = 0 if k == 0 else 2 * k
        rg = ch.rgb[k]
        a = outs[ic + 1].double()
        cin, cout, r, _, _ = conv_shape(ic, ch.cm)
        n_tile, n_nt = plan(cin, cout, r, B, 0, dt[0])
        if sms == SMS_NAMED:
            assert n_nt == n_tiles_named(cout, r, B), (k, n_tile, n_nt)
        s_rgb = ch.style(rg, lat[:, 2 * k + 1])
        w = rg["m"][None] * s_rgb[:, None, :]                              # fl(fl(w1 / sqrt(cin)) * s): exact
        assert torch.equal(f32(w), w)
        ref = torch.einsum("bchw,bjc->bjhw", a, w) + rg["bias"].view(1, 3, 1, 1)
        mag = torch.einsum("bchw,bjc->bjhw", a.abs(), w.abs()) + rg["bias"].abs().view(1, 3, 1, 1)
        # each partial: two fmaf chains of max(n_tile / 2, 32) products and their sum; then the bias, the n_nt
        # partials and the four up taps are added in fp32, one rounding each
        coef = (max(n_tile // 2, 32) + n_nt + 4) * U
        if prev is not None:
            ref = ref + up2(prev, rg["upk"])
            mag = mag + up2(prev.abs(), rg["upk"].abs())
            bound = coef * mag + up2(err, rg["upk"].abs())
        else:
            bound = coef * mag
        prev, err = ref, bound
    got = out_rgb.double()
    assert not (got - prev).abs().gt(err).any(), first_bad(got, prev, err, f"rgb of layer {layers[-1]} "
                                                                         f"({n_nt} N-tile partials)")
    # ---- the production epilogue variants give the same bits
    early2, out_feat2, out_rgb2, outs2 = call(False)
    assert early2 == early and outs2 is None
    assert torch.equal(out_rgb2, out_rgb), "out_rgb differs between the epilogue variants"
    if early:
        assert torch.equal(out_feat2, outs[executed[-1] + 1]), "out_feature differs from the observed feature"
        assert torch.equal(out_feat, out_feat2), "out_feature is not written when return_features is on"


def test_one_ulp_change_of_a_handed_off_activation_fails_the_check(dev, dt):
    """Sensitivity of the link check: move one 16-bit input element of a conv by one ulp (into a channel and pixel
    the conv reads) and the observed output no longer passes."""
    ch = chain("g16_D512_cm2", dt, dev)
    layers, lat, noise, _, _, _, call = run_case(ch, 0, 8, None, ch.B, 5)
    _, _, _, outs = call(True)
    for i in (2, 3, 4):                    # plain conv from the up-conv's handoff, up-conv from the plain one's, ...
        cv = ch.conv[i]
        s = ch.style(cv, lat[:, i])
        x16 = handoff(outs[i].double(), s, dt[1])
        bad, msg = check_conv(cv, accumulate(cv, x16), s, noise[i].double(), outs[i + 1].double())
        assert bad == 0, msg
        o, c, ty, tx = [int(v) for v in cv["w"].nonzero()[0]]
        inner = torch.zeros_like(x16[0, c], dtype=torch.bool)
        inner[1:-1, 1:-1] = True                                            # every tap lands inside the image
        ys, xs = ((x16[0, c] > 0) & inner).nonzero()[0].tolist()
        y = x16.clone()
        y[0, c, ys, xs] += lsb16(y[0, c, ys, xs], dt[1])                # the next 16-bit value up
        assert float(y[0, c, ys, xs].to(dt[1]).double()) == float(y[0, c, ys, xs])
        bad, _ = check_conv(cv, accumulate(cv, y), s, noise[i].double(), outs[i + 1].double())
        assert bad > 0, f"conv {i}: a one-ulp change of input ({c}, {ys}, {xs}) went unnoticed"

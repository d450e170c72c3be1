"""Exact-arithmetic tests of the SIMT kernels of SEAN (csrc/hf_sean.cu) and of CtrlHair's shape adaptor outside its
split-K GEMM (csrc/hf_shape.cu), through the C ABI so that the test controls every operand, pointer and shape.

Operands are small integers or dyadic values, so every fp32 intermediate is exact.  The reference is float64 torch on
the CPU, rounded ONCE to the output type; `r16` asserts that it is exact in fp32 first.  Outputs must then match bit for
bit: a misplaced tap, label, channel, pixel or rounding changes the result.  Lookup sums are kept below 256 in
magnitude where the output is 16-bit, so that they are exact in bf16 too and no rounding can hide a wrong entry.

The library is built without fast math: `/`, `1/x` and `sqrtf` are IEEE operations, so the LayerNorm statistics are
emulated in numpy float32 bit for bit.  Where exact operands cannot avoid a rounding (tanhf, LeakyReLU ahead of the
RGB convolution, an arbitrary LayerNorm gamma) the bound is stated beside the operation, as
"1 ulp + k * 2^-24 * sum|terms|".

Each case id names the path it takes: the (res, channels) of the decoder layer it serves, the pixel / channel tiles,
the table or NULL path, the LayerNorm block count G, the grid tail."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.gpu_util import enc_dtype_name

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

EPS = 2.0 ** -24                        # unit roundoff of fp32
N_CLASSES, STYLE = 19, 512
SLOPE32 = float(np.float32(0.2))        # 0.2f, the LeakyReLU slope the kernels multiply by


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
    return (_lib.HF_F16, torch.float16) if enc_dtype_name() == "fp16" else (_lib.HF_BF16, torch.bfloat16)


def call(name, *args):
    """Calls the C entry point with every tensor argument passed as its device pointer.  The tensors stay referenced
    until the launch is queued: a temporary freed earlier could be handed to the next operand by the caching
    allocator and overwritten before the kernel reads it."""
    from hairfastgan_b200 import _lib
    _lib.check(getattr(_lib.lib(), name)(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]), name)


def stream():
    from hairfastgan_b200 import _lib
    return _lib.stream_ptr()


# ------------------------------------------------------------------------------------------------ operands, checks
def ints(g, shape, lo, hi):
    """Seeded integers in [lo, hi] as float64."""
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def pick(g, shape, values):
    """Seeded draws from a list of (dyadic) values as float64."""
    v = torch.tensor(values, dtype=torch.float64)
    return v[torch.randint(0, len(values), shape, generator=g)]


def dev32(x, dev):
    return x.float().contiguous().to(dev)


def dev16(x, tdt, dev):
    """float64 tensor, exact in the 16-bit type -> the device tensor the kernel reads (same layout)."""
    y = x.to(tdt).contiguous().to(dev)
    assert torch.equal(y.cpu().double(), x), "operand not exact in 16 bits"
    return y


def r16(ref, tdt):
    """float64 reference rounded once to the 16-bit type; it must be exact in fp32 (no double rounding)."""
    f = ref.float()
    assert torch.equal(f.double(), ref), "reference not exact in fp32: the bit-exact comparison would be invalid"
    return f.to(tdt).double()


def ulp(ref, mant, emin):
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin)))
    return torch.pow(torch.tensor(2.0, dtype=torch.float64), e - mant)


def ulp16(ref, tdt):
    return ulp(ref, *((10, -14) if tdt == torch.float16 else (7, -126)))


def ulp32(ref):
    return ulp(ref, 23, -126)


def assert_equal(got, ref, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    bad = (got != ref) & ~(torch.isnan(got) & torch.isnan(ref))
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail(f"{what}: {int(bad.sum())} of {ref.numel()} values differ; first at {i}: got {float(got[i])!r}, "
                    f"expected {float(ref[i])!r}")


def assert_within(got, ref, bound, what):
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    over = ~((got - ref).abs() <= bound)
    if over.any():
        i = tuple(int(v) for v in over.nonzero()[0])
        pytest.fail(f"{what}: {int(over.sum())} of {ref.numel()} values out of bound; first at {i}: got "
                    f"{float(got[i])!r}, expected {float(ref[i])!r}, bound {float(bound[i]):.3g}")


def gather_taps(L, table, k, stride, pad_label):
    """sum over the k x k taps inside the map of table[tap][L(source)] -> [R, R, C] float64.  L [S, S] long; table
    [k*k][labels][C]; source (stride*y - 1 + ky, stride*x - 1 + kx); outside sources read `pad_label`, a zero row."""
    S = L.shape[0]
    R = (S + 2 - k) // stride + 1
    tab = torch.cat([table, torch.zeros(table.shape[0], 1, table.shape[2], dtype=table.dtype)], 1)
    Lp = F.pad(L, (1, 1, 1, 1), value=pad_label)
    out = torch.zeros(R, R, table.shape[2], dtype=torch.float64)
    for ky in range(k):
        for kx in range(k):
            idx = Lp[ky:ky + stride * (R - 1) + 1:stride, kx:kx + stride * (R - 1) + 1:stride]
            out += tab[ky * k + kx][idx]
    return out


# ================================================================================================ SEAN
LEVELS = [8, 16, 32, 64, 128, 256]


@pytest.mark.parametrize("size", [256, 64], ids=["size256_r8to256", "size64_r2to64"])
def test_sean_labels_six_levels_bit_exact(dev, size):
    """L_R[y, x] = label[y*size/R, x*size/R] for R = size/32 .. size, concatenated; every entry written."""
    g = torch.Generator().manual_seed(size)
    lab = torch.randint(0, N_CLASSES, (size, size), generator=g)
    lab[::32, ::32] = torch.arange((size // 32) ** 2).view(size // 32, size // 32) % N_CLASSES   # distinct per block
    levels = [size >> (5 - i) for i in range(6)]
    maps = torch.full((sum(r * r for r in levels),), 77, dtype=torch.int8, device=dev)
    bad = torch.full((1,), -5, dtype=torch.int32, device=dev)
    call("hf_sean_labels", lab.to(dev), maps, bad, size, stream())
    ref = torch.cat([lab[::size // r, ::size // r].reshape(-1) for r in levels]).to(torch.int8)
    assert_equal(maps.cpu(), ref, f"label maps of size {size}")
    assert int(bad) == 0


def test_sean_labels_out_of_range_values_map_to_0_and_are_counted(dev):
    size = 256
    g = torch.Generator().manual_seed(3)
    lab = torch.randint(1, N_CLASSES, (size, size), generator=g)
    bads = [-1, 19, 127, 2 ** 40, -2 ** 40, 255]
    pos = [(0, 0), (0, 255), (255, 0), (255, 255), (8, 40), (1, 3), (31, 32), (128, 128), (200, 7), (7, 200)]
    for k, (y, x) in enumerate(pos):
        lab[y, x] = bads[k % len(bads)]
    maps = torch.full((sum(r * r for r in LEVELS),), 77, dtype=torch.int8, device=dev)
    bad = torch.full((1,), -5, dtype=torch.int32, device=dev)
    call("hf_sean_labels", lab.to(dev), maps, bad, size, stream())
    clean = torch.where((lab >= 0) & (lab < N_CLASSES), lab, 0)
    ref = torch.cat([clean[::size // r, ::size // r].reshape(-1) for r in LEVELS]).to(torch.int8)
    assert_equal(maps.cpu(), ref, "label maps with out-of-range values")
    assert int(bad) == len(pos)
    assert int(ref[:64].eq(0).sum()) >= 1                    # (0, 0) is on every level


# ------------------------------------------------------------------------------------------------ one-hot conv lookup
# (res, channels) of SPADEGenerator.fc and of every SPADE.mlp_shared level decode runs
ONEHOT = [("fc", 8, 1024)] + [("mlp_shared", r, 128) for r in LEVELS]


@pytest.mark.parametrize("name,res,c", ONEHOT, ids=[f"{n}_r{r}_c{c}" for n, r, c in ONEHOT])
def test_sean_onehot_conv_bit_exact(dev, dt, name, res, c):
    """y = act(bias + sum over inside taps of table[tap][L][c]); integer table in [-8, 8] and bias in [-16, 16]: the
    sums stay below 256, exact in either 16-bit type."""
    g = torch.Generator().manual_seed(res * 10 + c)
    L = torch.randint(0, N_CLASSES, (res, res), generator=g)
    L[0, 0], L[0, -1], L[-1, 0], L[-1, -1] = 18, 1, 17, 2                 # corners: distinct labels
    L[0, 1:-1], L[1:-1, -1] = 3, 15                                      # two whole borders of one label
    table = ints(g, (9, N_CLASSES, c), -8, 8)
    bias = ints(g, (c,), -16, 16)
    s = gather_taps(L, table, 3, 1, N_CLASSES)
    Ld, td, bd = L.to(torch.int8).to(dev), dev32(table, dev), dev32(bias, dev)
    for use_bias in (False, True):
        for act in (0, 3):
            ref = s + (bias if use_bias else 0.0)
            if act == 3:
                ref = ref.clamp_min(0)
            y = torch.full((res, res, c), float("nan"), dtype=dt[1], device=dev)
            call("hf_sean_onehot_conv", Ld, td, bd if use_bias else None, act,
                 y, res, c, dt[0], stream())
            assert_equal(y.cpu().double(), r16(ref, dt[1]), f"bias {use_bias} act {act}")


# ------------------------------------------------------------------------------------------------ ACE style tables
# n2 = 2C of the 15 RGB ACEs in decode order: head_0, G_middle_0, G_middle_1 (C 1024), up_0 (1024, 1024, 512),
# up_1 (512, 512, 256), up_2 (256, 256, 128)
RGB_N2 = [2048] * 6 + [2048, 2048, 1024, 1024, 1024, 512, 512, 512, 256]


def style_operands(g, n2s):
    """Per ACE: integer fc_w in {-1, 0, 1} [19][512][512], fc_b in [-8, 8], tw in {-1, 0, 1} [9*n2][512]: mu <= 2056
    and every T < 2^21, all partial sums exact."""
    return [(torch.randint(-1, 2, (N_CLASSES, STYLE, STYLE), generator=g, dtype=torch.int8),
             ints(g, (N_CLASSES, STYLE), -8, 8),
             torch.randint(-1, 2, (9 * n2, STYLE), generator=g, dtype=torch.int8)) for n2 in n2s]


def style_reference(ops, n2s, code):
    """mu[a][j] = max(fc_w[a][j] . code_j + fc_b[a][j], 0) and T[a][j][tap][n] = tw[a][tap*n2 + n] . mu[a][j]."""
    mus, Ts = [], []
    for (fw, fb, tw), n2 in zip(ops, n2s):
        mu = (torch.bmm(fw.double(), code.unsqueeze(2)).squeeze(2) + fb).clamp_min(0)
        mus.append(mu)
        Ts.append((tw.double() @ mu.t()).view(9, n2, N_CLASSES).permute(2, 0, 1).contiguous())
    return mus, Ts


def run_style_tables(dev, ic, mc, dops, n2s):
    from hairfastgan_b200 import _lib
    n = len(n2s)
    tables = [torch.full((N_CLASSES, 9, n2), float("nan"), device=dev) for n2 in n2s]
    mu = torch.full((n, N_CLASSES, STYLE), float("nan"), device=dev)
    arr = (_lib.hf_sean_ace_tables * n)()
    for a, ((fw, fb, tw), t, n2) in enumerate(zip(dops, tables, n2s)):
        arr[a] = _lib.hf_sean_ace_tables(fw.data_ptr(), fb.data_ptr(), tw.data_ptr(), t.data_ptr(), n2)
    rc = _lib.lib().hf_sean_style_tables(ic.data_ptr(), mc.data_ptr(), arr, n, mu.data_ptr(), stream())
    return rc, mu, tables


def test_sean_style_tables_every_ace_boundary_and_mean_code_fallback(dev):
    """All 15 RGB ACEs of decode in one call (the CTA -> ACE search crosses every block_begin), then 16 (the maximum)
    and 1; 17 is rejected.  image_code rows: random integers; row 3 zero but for element 511 (the image code);
    row 5 all -0.0 and row 9 all +0.0 (the mean code: torch.all(code == 0) in the reference); row 7 with a NaN (the
    image code: every dot product is NaN, and the kernel's ReLU, fmaxf, returns 0 for it).  The tables start as NaN:
    a CTA that writes nothing leaves NaN behind."""
    g = torch.Generator().manual_seed(15)
    ic = ints(g, (N_CLASSES, STYLE), -4, 4)
    ic[3] = 0.0
    ic[3, 511] = 2.0
    ic[5] = -0.0
    ic[9] = 0.0
    ic[7, 100] = float("nan")
    mc = ints(g, (N_CLASSES, STYLE), -4, 4)
    assert bool(torch.signbit(ic[5]).all())
    code = torch.where(torch.all(ic == 0, dim=1, keepdim=True), mc, ic)
    assert torch.equal(code[5], mc[5]) and torch.equal(code[9], mc[9]) and torch.equal(code[3], ic[3])
    n2s = RGB_N2 + [8]
    ops = style_operands(g, n2s)
    mus, Ts = style_reference(ops, n2s, torch.nan_to_num(code, nan=0.0))
    for mu, T in zip(mus, Ts):                                   # NaN row: fmaxf(NaN, 0) = 0 for every row of mu_7
        mu[7] = 0.0
        T[7] = 0.0
    mean7, _ = style_reference(ops[:1], n2s[:1], mc)
    assert bool((mean7[0][7] > 0).any()), "the mean code would give the NaN row a non-zero mu: the case checks nothing"
    icd, mcd = dev32(ic, dev), dev32(mc, dev)
    dops = [(fw.float().to(dev), dev32(fb, dev), tw.float().to(dev)) for fw, fb, tw in ops]
    for n in (15, 16, 1):
        rc, mu, tables = run_style_tables(dev, icd, mcd, dops[:n], n2s[:n])
        assert rc == 0
        for a in range(n):
            what = f"n_ace {n}, ACE {a} (n2 {n2s[a]})"
            assert_equal(mu[a].cpu().double(), mus[a], what + " mu")
            assert_equal(tables[a].cpu().double(), Ts[a], what + " table")
    from hairfastgan_b200 import _lib
    rc, mu, _ = run_style_tables(dev, icd, mcd, dops[:16] + dops[:1], n2s[:16] + n2s[:1])
    assert rc == -1 and b"17 ACE layers (1..16)" in _lib.lib().hf_last_error()


# ------------------------------------------------------------------------------------------------ ACE apply
# (res, C) of the seven blocks' ACEs: head_0 .. up_3
ACE_SHAPES = [(8, 1024), (16, 1024), (32, 1024), (32, 512), (64, 512), (64, 256), (128, 256), (128, 128), (256, 128),
              (256, 64)]


@pytest.mark.parametrize("res,c", ACE_SHAPES,
                         ids=[f"r{r}_c{c}_ptiles{r * r // 32}_ctiles{c // 64}" for r, c in ACE_SHAPES])
def test_sean_ace_apply_bit_exact(dev, dt, res, c):
    """v = (x + n[h, w] * noise_var) * bn_scale + bn_shift with n[h, w] = noise[w*res + h]; out = v (1 + g) + b with
    g / b = gamma_beta[c / C + c][p] (+ the 9-tap gather of T on the table path); LeakyReLU(0.2).  Dyadic operands:
    v, g, b and out are exact in fp32; the LeakyReLU product is fl32(t * 0.2f), which the float64 product (exact:
    24 x 14 significant bits) rounded to fp32 reproduces.  gamma_beta differs per (channel, pixel), so a pixel or
    channel taken from the wrong place in the shared-memory transpose changes the result; an impulse noise at
    (h, w) = (0, 1) pins the transpose of the noise."""
    g = torch.Generator().manual_seed(res * 7 + c)
    hw = res * res
    x = ints(g, (hw, c), -8, 8) / 4
    noise = ints(g, (hw,), -4, 4) / 4
    nv = pick(g, (c,), [-1.0, -0.5, 0.5, 1.0, 2.0])
    sc = pick(g, (c,), [0.5, 1.0, 2.0])
    sh = ints(g, (c,), -4, 4) / 4
    gb = ints(g, (2 * c, hw), -8, 8) / 16
    T = ints(g, (N_CLASSES, 9, 2 * c), -4, 4) / 32
    L = torch.randint(0, N_CLASSES, (res, res), generator=g)
    tsum = gather_taps(L, T.permute(1, 0, 2), 3, 1, N_CLASSES).reshape(hw, 2 * c)
    xd = dev16(x, dt[1], dev)
    opsd = [dev32(v, dev) for v in (nv, sc, sh, gb)]
    Td, Ld = dev32(T, dev), L.to(torch.int8).to(dev)
    impulse = torch.zeros(hw, dtype=torch.float64)
    impulse[1 * res + 0] = 1.0                                                # noise[w*res + h] at h = 0, w = 1
    for noise_kind, nz in (("random", noise), ("impulse_h0_w1", impulse)):
        n_hw = nz.view(res, res).t().reshape(hw, 1)                           # n[h, w] = noise[w, h]
        v = (x + n_hw * nv) * sc + sh
        nzd = dev32(nz, dev)
        for use_table in (True, False):
            gg = gb.t() + (tsum if use_table else 0.0)
            t = v * (1 + gg[:, :c]) + gg[:, c:]
            for lrelu in (0, 1):
                what = f"noise {noise_kind} table {use_table} lrelu {lrelu}"
                want = r16(t, dt[1])                          # asserts t exact in fp32
                if lrelu:
                    want = torch.where(t < 0, (t * SLOPE32).float().double(), t).float().to(dt[1]).double()
                y = torch.full((hw, c), float("nan"), dtype=dt[1], device=dev)
                call("hf_sean_ace_apply", xd, nzd, *opsd,
                     Td if use_table else None, Ld, lrelu, y, res, c, dt[0], stream())
                assert_equal(y.cpu().double(), want, what)


# ------------------------------------------------------------------------------------------------ conv_img + tanh
def conv_img_ref(x, w, b):
    """[R*R, C] (LeakyReLU already applied), [3][C][3][3], [3] -> [3, R, R] float64 pre-activation."""
    res = int(round(x.shape[0] ** 0.5))
    return F.conv2d(x.t().reshape(1, -1, res, res), w, b, padding=1)[0]


def run_conv_img(dev, dt, xd, w, b, res, c):
    y = torch.full((3, res, res), float("nan"), device=dev)
    call("hf_sean_conv_img", xd, dev32(w, dev), dev32(b, dev), y, res, c,
         dt[0], stream())
    return y.cpu().double()


def tanh_bound(acc, err):
    """tanhf is within 2 ulps (CUDA's documented bound); tanh' <= 1 carries the accumulator's error."""
    return 2 * ulp32(torch.tanh(acc)) + err


# (res, C): the decoder's 256^2 x 64, the smallest C and the largest C the shared-memory weights hold; 33^2 and 17^2
# leave a partial last CTA
CONV_IMG = [(256, 64), (33, 8), (17, 256)]


@pytest.mark.parametrize("res,c", CONV_IMG, ids=[f"r{r}_c{c}" + ("_grid_tail" if r * r % 256 else "")
                                                 for r, c in CONV_IMG])
def test_sean_conv_img(dev, dt, res, c):
    """tanh(b + sum over inside taps and channels of w * lrelu(x)).  x >= 0: LeakyReLU is the identity and the
    accumulator (multiples of 2^-8 below 2^10) is exact, so only tanhf rounds.  x of both signs: lrelu(x) =
    fl32(0.2f x) rounds once, and each of the 9C + 1 accumulator additions (or fmaf) once: k = 9C + 2 roundoffs of
    sum|terms|.  Impulse weights, one (channel, tap) per call with a distinct weight per output, pin the index of
    every output, channel and tap: x differs per (pixel, channel)."""
    g = torch.Generator().manual_seed(res + c)
    hw = res * res
    w = ints(g, (3, c, 3, 3), -2, 2) / 64
    b = ints(g, (3,), -4, 4) / 8
    xp = ints(g, (hw, c), 0, 4) / 4
    acc = conv_img_ref(xp, w, b)
    got = run_conv_img(dev, dt, dev16(xp, dt[1], dev), w, b, res, c)
    assert_within(got, torch.tanh(acc), tanh_bound(acc, 0.0), "x >= 0")
    xs = ints(g, (hw, c), -8, 8) / 4
    a = torch.where(xs < 0, xs * SLOPE32, xs)                                     # exact in float64
    acc = conv_img_ref(a, w, b)
    terms = conv_img_ref(a.abs(), w.abs(), b.abs())
    got = run_conv_img(dev, dt, dev16(xs, dt[1], dev), w, b, res, c)
    assert_within(got, torch.tanh(acc), tanh_bound(acc, (9 * c + 2) * EPS * terms), "x of both signs")
    p = torch.arange(hw, dtype=torch.float64).view(hw, 1)
    xi = ((p * 5 + torch.arange(c, dtype=torch.float64) * 3) % 16) / 4                  # 0 .. 3.75, >= 0
    xid = dev16(xi, dt[1], dev)
    zero_b = torch.tensor([0.25, -0.5, 0.0], dtype=torch.float64)
    for ch in sorted({0, 7, c // 2 + 1, c - 8, c - 1}):
        for tap in range(9):
            wi = torch.zeros(3, c, 3, 3, dtype=torch.float64)
            wi[:, ch, tap // 3, tap % 3] = torch.tensor([1.0, -2.0, 3.0]) / 8
            acc = conv_img_ref(xi, wi, zero_b)
            got = run_conv_img(dev, dt, xid, wi, zero_b, res, c)
            assert_within(got, torch.tanh(acc), tanh_bound(acc, 0.0), f"impulse channel {ch} tap {tap}")


# ------------------------------------------------------------------------------------------------ class means
# (name, B, C, HW, label stride)
CLASS_MEANS = [("b3_c5_hw1000_stride1100", 3, 5, 1000, 1100), ("b2_c512_hw16384_stride21844", 2, 512, 16384, 21844),
               ("b1_c3_hw1_stride1", 1, 3, 1, 1)]


@pytest.mark.parametrize("name,b,c,hw,stride", CLASS_MEANS, ids=[m[0] for m in CLASS_MEANS])
def test_sean_class_means_bit_exact(dev, name, b, c, hw, stride):
    """codes[b][j][c] = (sum of tanhf(y) over the class-j pixels) / count, 0 for an absent class.  y in {-20, 0, 20}:
    tanhf gives exactly -1, 0 or 1, so the sums are integers and the IEEE quotient is float64 s / n rounded to fp32
    (an innocuous double rounding: 53 >= 2 * 24 + 2).  Classes 4 and 17 are absent, class 11 is at a single pixel
    per sample, labels outside 0..18 are skipped, and the pixels between hw and the label stride (class 4) are never
    read."""
    g = torch.Generator().manual_seed(hw + c)
    y = pick(g, (b, c, hw), [-20.0, 0.0, 20.0])
    present = torch.tensor([j for j in range(N_CLASSES) if j not in (4, 11, 17)] + [-1, 19, 100, -128])
    lab = present[torch.randint(0, len(present), (b, hw), generator=g)]
    for i in range(b):
        lab[i, (37 * i + 5) % hw] = 11
    buf = torch.full((b, stride), 4, dtype=torch.int64)
    buf[:, :hw] = lab
    s = torch.zeros(b, N_CLASSES, c, dtype=torch.float64)
    n = torch.zeros(b, N_CLASSES, 1, dtype=torch.float64)
    for j in range(N_CLASSES):
        m = (lab == j).double()
        s[:, j] = torch.einsum("bcp,bp->bc", torch.tanh(y).round(), m)
        n[:, j, 0] = m.sum(1)
    ref = torch.where(n > 0, s / n.clamp_min(1), 0.0).float().double()
    assert bool((n[:, 11] == 1).all()) and bool((n[:, 4] == 0).all()) and bool((n[:, 17] == 0).all())
    codes = torch.full((b, N_CLASSES, c), float("nan"), device=dev)
    labd = buf.to(torch.int8).reshape(-1).to(dev)
    call("hf_sean_class_means", dev32(y, dev), labd, stride, codes, b, c, hw,
         stream())
    assert_equal(codes.cpu().double(), ref, name)


# ================================================================================================ shape adaptor
def test_shape_labels_rewrite_and_count(dev):
    """255 -> 19 in the caller's mask; 0..19 kept; everything else counted and mapped to 19 in the labels (the mask
    keeps it)."""
    n = 65536 + 37
    g = torch.Generator().manual_seed(19)
    mask = torch.randint(0, 20, (n,), generator=g)
    mask[torch.randint(0, n, (300,), generator=g)] = 255
    bads = torch.tensor([20, -1, 254, 256, 2 ** 40, -2 ** 40, 127, 128])
    where = torch.randperm(n, generator=g)[:50]
    where[0], where[1] = 0, n - 1
    mask[where] = bads[torch.arange(50) % len(bads)]
    md = mask.to(dev)
    L = torch.full((n,), -7, dtype=torch.int8, device=dev)
    bad = torch.full((1,), -5, dtype=torch.int32, device=dev)
    call("hf_shape_labels", md, L, bad, n, stream())
    want_mask = torch.where(mask == 255, 19, mask)
    ok = (want_mask >= 0) & (want_mask <= 19)
    assert torch.equal(md.cpu(), want_mask)
    assert_equal(L.cpu(), torch.where(ok, want_mask, 19).to(torch.int8), "labels")
    assert int(bad) == 50 == int((~ok).sum())


# ------------------------------------------------------------------------------------------------ stride-2 lookup
ONEHOT_S2 = [(128, 32), (7, 8), (9, 64), (1, 8)]


@pytest.mark.parametrize("res,c", ONEHOT_S2, ids=[f"r{r}_c{c}" for r, c in ONEHOT_S2])
def test_shape_onehot_s2_bit_exact(dev, dt, res, c):
    """y[oy, ox] = cmap + sum over the 4 x 4 taps inside the (2 res)^2 map of table[tap][L(2oy - 1 + ky, 2ox - 1 +
    kx)]; label 19's rows are non-zero here, so the kernel's indexing, not the model's zero rows, is checked.  Integer
    table in [-8, 8] and cmap in [-32, 32]: sums below 256, exact in either 16-bit type.  A random map, then impulse
    labels on the stride-2 borders (rows / columns 0, 1, S-2, S-1) over a map of label 19."""
    S = 2 * res
    g = torch.Generator().manual_seed(res * 100 + c)
    table = ints(g, (16, 20, c), -8, 8)
    table[:, 19] = ints(g, (16, c), 1, 8)
    cmap = ints(g, (res * res, c), -32, 32)
    imp = torch.full((S, S), 19, dtype=torch.int64)
    for k, (yy, xx) in enumerate([(0, 0), (0, S - 1), (S - 1, 0), (S - 1, S - 1), (1, 1), (0, 1), (1, 0),
                                  (S - 2, S - 1), (S - 1, S - 2), (0, S // 2), (S // 2, 0)]):
        imp[min(yy, S - 1), min(xx, S - 1)] = k % 19
    td, cd = dev32(table, dev), dev32(cmap, dev)
    for kind, L in (("random", torch.randint(0, 20, (S, S), generator=g)), ("border_impulses", imp)):
        ref = cmap.view(res, res, c) + gather_taps(L, table, 4, 2, 20)
        y = torch.full((res, res, c), float("nan"), dtype=dt[1], device=dev)
        call("hf_shape_onehot_s2", L.to(torch.int8).to(dev), td, cd, y,
             res, c, dt[0], stream())
        assert_equal(y.cpu().double(), r16(ref, dt[1]), kind)


# ------------------------------------------------------------------------------------------------ LayerNorm + LeakyReLU
def ln_blocks(n8, sms):
    return max(1, min(2 * sms, n8 // 512))


def ln_emulated(d, S, n, gamma, beta, slope, divisor):
    """The kernel's fp32 arithmetic in numpy float32: inv = 1 / (sqrtf(S / divisor) + 1e-5f), a = fl(d * inv),
    t = fl(a * gamma + beta) (gamma a power of two: the product is exact, so fmaf or not gives the same), LeakyReLU
    t * slope.  d = x - mean exact, S the exact sum of d^2; returns (a * gamma as float64, t_lrelu as float32)."""
    f = np.float32
    inv = f(1) / (np.sqrt(f(S) / f(divisor)) + f(1e-5))
    a = d.astype(np.float32) * inv
    ag = a.astype(np.float64) * gamma
    t = (ag + beta).astype(np.float32)
    return ag, np.where(t > 0, t, t * f(slope))


# (name, pixels, channels, mean, d_max): pixels * channels a power of two
LAYER_NORM = [("g1_p64_c32", 64, 32, 3, 2), ("g1_p256_c8", 256, 8, -5, 3), ("g2_p4_c2048", 4, 2048, 1, 2),
              ("g16_p1024_c64", 1024, 64, 0, 2), ("cap_tail_p65536_c32", 65536, 32, 1, 2),
              ("g1_mean_over_std_p64_c64", 64, 64, 2048, 2)]


@pytest.mark.parametrize("name,pixels,c,mean,dmax", LAYER_NORM, ids=[v[0] for v in LAYER_NORM])
def test_shape_layer_norm_lrelu_bit_exact(dev, sms, dt, name, pixels, c, mean, dmax):
    """(x - mean) / (unbiased std + 1e-5) * gamma[c] + beta[c], LeakyReLU(0.2), over the whole sample.  x = mean + d
    with integer d of zero sum (the pairs e, -e shuffled), n a power of two: the mean and the centred sum of squares
    are exact, and inv is emulated in float32 bit for bit; gamma in {0.5, 1, 2, 4} and dyadic beta make the output
    bit-exact.  The shapes reach G = 1, an intermediate G and the cap of 2 SMs (derived from hf_sm_count) with a
    chunk tail.  On the samples of up to 8192 values the same emulation with a biased variance (S / n) must disagree
    with the kernel."""
    n = pixels * c
    n8 = n // 8
    G = ln_blocks(n8, sms)
    chunk8 = -(-n8 // G)
    if name.startswith("g1_"):
        assert G == 1
    elif name.startswith("cap"):
        assert G == 2 * sms and G * chunk8 > n8, (G, chunk8, n8)
    else:
        assert 1 < G < 2 * sms and G == int(name[1:name.index("_")])
    g = torch.Generator().manual_seed(n + c)
    step = 16 if mean > 1000 else 1                          # bf16 spacing at 2048
    e = torch.randint(-dmax, dmax + 1, (n // 2,), generator=g) * step
    d = torch.cat([e, -e])[torch.randperm(n, generator=g)].double()
    x = (mean + d).view(pixels, c)
    S = float((d * d).sum())
    assert abs(mean) * n < 2 ** 24 and S < 2 ** 24
    from hairfastgan_b200 import _lib
    nbytes = _lib.lib().hf_shape_layer_norm_workspace_bytes(n)
    assert nbytes == 2 * G * 4
    ws = torch.full((2 * G,), float("nan"), device=dev)
    xd = dev16(x, dt[1], dev)
    gamma = pick(g, (c,), [0.5, 1.0, 2.0, 4.0])
    beta = ints(g, (c,), -8, 8) / 8
    dv = d.view(pixels, c).numpy()

    def run(gm):
        y = torch.full((pixels, c), float("nan"), dtype=dt[1], device=dev)
        call("hf_shape_layer_norm_lrelu", xd, dev32(gm, dev), dev32(beta, dev),
             y, ws, pixels, c, 0.2, dt[0], stream())
        return y.cpu().double()

    got = run(gamma)
    gn, bn = gamma.numpy(), beta.numpy()
    _, want = ln_emulated(dv, S, n, gn, bn, 0.2, n - 1)
    assert_equal(got, torch.from_numpy(want).to(dt[1]).double(), f"{name} (G {G})")
    if n <= 8192:            # S / n moves the output by a relative 1 / 2n: visible in 16 bits for small samples only
        _, biased = ln_emulated(dv, S, n, gn, bn, 0.2, n)
        assert not torch.equal(got, torch.from_numpy(biased).to(dt[1]).double()), "a biased variance passes the test"
    # arbitrary gamma: a * gamma rounds (or fuses with + beta), then + beta and the slope product: each within
    # 2^-24 of |a gamma| + |t|; 1 ulp of the 16-bit store
    ga = torch.rand(c, generator=g, dtype=torch.float64).float().double() * 1.5 + 0.25
    ag, _ = ln_emulated(dv, S, n, ga.numpy(), bn, 0.2, n - 1)
    t = torch.from_numpy(ag) + beta
    ref = torch.where(t > 0, t, t * SLOPE32)
    bound = ulp16(ref, dt[1]) + 2 * EPS * (torch.from_numpy(ag).abs() + t.abs())
    assert_within(run(ga), ref, bound, f"{name} arbitrary gamma")


# ------------------------------------------------------------------------------------------------ logits + arg-max
def logits_ref(hair, face, table, bias):
    """[19, R, R] float64: conv 3x3 pad 1 of cat[face[:13], hair, face[13:]]; hair / face [R, R, 32]."""
    R = hair.shape[0]
    w = torch.zeros(N_CLASSES, 64, 3, 3, dtype=torch.float64)
    tw = table.view(N_CLASSES, 3, 3, 32).permute(0, 3, 1, 2)
    for j in range(N_CLASSES):
        if j == 13:
            w[j, 32:] = tw[j]
        else:
            w[j, :32] = tw[j]
    inp = torch.cat([face, hair], 2).permute(2, 0, 1).reshape(1, 64, R, R)
    return F.conv2d(inp, w, bias, padding=1)[0]


# (name, first, second): exact ties built on purpose
TIES = [("face2_face5", 2, 5), ("face12_hair13", 12, 13), ("hair13_face13_at14", 13, 14)]


@pytest.mark.parametrize("res", [256, 15, 1], ids=["r256", "r15_grid_tail", "r1"])
def test_shape_logits_argmax_exact_with_ties(dev, dt, res):
    """Integer table in [-4, 4] and bias, activations k/8: every logit is exact, so the labels must equal the float64
    argmax (first index on ties, as torch.argmax).  Random data (hair differs from face, so a hair channel at the
    wrong index fails), then exact ties: the two tied rows share table and bias (hair := face where the hair row is
    one of them) and get a boost that makes them the maximum at about half the pixels."""
    g = torch.Generator().manual_seed(res)
    hair = ints(g, (res, res, 32), -16, 16) / 8
    face = ints(g, (res, res, 32), -16, 16) / 8
    table = ints(g, (N_CLASSES, 9, 32), -4, 4)
    bias = ints(g, (N_CLASSES,), -32, 32)

    def run(hr, fc, tb, bs):
        out = torch.full((res * res,), -7, dtype=torch.int64, device=dev)
        call("hf_shape_logits_argmax", dev16(hr, dt[1], dev), dev16(fc, dt[1], dev),
             dev32(tb, dev), dev32(bs, dev), out, res, dt[0], stream())
        return out.cpu()

    lg = logits_ref(hair, face, table, bias)
    assert_equal(run(hair, face, table, bias), lg.argmax(0).reshape(-1), "random")
    for name, a, b in TIES:
        tb, bs = table.clone(), bias.clone()
        tb[b], bs[b] = tb[a], bs[a]
        hr = face.clone() if 13 in (a, b) else hair
        lg = logits_ref(hr, face, tb, bs)
        others = torch.cat([lg[:min(a, b)], lg[min(a, b) + 1:max(a, b)], lg[max(a, b) + 1:]]).amax(0)
        boost = float((others - lg[a]).median().ceil())
        bs[a] += boost
        bs[b] += boost
        lg = logits_ref(hr, face, tb, bs)
        assert torch.equal(lg[a], lg[b])
        top = lg.amax(0)
        assert res == 1 or float((lg[a] == top).double().mean()) > 0.2, "the tied pair is rarely the maximum"
        assert_equal(run(hr, face, tb, bs), lg.argmax(0).reshape(-1), f"tie {name}")

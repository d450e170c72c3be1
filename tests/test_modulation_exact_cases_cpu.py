"""CPU checks of the float32 emulation that tests/test_gpu_modulation_exact.py compares the modulation kernels with
(tests/modulation_exact_cases.py): its exact fmaf against Fraction, its operand designs, and the emulated kernels on
generic operands against the float64 oracle (oracle/modulation_oracle.py).  With float32 in place of the 16-bit type
the emulation must match the unrounded oracle to summation order, which ties it to HairFast's arithmetic (biased
variance, LayerNorm eps 1e-5, PixelNorm eps 1e-8); with 16-bit operands it matches the operand-rounded oracle to the
16-bit rounding level."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import modulation_oracle as O
from tests import modulation_exact_cases as X

f32 = np.float32


def exact_f32(a, b, c):
    return X.round_fraction_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def test_fmaf_matches_fraction_on_double_rounding_cases():
    """a b + c whose float64 sum lands exactly on a float32 midpoint while the exact value does not: rounding the
    float64 sum to float32 goes the wrong way, fmaf must not.  Then random operands across exponent ranges."""
    cases = [(64 * (1 + 2.0 ** -18), 1 - 2.0 ** -18, 2.0 ** 30 + 128),          # just below the midpoint, odd
             (64 * (1 + 2.0 ** -12), 1 - 2.0 ** -12 + 2.0 ** -24, 2.0 ** 30),   # just above the midpoint, even
             (-64 * (1 + 2.0 ** -12), 1 - 2.0 ** -12 + 2.0 ** -24, -2.0 ** 30)]
    a, b, c = (np.array(v, f32) for v in zip(*cases))
    assert all(np.float64(x) == y for x, y in zip(a, (v[0] for v in cases)))
    naive = (a.astype(np.float64) * b + c).astype(f32)
    want = np.array([exact_f32(*v) for v in zip(a, b, c)], f32)
    assert (naive != want).all()
    assert np.array_equal(X.fmaf(a, b, c), want)
    rng = np.random.default_rng(0)
    n = 4000
    a = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(f32)
    b = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(f32)
    c = (rng.standard_normal(n) * np.exp2(rng.integers(-40, 40, n))).astype(f32)
    want = np.array([exact_f32(*v) for v in zip(a, b, c)], f32)
    assert np.array_equal(X.fmaf(a, b, c), want)


def test_tree_sum_order():
    """The CTA sum is not a plain left-to-right sum: values chosen so that the butterfly order decides the result."""
    v = np.zeros((1, 256), f32)
    v[0, 0], v[0, 16], v[0, 1] = 2.0 ** 24, 1.0, 1.0
    # lane 0 + lane 16 = 2^24 + 1 -> 2^24 (tie to even); then + (lane 1 + lane 17 = 1) -> 2^24 + 1 -> 2^24
    assert X.tree_sum(v, np.ones(v.shape, bool), False) == f32(2.0 ** 24)
    assert v.astype(np.float64).sum() == 2.0 ** 24 + 2


@pytest.mark.parametrize("L", [1, 6, 17])
def test_pixel_x0_design(L):
    """UNIT columns normalise exactly (to integers over 2 or 4), ZERO columns stay zero, EPS_VISIBLE columns differ
    from the eps-free normalisation."""
    rng = np.random.default_rng(L)
    x = X.pixel_x0(rng, 2, L)
    kinds = X.column_kinds()
    y = X.pixel_norm(x.astype(f32), torch.bfloat16)
    unit = kinds == X.UNIT
    ms = (x[:, :, unit] ** 2).mean(1)
    assert np.array_equal(np.log2(ms) % 2, np.zeros_like(ms))                  # powers of 4
    assert np.array_equal(y[:, :, unit], x[:, :, unit] / np.sqrt(ms)[:, None])
    assert (y[:, :, kinds == X.ZERO] == 0).all()
    eps = kinds == X.EPS_VISIBLE
    xe = x[:, :, eps]
    ms = np.broadcast_to((xe ** 2).mean(1, keepdims=True), xe.shape)
    nz = ms > 0
    assert nz.any() and (np.abs(y[:, :, eps][nz]) < 0.9 * np.abs(xe[nz] / np.sqrt(ms[nz]))).any()


def chain_case(L, stacks, tdt, B=2):
    """Random operands of the chain (fc weights rounded to tdt) and the emulation's output and the oracle's 0.1 dt
    for them: (out, base + 0.1 dt, 0.1 dt).  Every 16th column of x0 is scaled by 1e-5, so that PixelNorm's 1e-8
    dominates its mean square."""
    g = torch.Generator().manual_seed(L)
    x0 = [torch.randn(B, L, 512, generator=g) for _ in range(stacks)]
    for x in x0:
        x[..., ::16] *= 1e-5
    base = torch.randn(B, L, 512, generator=g)
    gb = 0.3 * torch.randn(10 * stacks, B * L, 512, generator=g)
    fc_w = (torch.randn(stacks, 5, 512, 512, generator=g) / 512 ** 0.5).to(tdt).double()
    fc_b = 0.1 * torch.randn(stacks, 5, 512, generator=g)
    with X.generic_operands():
        got = X.chain([x.numpy() for x in x0], fc_w.numpy(), fc_b.numpy(), gb.numpy(), base.numpy(), tdt)
    dts = []
    for s in range(stacks):
        params = [{"fc.weight": fc_w[s, i], "fc.bias": fc_b[s, i]} for i in range(5)]
        gbs = [(gb[s * 10 + 2 * i].view(B, L, 512), gb[s * 10 + 2 * i + 1].view(B, L, 512)) for i in range(5)]
        dts.append(O.stack(x0[s], None, params, None if tdt == torch.float32 else tdt, gbs))
    dt = 0.1 * sum(dts)
    return torch.from_numpy(got).double(), base.double() + dt, dt


@pytest.mark.parametrize("L,stacks", [(1, 1), (6, 1), (18, 2)])
def test_chain_emulation_matches_oracle_in_float32(L, stacks):
    """With float32 in place of the 16-bit type every rounding to 16 bits is the identity, so the emulation must agree
    with the unrounded float64 oracle to summation order: max-abs over RMS of 0.1 dt below 5e-6 (measured 1.2e-6 to
    1.4e-6).  This ties the emulation, and through it the kernels, to HairFast's arithmetic.  In the emulation, a
    LayerNorm without eps gives 3e-5 or more here, an unbiased variance 3e-4 or more, and a PixelNorm eps of 1e-5 or
    none 9e-2 or more."""
    got, ref, dt = chain_case(L, stacks, torch.float32)
    err = float((got - ref).abs().max() / dt.pow(2).mean().sqrt())
    assert err < 5e-6, err


@pytest.mark.parametrize("tdt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("L,stacks", [(6, 1), (18, 2)])
def test_chain_emulation_matches_operand_rounded_oracle(tdt, L, stacks):
    """The same with 16-bit operands, against oracle.stack rounding the same operands: once an operand rounds the
    other way near a 16-bit boundary the following modules carry the 16-bit rounding level, so this holds only to the
    bound tests/test_gpu_modulation.py holds the kernel to (measured up to 1.3e-3 fp16 / 3.9e-3 bf16 at these
    seeds).  It checks the placement of the roundings, not the arithmetic between them."""
    got, ref, dt = chain_case(L, stacks, tdt)
    err = float((got - ref).abs().max() / dt.pow(2).mean().sqrt())
    assert err < (4e-3 if tdt == torch.float16 else 1.5e-2), err


def hidden_case(tdt):
    """Random operands of hidden and the layer-2 GEMM for Rotate's shapes; the gamma branch of module 0 has its first
    Linear scaled by 1e-3, so its variance (about 1e-6) is below eps.  Returns (params, keys, e, emulated h)."""
    layers = 6
    inp, middle = O.CONFIGS[layers]
    p = O.synth_params(3, layers)
    for k in ("weight", "bias"):
        p[0][f"gamma_function.0.{k}"] = p[0][f"gamma_function.0.{k}"] * 1e-3
    keys = [(i, f) for i in range(5) for f in O.FNS]
    e = torch.randn(2 * layers, inp, generator=torch.Generator().manual_seed(1)).to(tdt).double()
    w1 = torch.cat([p[i][f"{f}.0.weight"] for i, f in keys]).to(tdt).double()
    b1 = torch.cat([p[i][f"{f}.0.bias"] for i, f in keys])
    lw = torch.stack([p[i][f"{f}.1.weight"] for i, f in keys])
    lb = torch.stack([p[i][f"{f}.1.bias"] for i, f in keys])
    with X.generic_operands():
        h = X.hidden(e[None].numpy(), w1[None].numpy(), b1[None].numpy(), lw[None].numpy(), lb[None].numpy(),
                     middle, 2, tdt)
    return p, keys, e, torch.from_numpy(h).double()


def test_hidden_emulation_matches_oracle_in_float32():
    """hidden with float32 in place of the 16-bit type against the unrounded oracle.hidden, to summation order:
    |difference| / (|reference| + 1) below 2e-6 (measured 1.8e-7).  In the emulation, a LayerNorm without eps gives
    1.6 here (the low-variance branch), an unbiased variance 9e-4."""
    p, keys, e, h = hidden_case(torch.float32)
    ref = torch.cat([O.hidden(e, p[i], f) for i, f in keys], 1)
    err = float(((h - ref).abs() / (ref.abs() + 1)).max())
    assert err < 2e-6, err


@pytest.mark.parametrize("tdt", [torch.float16, torch.bfloat16])
def test_hidden_and_gemm_emulation_match_operand_rounded_oracle(tdt):
    """hidden (layer 1 + LayerNorm + LeakyReLU) and the layer-2 GEMM with 16-bit operands against oracle.hidden /
    gamma_beta rounding the same operands: within half a 16-bit ulp of the hidden rows plus 1e-4 (the emulation
    rounds them once, the oracle not at all), and the GEMM at fp32 summation-order tolerance."""
    p, keys, e, hd = hidden_case(tdt)
    middle = O.CONFIGS[6][1]
    ref = torch.cat([O.hidden(e, p[i], f, tdt) for i, f in keys], 1)
    half_ulp = 2.0 ** (-11 if tdt == torch.float16 else -8)
    excess = (hd - ref).abs() - ref.abs() * half_ulp
    assert float(excess.max()) <= 1e-4, float(excess.max())
    w2 = torch.stack([p[i][f"{f}.3.weight"] for i, f in keys]).to(tdt).double()
    b2 = torch.stack([p[i][f"{f}.3.bias"] for i, f in keys])
    with X.generic_operands():
        y = X.gemm(2, hd.numpy(), w2.numpy(), b2.numpy(), 1, middle, 2)
    ref2 = torch.stack([hd[:, j * middle:(j + 1) * middle] @ w2[j].t() + b2[j].double() for j in range(10)])
    err = (torch.from_numpy(y).double() - ref2).abs() / (ref2.abs() + 1)
    assert float(err.max()) < 1e-5, float(err.max())

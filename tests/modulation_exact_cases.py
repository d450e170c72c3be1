"""Float32 emulation of the latent modulation kernels (csrc/hf_modulation.cu) and the operand designs that make their
MMA sums exact.  tests/test_gpu_modulation_exact.py compares the kernels with it bit for bit;
tests/test_modulation_exact_cases_cpu.py checks it on the CPU, against oracle/modulation_oracle.py among others.

The emulation restates each kernel's stated arithmetic: float64 where the kernel is exact (every MMA sum, which
`exact_dot` asserts), numpy float32 for each fp32 operation, one RNE rounding where the kernel stores 16 bits.  The
library is built without fast math and without flush-to-zero, and the SASS of hf_modulation.cu fixes these
contractions, which the emulation follows:
  * hidden LayerNorm:  rstd = 1 / sqrtf(fl(S / middle) + 1e-5f) (FADD), t = FFMA(fl(fl(v - mean) rstd), w, b);
  * chain LayerNorm:   inv_n = fl(1 / (L 512)), mean = fl(total inv_n), var + eps = FFMA(S, inv_n, 1e-5f),
                       t = FFMA(fl(fl(v - mean) rstd), fl(1 + gamma), beta);
  * LeakyReLU:         FMUL by fl(0.01) (hidden: unless t > 0; chain: where t <= 0, modules 1..4);
  * PixelNorm:         ss = FFMA(x, x, ss) over the rows in order, inv = 1 / sqrtf(fl(fl(ss / L) + 1e-8f));
  * epilogue:          FFMA(dt, 0.1f, base), with two stacks FFMA(fl(dt_0 + dt_1), 0.1f, base);
  * sqrtf and the divisions are IEEE (correctly rounded), as numpy's float32 operations are.
The CTA and cluster sums follow the kernels' documented order: each thread's elements i = tid + 256 e in order of e,
the xor butterfly 16, 8, 4, 2, 1, the 8 warp sums in order, then (chain) the 8 rank sums in order."""
import contextlib
from fractions import Fraction

import numpy as np
import torch

f32, f64 = np.float32, np.float64
DIM, MODULES, CTA, THREADS = 512, 5, 8, 256
SLOPE = f32(0.01)
LN_EPS, PIXEL_EPS, DT_SCALE = f32(1e-5), f32(1e-8), f32(0.1)


# ------------------------------------------------------------------------------------------------ exact float32 ops
def round_fraction_f32(x: Fraction) -> np.float32:
    """x rounded to the nearest float32, ties to even (normal range)."""
    r = f32(float(x))
    best = None
    for c in (np.nextafter(r, f32(-np.inf)), r, np.nextafter(r, f32(np.inf))):
        d = abs(Fraction(float(c)) - x)
        key = (d, int(np.array(c).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return f32(best[1])


def fmaf(a, b, c) -> np.ndarray:
    """fmaf(a, b, c) on float32 arrays: a b is exact in float64; a + b in float64 is corrected by TwoSum.  The float64
    sum rounded to float32 is the correctly rounded result unless that sum is itself inexact and sits exactly on a
    float32 midpoint (then the float64 rounding decided the tie); those elements are recomputed with Fraction."""
    a, b, c = np.broadcast_arrays(np.asarray(a, f32), np.asarray(b, f32), np.asarray(c, f32))
    p = a.astype(f64) * b.astype(f64)
    cc = c.astype(f64)
    s = p + cc
    bb = s - p
    err = (p - (s - bb)) + (cc - bb)
    r = s.astype(f32)
    toward = np.nextafter(r, np.where(s > r.astype(f64), f32(np.inf), f32(-np.inf)).astype(f32))
    mid = (r.astype(f64) + toward.astype(f64)) / 2
    bad = (err != 0) & (s != r.astype(f64)) & (s == mid)
    if bad.any():
        r = r.copy()
        for i in zip(*np.nonzero(bad)):
            r[i] = round_fraction_f32(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
    return r


def round16(x, tdt) -> np.ndarray:
    """float32 -> the 16-bit type with RNE (the kernels' Half2T::one / st8), returned as float32 values."""
    return torch.from_numpy(np.ascontiguousarray(x, f32)).to(tdt).float().numpy()


def lsb_log2(x: np.ndarray) -> np.ndarray:
    """log2 of the lowest set bit of each float64 value (+inf for zero)."""
    m, e = np.frexp(x)
    i = np.abs(m * 2.0 ** 53).astype(np.int64)
    low = np.where(i == 0, 1, i & -i)
    return np.where(x == 0, np.inf, np.log2(low.astype(f64)) + e - 53)


_CHECK_EXACT = [True]


@contextlib.contextmanager
def generic_operands():
    """Within it exact_dot does not assert exactness: the emulation on generic operands, for comparisons with the
    float64 oracle at summation-order tolerance."""
    _CHECK_EXACT[0] = False
    try:
        yield
    finally:
        _CHECK_EXACT[0] = True


def exact_dot(x: np.ndarray, w: np.ndarray, k_ranges) -> list:
    """[x[..., k] @ w[n, k] for k in each range] in float64, asserting that every one is exact in fp32: all terms are
    multiples of one quantum q and sum |terms| < 2^24 q, so no MMA accumulation order can round.  x [..., K],
    w [N, K].  q is exact where w has at most one nonzero per output in the range, a lower bound (the smallest
    quantum of the row of x over the columns w uses times that of the row of w) otherwise."""
    out = []
    for k0, k1 in k_ranges:
        xs, ws = x[..., k0:k1].astype(f64), w[:, k0:k1].astype(f64)
        y = xs @ ws.T
        out.append(y)
        if not _CHECK_EXACT[0]:
            continue
        mag = np.abs(xs) @ np.abs(ws).T
        lx, lw = lsb_log2(xs), lsb_log2(ws)
        nnz = (ws != 0).sum(1)
        if nnz.max(initial=0) <= 1:
            k = np.argmax(ws != 0, 1)
            q = lx[..., k] + lw[np.arange(len(k)), k]
        else:
            q = lx[..., (ws != 0).any(0)].min(-1, initial=np.inf)[..., None] + lw.min(-1)
        ok = (mag == 0) | (mag < np.exp2(np.minimum(q + 24, 1000)))
        assert ok.all(), f"MMA sum over k {k0}..{k1} not exact in fp32 for {int((~ok).sum())} outputs"
    return out


def tree_sum(vals: np.ndarray, mask: np.ndarray, ranks: bool) -> np.ndarray:
    """The kernels' CTA (and cluster) sum of per-element float32 values.  vals / mask [..., (CTA,) per, 256]: element
    e of thread tid.  Per thread in order of e, xor butterfly over each warp's 32 lanes, warp sums 0..7 in order, then
    (ranks) the 8 rank sums in order.  Returns [...]."""
    t = np.zeros(vals.shape[:-2] + (THREADS,), f32)
    for e in range(vals.shape[-2]):
        t = np.where(mask[..., e, :], t + vals[..., e, :], t)
    lanes = t.reshape(t.shape[:-1] + (THREADS // 32, 32))
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[..., idx ^ o]
    w = lanes[..., 0]
    tot = np.zeros(w.shape[:-1], f32)
    for i in range(THREADS // 32):
        tot = tot + w[..., i]
    if not ranks:
        return tot
    out = np.zeros(tot.shape[:-1], f32)
    for r in range(CTA):
        out = out + tot[..., r]
    return out


def lrelu(t: np.ndarray, positive_strict: bool) -> np.ndarray:
    return np.where(t > 0 if positive_strict else ~(t <= 0), t, t * SLOPE)


# ------------------------------------------------------------------------------------------------ kernels
def embed16(sources, stacks: int, inp: int, tdt) -> np.ndarray:
    """hf_mod_embed16: sources = the 512-wide blocks [B, L, 512] float32 in the order src[s * inp / 512 + j] ->
    e16 [stacks, B L, inp]."""
    nseg = inp // DIM
    out = []
    for s in range(stacks):
        blocks = [np.asarray(sources[s * nseg + j], f32) for j in range(nseg)]
        out.append(np.concatenate([b.reshape(-1, DIM) for b in blocks], -1))
    return round16(np.stack(out), tdt)


def split_ranges(K: int, splits: int):
    """The split-K GEMM's K ranges: split s covers 64-wide k tiles kt s / S .. kt (s + 1) / S."""
    kt = -(-K // 64)
    return [(kt * s // splits * 64, min(K, kt * (s + 1) // splits * 64)) for s in range(splits)]


def splitk(x: np.ndarray, w: np.ndarray, bias, splits: int, reverse: bool = False) -> np.ndarray:
    """The split-K GEMM and its reduction: bias + part_0 + part_1 + ... in fp32, in split order (0 without bias);
    `reverse` adds the partials in the opposite order, which the tests must be able to tell apart."""
    parts = exact_dot(x, w, split_ranges(w.shape[1], splits))[::-1 if reverse else 1]
    y = np.zeros(x.shape[:-1] + (w.shape[0],), f32) if bias is None else np.broadcast_to(
        np.asarray(bias, f32), x.shape[:-1] + (w.shape[0],)).copy()
    for p in parts:
        y = y + p.astype(f32)
    return y


def gemm(layer: int, x16, w16, bias, stacks: int, middle: int, splits: int) -> np.ndarray:
    """hf_mod_gemm: layer 1 x16 [stacks, rows, inp], w16 [stacks, 10 middle, inp] -> [stacks, rows, 10 middle];
    layer 2 x16 [rows, 10 stacks middle], w16 [10 stacks, 512, middle] -> [10 stacks, rows, 512]."""
    if layer == 1:
        return np.stack([splitk(x16[s], w16[s], None if bias is None else bias[s], splits) for s in range(stacks)])
    return np.stack([splitk(x16[:, g * middle:(g + 1) * middle], w16[g], None if bias is None else bias[g], splits)
                     for g in range(10 * stacks)])


def hidden(e16, w16, bias, ln_w, ln_b, middle: int, splits: int, tdt, reverse: bool = False) -> np.ndarray:
    """hf_mod_hidden: e16 [stacks, rows, inp], w16 [stacks, 10 middle, inp], bias [stacks, 10 middle],
    ln_w / ln_b [stacks, 10, middle] -> h16 [rows, stacks 10 middle] (16-bit values as float32)."""
    stacks, rows = e16.shape[:2]
    v = np.stack([splitk(e16[s], w16[s], bias[s], splits, reverse) for s in range(stacks)])
    v = v.reshape(stacks, rows, 10, middle // THREADS, THREADS)         # [s, p, j, e, tid]: n = tid + 256 e
    mask = np.ones(v.shape, bool)
    mean = tree_sum(v, mask, False) / f32(middle)
    d = v - mean[..., None, None]
    sq = np.zeros(d.shape[:-2] + (THREADS,), f32)
    for e in range(d.shape[-2]):
        sq = fmaf(d[..., e, :], d[..., e, :], sq)
    S = tree_sum(sq[..., None, :], np.ones(sq[..., None, :].shape, bool), False)
    rstd = f32(1) / np.sqrt(S / f32(middle) + LN_EPS)
    a = d * rstd[..., None, None]
    g = np.asarray(ln_w, f32).reshape(stacks, 1, 10, middle // THREADS, THREADS)
    b = np.asarray(ln_b, f32).reshape(stacks, 1, 10, middle // THREADS, THREADS)
    t = lrelu(fmaf(a, g, b), True).reshape(stacks, rows, 10 * middle)
    return round16(t.transpose(1, 0, 2).reshape(rows, stacks * 10 * middle), tdt)


def pixel_norm(x0: np.ndarray, tdt) -> np.ndarray:
    """The chain's prologue on x0 [B, L, 512] -> the 16-bit operand [B, L, 512]."""
    x0 = np.asarray(x0, f32)
    ss = np.zeros((x0.shape[0], DIM), f32)
    for l in range(x0.shape[1]):
        ss = fmaf(x0[:, l], x0[:, l], ss)
    inv = f32(1) / np.sqrt(ss / f32(x0.shape[1]) + PIXEL_EPS)
    return round16(x0 * inv[:, None], tdt)


def chain_stack(x0, fc_w, fc_b, gb, tdt) -> np.ndarray:
    """dt of one stack in hf_mod_chain: x0 [B, L, 512] fp32, fc_w [5, 512, 512] (16-bit values), fc_b [5, 512],
    gb [10, B L, 512] (gamma / beta of module m at 2 m / 2 m + 1) -> [B, L, 512] float32."""
    B, L = x0.shape[:2]
    NT = -(-L // 8)
    per = 2 * NT
    inv_n = f32(1) / f32(L * DIM)
    x = pixel_norm(x0, tdt)
    # element i = tid + 256 e of CTA r: row l = i / 64, column r 64 + i % 64
    i = np.arange(per)[:, None] * THREADS + np.arange(THREADS)[None]
    li, ci = i // 64, i % 64
    mask = np.broadcast_to((li < L)[None, None], (B, CTA, per, THREADS))
    lc = np.minimum(li, L - 1)
    cols = np.arange(CTA)[:, None, None] * 64 + ci[None]                      # [r, e, tid]

    def to_threads(a):                                                         # [B, L, 512] -> [B, r, e, tid]
        return a[:, lc[None], cols]

    for m in range(MODULES):
        h0, h1 = exact_dot(x, fc_w[m], [(0, 256), (256, 512)])
        v = (h0.astype(f32) + h1.astype(f32)) + np.asarray(fc_b[m], f32)
        vt = to_threads(v)
        mean = tree_sum(vt, mask, True) * inv_n
        d = vt - mean[:, None, None, None]
        sq = np.zeros((B, CTA, THREADS), f32)
        for e in range(per):
            sq = np.where(mask[:, :, e], fmaf(d[:, :, e], d[:, :, e], sq), sq)
        S = tree_sum(sq[:, :, None], np.ones(sq[:, :, None].shape, bool), True)
        rstd = f32(1) / np.sqrt(fmaf(S, inv_n, LN_EPS))
        gam = np.asarray(gb[2 * m], f32).reshape(B, L, DIM)
        bet = np.asarray(gb[2 * m + 1], f32).reshape(B, L, DIM)
        a = (v - mean[:, None, None]) * rstd[:, None, None]
        t = fmaf(a, f32(1) + gam, bet)
        if m + 1 < MODULES:
            x = round16(lrelu(t, False), tdt)
        else:
            return t


def chain(x0s, fc_w, fc_b, gb, base, tdt) -> np.ndarray:
    """hf_mod_chain: x0s per stack [B, L, 512], fc_w [stacks, 5, 512, 512], fc_b [stacks, 5, 512],
    gb [10 stacks, B L, 512], base [B, L, 512] -> out [B, L, 512] float32."""
    dts = [chain_stack(x0s[s], fc_w[s], fc_b[s], gb[10 * s:10 * s + 10], tdt) for s in range(len(x0s))]
    dt = dts[0] if len(dts) == 1 else dts[0] + dts[1]
    return fmaf(dt, DT_SCALE, np.asarray(base, f32))


def run_stacks(sources, x0s, base, fc_w, fc_b, w1, b1, ln_w, ln_b, w2, b2, inp, middle, splits, tdt):
    """The six launches of modulation.run composed: embed16, hidden, layer-2 gemm, chain.  splits = (layer 1,
    layer 2) split counts of the plan."""
    stacks = len(x0s)
    e16 = embed16(sources, stacks, inp, tdt)
    h16 = hidden(e16, w1, b1, ln_w, ln_b, middle, splits[0], tdt)
    gb = gemm(2, h16, w2, b2, stacks, middle, splits[1])
    return chain(x0s, fc_w, fc_b, gb, base, tdt)


# ------------------------------------------------------------------------------------------------ operand designs
def _four_squares(limit: int) -> dict:
    """n -> (a, b, c, d) with a^2 + b^2 + c^2 + d^2 = n, for n <= limit (Lagrange)."""
    out = {}
    r = int(limit ** 0.5) + 1
    for a in range(r):
        for b in range(a, r):
            for c in range(b, r):
                for d in range(c, r):
                    n = a * a + b * b + c * c + d * d
                    if n <= limit and n not in out:
                        out[n] = (a, b, c, d)
    return out


_SQUARES = _four_squares(24 * 16)


def unit_columns(rng: np.random.Generator, L: int, n: int) -> np.ndarray:
    """[L, n] integer columns a with sum_l a^2 = L 4^m, m in {1, 2} per column: PixelNorm of a 2^t divides by the
    exact power of two 2^(m + t).  Four-square completion for L >= 4, +-2^m for smaller L."""
    out = np.zeros((L, n))
    for j in range(n):
        m = int(rng.integers(1, 3))
        T = L * 4 ** m
        if L < 4:
            col = np.full(L, 2.0 ** m)
        else:
            while True:
                head = rng.integers(-2 ** m - 1, 2 ** m + 2, L - 4)
                rest = T - int((head * head).sum())
                if 0 <= rest <= max(_SQUARES):
                    break
            col = np.concatenate([head, _SQUARES[rest]]).astype(f64)
            rng.shuffle(col)
        out[:, j] = col * rng.choice([-1.0, 1.0], L)
    return out


# x0 column kinds in the second K half (columns 256..511): the first K half is all UNIT
UNIT, ZERO, EPS_VISIBLE = 0, 1, 2


def column_kinds() -> np.ndarray:
    k = np.full(DIM, UNIT)
    k[256 + 1::4] = EPS_VISIBLE
    k[256 + 2::8] = ZERO
    return k


def pixel_x0(rng: np.random.Generator, B: int, L: int) -> np.ndarray:
    """[B, L, 512] float64: UNIT columns a 2^t (t in {-2, -1, 0}, mean square 4^(m + t) in 1/4 .. 16 absorbs 1e-8
    but not 1e-5), so PixelNorm is exact; ZERO columns; EPS_VISIBLE columns of mean square about 2^-32, where the
    1e-8 dominates and the kernel's rounding of ss / L + 1e-8, sqrtf and 1 / x all count."""
    kinds = column_kinds()
    x = np.zeros((B, L, DIM))
    for b in range(B):
        u = unit_columns(rng, L, DIM) * np.exp2(rng.integers(-2, 1, DIM))[None]
        eps = rng.integers(-3, 4, (L, DIM)) * 2.0 ** -17
        x[b] = np.where(kinds == UNIT, u, np.where(kinds == EPS_VISIBLE, eps, 0.0))
    return x


def permutation_weights(rng: np.random.Generator, n_out: int, ranges, exps=(-1, 0, 1)) -> np.ndarray:
    """[n_out, K]: in each K range, each output has one weight +-2^e on a column drawn by a permutation of the
    range (an output's columns cross every CTA slice and K half), so every partial sum is a single exact product."""
    K = ranges[-1][1]
    w = np.zeros((n_out, K))
    for k0, k1 in ranges:
        cols = np.concatenate([rng.permutation(k1 - k0) for _ in range(-(-n_out // (k1 - k0)))])[:n_out] + k0
        w[np.arange(n_out), cols] = rng.choice([-1.0, 1.0], n_out) * np.exp2(rng.choice(exps, n_out))
    return w


def module1_weights(rng: np.random.Generator) -> np.ndarray:
    """fc weight of module 1 [512, 512]: dense integers in -3..3 on the first K half (the exact PixelNorm output),
    a signed power-of-two permutation on the second (ZERO / EPS_VISIBLE columns make it generic)."""
    w = permutation_weights(rng, DIM, [(256, 512)])
    w[:, :256] = rng.integers(-3, 4, (DIM, 256))
    return w


def fc_weights(rng: np.random.Generator) -> np.ndarray:
    """[5, 512, 512]: module 1 as above, modules 2..5 one signed power-of-two weight per output per K half."""
    return np.stack([module1_weights(rng)] + [permutation_weights(rng, DIM, [(0, 256), (256, 512)])
                                              for _ in range(MODULES - 1)])

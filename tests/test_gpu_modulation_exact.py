"""Exact-arithmetic tests of the latent modulation kernels (csrc/hf_modulation.cu) through the C ABI, and of the three
drop-ins (hairfastgan_b200/modulation.py) end to end, against the float32 emulation in tests/modulation_exact_cases.py.

Every MMA sum is exact by design (the emulation asserts it): dense integer weights where the MMA input is short
(small-integer or dyadic embeddings, the PixelNorm output of columns whose mean square is a power of 4), otherwise at
most one signed power-of-two weight per output per K half (the chain) or per K split (the split-K GEMMs), drawn by
permutations that cross CTA slices and K halves.  Everything after the MMAs (split reductions, LayerNorm statistics
in the kernels' documented order, the modulation FFMA, LeakyReLU, 16-bit rounding, the epilogue) is emulated
operation by operation, so outputs are compared bit for bit.  gamma / beta, LayerNorm affines, biases and bases are
arbitrary fp32 values, different for every element, so a transposed or shifted read changes bits.

Each case id names the path it takes: the configuration, the chain's NT instantiation (rows of 8) and whether L is a
tail or a full tile, the split count of the plan (derived from hf_mod_gemm_plan and hf_sm_count), the row tile."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import modulation_oracle as O
from tests import modulation_exact_cases as X
from tests.gpu_util import enc_dtype_name

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ROWS, PER_SAMPLE, PER_LAYER = "rows", "per_sample", "per_layer"


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


def lib():
    from hairfastgan_b200 import _lib
    return _lib


def call(name, *args):
    """The C entry point with every tensor passed as its device pointer (the tensors stay referenced until the launch
    is queued)."""
    L = lib()
    L.check(getattr(L.lib(), name)(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]), name)


def plan(d, batch, layer, sms):
    out = (C.c_int * 5)()
    assert lib().lib().hf_mod_gemm_plan(C.byref(d), batch, layer, sms, out) == 0, lib().lib().hf_last_error()
    return list(out)


def nan_workspace(d, batch, dev):
    """The call's workspace with every byte 0xFF: NaN partials and dt, completion counters at -1."""
    n = lib().lib().hf_mod_workspace_bytes(C.byref(d), batch)
    assert n > 0, lib().lib().hf_last_error()
    return torch.full((n,), 0xFF, dtype=torch.uint8, device=dev)


def assert_equal(got, ref, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bad = ~(got == ref)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        pytest.fail(f"{what}: {int(bad.sum())} of {ref.size} values differ; first at {i}: got {got[i]!r}, "
                    f"expected {ref[i]!r}")


def dev16(x, tdt, dev):
    y = torch.from_numpy(np.asarray(x, np.float64)).to(tdt)
    assert torch.equal(y.double(), torch.from_numpy(np.asarray(x, np.float64))), "operand not exact in 16 bits"
    return y.contiguous().to(dev)


def dev32(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev)


def rows_view(x, form, dev, pad=3):
    """A strided fp32 device view of the logical [B, L, 512] array x in `form` (x must be constant along the
    broadcast axis), with an element offset of `pad` and padded rows: (hf_mod_rows, tensor to keep)."""
    B, L, _ = x.shape
    if form == ROWS:
        buf = torch.zeros(B, L + 1, 512 + 2 * pad)
        buf[:, 1:, pad:pad + 512] = torch.from_numpy(x)
        v = buf.to(dev)[:, 1:, pad:pad + 512]
        bs, rs = v.stride(0), v.stride(1)
    elif form == PER_SAMPLE:
        buf = torch.zeros(B, 512 + pad)
        buf[:, pad:] = torch.from_numpy(x[:, 0])
        v = buf.to(dev)[:, pad:]
        bs, rs = v.stride(0), 0
    else:
        buf = torch.zeros(L, 512 + pad)
        buf[:, pad:] = torch.from_numpy(x[0])
        v = buf.to(dev)[:, pad:]
        bs, rs = 0, v.stride(0)
    return lib().hf_mod_rows(v.data_ptr(), bs, rs), v


def broadcast(x, form):
    """[B, L, 512] constant along the axis `form` broadcasts."""
    if form == PER_SAMPLE:
        return np.broadcast_to(x[:, :1], x.shape).copy()
    if form == PER_LAYER:
        return np.broadcast_to(x[:1], x.shape).copy()
    return x


# ------------------------------------------------------------------------------------------------ hf_mod_embed16
def ties(rng, n, tdt):
    """n float32 values exactly halfway between two consecutive 16-bit values, half of them on an odd lower
    neighbour (RNE rounds away from zero) and half on an even one (RNE rounds toward zero)."""
    mant = 10 if tdt == torch.float16 else 7
    a = torch.from_numpy(rng.standard_normal(n) * 4).to(tdt).double()
    a[a == 0] = 1.0
    ulp = torch.pow(2.0, torch.floor(torch.log2(a.abs())) - mant)
    t = (a + torch.sign(a) * ulp / 2).numpy()
    assert np.array_equal(t.astype(np.float32).astype(np.float64), t)
    return t


# (name, L, inp, stacks, forms of the stacks' 512-wide blocks in src order)
EMBED = [("rotate_s1_rows", 6, 512, 1, [ROWS]),
         ("blending_s1_rows_sample_sample", 12, 1536, 1, [ROWS, PER_SAMPLE, PER_SAMPLE]),
         ("s1_inp1024_layer_rows", 5, 1024, 1, [PER_LAYER, ROWS]),
         ("post_s2_rows_rows", 18, 512, 2, [ROWS, ROWS]),
         ("s2_sample_layer_L1", 1, 512, 2, [PER_SAMPLE, PER_LAYER])]


@pytest.mark.parametrize("name,L,inp,stacks,forms", EMBED, ids=[e[0] for e in EMBED])
def test_embed16_bit_exact(dev, dt, name, L, inp, stacks, forms):
    """e16[s][p][k] = RNE16(src[s inp / 512 + k / 512][b][l][k % 512]) from strided, offset sources in every form,
    with a quarter of the values on a rounding tie: the stack / segment mapping, the strides and the rounding mode."""
    B = 3
    rng = np.random.default_rng(L * 100 + inp + stacks)
    srcs, keep, logical = [], [], []
    for j, form in enumerate(forms):
        x = (rng.standard_normal((B, L, 512)) * (j + 1)).astype(np.float32).astype(np.float64)
        tie = rng.random((B, L, 512)) < 0.25
        x[tie] = ties(rng, int(tie.sum()), dt[1])
        x = broadcast(x, form)
        r, v = rows_view(x, form, dev)
        srcs.append(r)
        keep.append(v)
        logical.append(x.astype(np.float32))
    ref = X.embed16(logical, stacks, inp, dt[1])
    t = np.concatenate(logical, -1).reshape(-1)
    rne = torch.from_numpy(t).to(dt[1]).float().numpy()
    assert (rne != t).any() and ((rne - t) * np.sign(t) > 0).any() and ((rne - t) * np.sign(t) < 0).any()
    d = lib().hf_mod_desc(L, inp, 512, stacks, dt[0])
    e16 = torch.full((stacks, B * L, inp), float("nan"), dtype=dt[1], device=dev)
    call("hf_mod_embed16", C.byref(d), B, (lib().hf_mod_rows * len(srcs))(*srcs), e16, lib().stream_ptr())
    assert_equal(e16.float().cpu().numpy(), ref, name)


# ------------------------------------------------------------------------------------------------ style layer 1
def split_scaled_embedding(rng, shape, K, splits, scales=(0, -9, 5, -4, 3, -7)):
    """Small integers times a power of two that changes from split to split: each split's partial sum is exact, the
    fp32 sum of the partials in split order is not, so the order shows."""
    x = rng.integers(-4, 5, shape + (K,)).astype(np.float64)
    for s, (k0, k1) in enumerate(X.split_ranges(K, splits)):
        x[..., k0:k1] *= 2.0 ** scales[s % len(scales)]
    return x


# (name, L, inp, middle, stacks, B, expect more than one split)
HIDDEN = [("m256_per1_splits_gt1", 6, 1536, 256, 1, 1, True),
          ("m512_per2_s2_splits_gt1", 18, 512, 512, 2, 1, True),
          ("m768_per3_splits_gt1", 12, 1024, 768, 1, 2, True),
          ("m1024_per4_s2_splits_1", 12, 512, 1024, 2, 6, False),
          ("m768_per3_splits_1", 24, 512, 768, 1, 12, False)]


@pytest.mark.parametrize("name,L,inp,middle,stacks,B,multi", HIDDEN, ids=[h[0] for h in HIDDEN])
def test_hidden_bit_exact(dev, sms, dt, name, L, inp, middle, stacks, B, multi):
    """Layer-1 GEMM, split reduction (bias then splits in order), LayerNorm([middle]) with the CTA sums in order,
    the affine FFMA, LeakyReLU and the 16-bit store.  Branch 0 of stack 0 has zero weights and a bias of spread
    about 2^-11: its variance (< 2.5e-7) is below eps, so eps and its place in rstd count.  The other branches add
    partials of spread about 1 to a bias offset of +-2^20, whose fp32 ulp (1/8) the LayerNorm magnifies: with more than
    one split, adding the partials in another order changes outputs even in bf16 (asserted on the emulation)."""
    d = lib().hf_mod_desc(L, inp, middle, stacks, dt[0])
    pl = plan(d, B, 1, sms)
    assert (pl[1] > 1) == multi, pl
    rows = B * L
    rng = np.random.default_rng(middle + L)
    e = split_scaled_embedding(rng, (stacks, rows), inp, pl[1], (-4, -8, -5, -7, -6, -9))
    w = rng.integers(-2, 3, (stacks, 10 * middle, inp)).astype(np.float64)
    w[0, :middle] = 0
    offset = np.repeat(rng.choice([-1.0, 1.0], (stacks, 10)) * 2.0 ** 20, middle, 1)
    bias = (offset + rng.standard_normal((stacks, 10 * middle))).astype(np.float32)
    bias[0, :middle] = rng.integers(-2, 3, middle) * 2.0 ** -12
    ln_w = (1 + 0.3 * rng.standard_normal((stacks, 10, middle))).astype(np.float32)
    ln_b = (0.2 * rng.standard_normal((stacks, 10, middle))).astype(np.float32)
    ref = X.hidden(e, w, bias, ln_w, ln_b, middle, pl[1], dt[1])
    assert (ref > 0).any() and (ref < 0).any()
    if multi:
        assert not np.array_equal(X.hidden(e, w, bias, ln_w, ln_b, middle, pl[1], dt[1], reverse=True), ref)
    h = torch.full((rows, stacks * 10 * middle), float("nan"), dtype=dt[1], device=dev)
    call("hf_mod_hidden", C.byref(d), B, dev16(w, dt[1], dev), dev16(e, dt[1], dev), dev32(bias, dev),
         dev32(ln_w, dev), dev32(ln_b, dev), h, nan_workspace(d, B, dev), lib().stream_ptr())
    assert_equal(h.float().cpu().numpy(), ref, f"{name} (splits {pl[1]})")


# ------------------------------------------------------------------------------------------------ hf_mod_gemm
# (name, layer, L, inp, middle, stacks, B, NULL bias, row tile, expect more than one split)
GEMM = [("l2_rows8_tile8", 2, 8, 512, 1024, 1, 1, False, 8, True),
        ("l2_rows9_tile64_tail", 2, 9, 512, 512, 1, 1, False, 64, True),
        ("l2_rows65_tile64_tail_s2_m256_splits_1", 2, 13, 512, 256, 2, 5, False, 64, False),
        ("l2_rows408_splits_1_null_bias", 2, 24, 512, 512, 1, 17, True, 64, False),
        ("l1_rows65_tail_inp1536_null_bias", 1, 13, 1536, 512, 1, 5, True, 64, True),
        ("l1_rows9_tail_inp1024_m768", 1, 9, 1024, 768, 1, 1, False, 64, True),
        ("l1_rows96_s2_splits_1", 1, 24, 512, 1024, 2, 4, False, 64, False)]


@pytest.mark.parametrize("name,layer,L,inp,middle,stacks,B,null_bias,tile,multi", GEMM, ids=[g[0] for g in GEMM])
def test_gemm_bit_exact(dev, sms, dt, name, layer, L, inp, middle, stacks, B, null_bias, tile, multi):
    """Style layers 1 and 2 with their split reduction, at row-tile tails, splits = 1 and a NULL bias.  Layer 1 reads
    split-scaled small-integer embeddings with dense weights; layer 2 reads generic 16-bit hidden rows with one
    signed power-of-two weight per output per split, so each partial is one exact product and the split order of
    the fp32 reduction shows."""
    d = lib().hf_mod_desc(L, inp, middle, stacks, dt[0])
    pl = plan(d, B, layer, sms)
    assert pl[0] == tile and (pl[1] > 1) == multi, pl
    rows = B * L
    rng = np.random.default_rng(layer * 1000 + rows)
    if layer == 1:
        x = split_scaled_embedding(rng, (stacks, rows), inp, pl[1])
        w = rng.integers(-2, 3, (stacks, 10 * middle, inp)).astype(np.float64)
        bias = rng.standard_normal((stacks, 10 * middle)).astype(np.float32)
        shape = (stacks, rows, 10 * middle)
    else:
        x = torch.from_numpy(rng.standard_normal((rows, 10 * stacks * middle))).to(dt[1]).double().numpy()
        ranges = X.split_ranges(middle, pl[1])
        w = np.stack([X.permutation_weights(rng, 512, ranges, (-2, -1, 0, 1, 2)) for _ in range(10 * stacks)])
        bias = rng.standard_normal((10 * stacks, 512)).astype(np.float32)
        shape = (10 * stacks, rows, 512)
    ref = X.gemm(layer, x, w, None if null_bias else bias, stacks, middle, pl[1])
    y = torch.full(shape, float("nan"), device=dev)
    bd = dev32(bias, dev)
    call("hf_mod_gemm", C.byref(d), B, layer, dev16(w, dt[1], dev), dev16(x, dt[1], dev), None if null_bias else bd,
         y, nan_workspace(d, B, dev), lib().stream_ptr())
    assert_equal(y.cpu().numpy(), ref, f"{name} (splits {pl[1]}, row tile {pl[0]})")


# ------------------------------------------------------------------------------------------------ hf_mod_chain
# (name, L, stacks, B, base form)
CHAIN = [("nt1_L1_tail_s1_b1", 1, 1, 1, ROWS),
         ("nt1_L6_tail_s2_b3", 6, 2, 3, PER_LAYER),
         ("nt1_L8_full_s1_b3", 8, 1, 3, ROWS),
         ("nt2_L9_tail_s2_b1", 9, 2, 1, ROWS),
         ("nt2_L12_tail_s1_b3", 12, 1, 3, PER_LAYER),
         ("nt2_L16_full_s2_b3", 16, 2, 3, ROWS),
         ("nt3_L17_tail_s1_b1", 17, 1, 1, PER_LAYER),
         ("nt3_L18_tail_s2_b3", 18, 2, 3, PER_LAYER),
         ("nt3_L24_full_s1_b3", 24, 1, 3, ROWS),
         ("nt3_L24_full_s2_b1", 24, 2, 1, ROWS),
         ("waves_nt1_L6_s2_b48", 6, 2, 48, ROWS)]


def chain_operands(rng, L, stacks, B):
    x0 = [X.pixel_x0(rng, B, L) for _ in range(stacks)]
    fc_w = np.stack([X.fc_weights(rng) for _ in range(stacks)])
    fc_b = (0.1 * rng.standard_normal((stacks, 5, 512))).astype(np.float32)
    gb = rng.standard_normal((10 * stacks, B * L, 512)) * np.tile([0.3, 0.2], 5 * stacks)[:, None, None]
    return x0, fc_w, fc_b, gb.astype(np.float32)


@pytest.mark.parametrize("name,L,stacks,B,base_form", CHAIN, ids=[c[0] for c in CHAIN])
def test_chain_bit_exact(dev, dt, name, L, stacks, B, base_form):
    """PixelNorm (exact UNIT columns, ZERO columns, EPS_VISIBLE columns), five fc + whole-sample LayerNorm +
    modulation steps with the cluster sums in rank order, the 16-bit handoff through every CTA's operand copy, and
    the epilogue: strided x0 views, base as rows or per layer, out and workspace filled with NaN (a counter that is
    not reset or a row that is not written fails).  A second call on the same workspace is bit-identical."""
    rng = np.random.default_rng(L * 10 + stacks + B)
    x0, fc_w, fc_b, gb = chain_operands(rng, L, stacks, B)
    base = broadcast(rng.standard_normal((B, L, 512)).astype(np.float32).astype(np.float64), base_form)
    ref = X.chain([x.astype(np.float32) for x in x0], fc_w, fc_b, gb, base, dt[1])
    inp = 512
    d = lib().hf_mod_desc(L, inp, 512, stacks, dt[0])
    x0r = [rows_view(x, ROWS, dev, pad=5 + s) for s, x in enumerate(x0)]
    br = rows_view(base, base_form, dev)
    ws = nan_workspace(d, B, dev)
    args = (dev16(fc_w, dt[1], dev), dev32(fc_b, dev), dev32(gb, dev))
    outs = []
    for _ in range(2):
        out = torch.full((B, L, 512), float("nan"), device=dev)
        call("hf_mod_chain", C.byref(d), B, *args, (lib().hf_mod_rows * 2)(*[r for r, _ in (x0r + x0r)[:2]]),
             C.byref(br[0]), out, ws, lib().stream_ptr())
        outs.append(out.cpu().numpy())
    assert_equal(outs[0], ref, name)
    assert_equal(outs[1], outs[0], f"{name}, second call")


# ------------------------------------------------------------------------------------------------ the drop-ins
def standin_params(rng, layers, splits2):
    """Per-module parameter dicts built to the exactness rules: dense integer first Linears (zero on the
    EPS_VISIBLE columns an embedding may carry), second Linears one signed power of two per output per layer-2
    split, fc weights as in the chain test; every bias and LayerNorm affine an arbitrary fp32 value."""
    inp, middle = O.CONFIGS[layers]
    fc_w = X.fc_weights(rng)
    eps_cols = np.tile(X.column_kinds() == X.EPS_VISIBLE, inp // 512)
    out = []
    for i in range(5):
        p = {"fc.weight": fc_w[i], "fc.bias": 0.1 * rng.standard_normal(512)}
        for f in O.FNS:
            w1 = rng.integers(-2, 3, (middle, inp)).astype(np.float64)
            w1[:, eps_cols] = 0
            p.update({f"{f}.0.weight": w1, f"{f}.0.bias": 0.1 * rng.standard_normal(middle),
                      f"{f}.1.weight": 1 + 0.3 * rng.standard_normal(middle),
                      f"{f}.1.bias": 0.2 * rng.standard_normal(middle),
                      f"{f}.3.weight": X.permutation_weights(rng, 512, X.split_ranges(middle, splits2)),
                      f"{f}.3.bias": 0.1 * rng.standard_normal(512)})
        out.append({k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in p.items()})
    return out


def packed(params_per_stack):
    """The layouts hf_modulation.cu reads, built from the per-module dicts: branch j = 2 i + (gamma 0 | beta 1)."""
    keys = [(i, f) for i in range(5) for f in O.FNS]
    n = lambda t: t.double().numpy()        # noqa: E731
    w1 = np.stack([np.concatenate([n(p[i][f"{f}.0.weight"]) for i, f in keys]) for p in params_per_stack])
    b1 = np.stack([np.concatenate([n(p[i][f"{f}.0.bias"]) for i, f in keys]) for p in params_per_stack])
    ln_w = np.stack([np.stack([n(p[i][f"{f}.1.weight"]) for i, f in keys]) for p in params_per_stack])
    ln_b = np.stack([np.stack([n(p[i][f"{f}.1.bias"]) for i, f in keys]) for p in params_per_stack])
    w2 = np.stack([n(p[i][f"{f}.3.weight"]) for p in params_per_stack for i, f in keys])
    b2 = np.stack([n(p[i][f"{f}.3.bias"]) for p in params_per_stack for i, f in keys])
    fc_w = np.stack([np.stack([n(p[i]["fc.weight"]) for i in range(5)]) for p in params_per_stack])
    fc_b = np.stack([np.stack([n(p[i]["fc.bias"]) for i in range(5)]) for p in params_per_stack])
    return dict(w1=w1, b1=b1.astype(np.float32), ln_w=ln_w.astype(np.float32), ln_b=ln_b.astype(np.float32),
                w2=w2, b2=b2.astype(np.float32), fc_w=fc_w, fc_b=fc_b.astype(np.float32))


DROP_INS = [("rotate_b2", 6, 2), ("blending_b3", 12, 3), ("postprocess_b1", 18, 1), ("postprocess_b18", 18, 18)]


@pytest.mark.parametrize("name,layers,B", DROP_INS, ids=[c[0] for c in DROP_INS])
def test_drop_ins_bit_exact(dev, sms, dt, name, layers, B):
    """rotate_forward, blending_forward and postprocess_forward on stand-in stacks against the composed emulation
    (embed16, hidden, layer-2 gemm, chain): which stack reads which embedding, the CLIP rows broadcast per sample,
    latent_avg per layer (at B = 18 it has the shape of a per-sample row and must still be read per layer), the
    base, and every stack's parameter packing."""
    from hairfastgan_b200 import modulation as M
    stacks = 2 if layers == 18 else 1
    inp, middle = O.CONFIGS[layers]
    d = lib().hf_mod_desc(layers, inp, middle, stacks, dt[0])
    splits = (plan(d, B, 1, sms)[1], plan(d, B, 2, sms)[1])
    rng = np.random.default_rng(layers * 100 + B)
    params = [standin_params(rng, layers, splits[1]) for _ in range(stacks)]
    lat = [X.pixel_x0(rng, B, layers).astype(np.float32) for _ in range(2)]
    g = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    if name.startswith("rotate"):
        model = O.StandInRotate(params[0], dev)
        got = M.rotate_forward(model, g(lat[0]), g(lat[1]))
        sources, x0s, base = [lat[1]], [lat[0]], lat[0]
    elif name.startswith("blending"):
        model = O.StandInBlending(params[0], dev)
        emb = rng.integers(-4, 5, (2, B, 512)).astype(np.float32)
        got = M.blending_forward(model, g(lat[0]), g(lat[1]), g(emb[0]), g(emb[1]))
        sources = [lat[1]] + [np.broadcast_to(e[:, None], (B, layers, 512)) for e in emb]
        x0s, base = [lat[0]], lat[0]
    else:
        avg = rng.standard_normal((layers, 512)).astype(np.float32)
        model = O.StandInPostProcess(params[0], params[1], torch.from_numpy(avg), dev)
        got = M.postprocess_forward(model, g(lat[0]), g(lat[1]))[0]
        sources, x0s, base = [lat[1], lat[0]], [lat[0], lat[1]], np.broadcast_to(avg, (B, layers, 512))
    pk = packed(params)
    ref = X.run_stacks(sources, x0s, base, pk["fc_w"], pk["fc_b"], pk["w1"], pk["b1"], pk["ln_w"], pk["ln_b"],
                       pk["w2"], pk["b2"], inp, middle, splits, dt[1])
    assert_equal(got.cpu().numpy(), ref, f"{name} (splits {splits})")

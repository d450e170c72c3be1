"""CtrlHair's shape adaptor on the GPU (hairfastgan_b200/shape_adaptor.py): the split-K GEMM bit for bit on integer
operands for every layer shape it serves, the layer-0 lookup and the LayerNorm against the oracle, and both drop-ins
against the golden of the unmodified reference (tests/golden/shape_adaptor.npz, oracle/gen_golden_shape_adaptor.py).
The mask generator is a stand-in module tree carrying the seeded golden parameters under the reference's names."""
import ctypes as C
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from baseline import refenv
from oracle import shape_adaptor_oracle as O
from tests.gpu_util import ROOT, enc_dtype_name, record, rel_err

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

# Codes against the golden: max-abs error relative to the RMS of the reference codes (16-bit activations, fp32
# accumulation and statistics).  Labels: the share of pixels that may differ from the reference's, and the largest
# reference top-2 logit margin a differing pixel may have.  The seeded weights give a noisy label map full of near
# ties (median margin about 0.25).  Measured on an H100 80GB HBM3 over the six golden cases: codes up to 3.7e-3 fp16 /
# 3.0e-2 bf16, flip rate up to 0.16 % fp16 / 1.13 % bf16, flipped margins up to 0.0066 fp16 / 0.066 bf16.  The bounds
# leave about 2x (fp16's flip rate keeps 0.5 %).
TOL_CODES = {"fp16": 8e-3, "bf16": 6e-2}
MAX_FLIP_RATE = {"fp16": 5e-3, "bf16": 2.5e-2}
MAX_FLIP_MARGIN = {"fp16": 0.015, "bf16": 0.15}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture()
def dt(hf_dtype):
    from hairfastgan_b200 import _lib
    return (_lib.HF_F16, torch.float16) if enc_dtype_name() == "fp16" else (_lib.HF_BF16, torch.bfloat16)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "shape_adaptor.npz"))


@pytest.fixture(scope="module")
def params(golden):
    return O.synth_params(int(golden["seed"]))


def gen_model(params):
    return O.stand_in_generator(params, torch.device("cuda:0"))


def mask_of(golden, name, dev):
    return torch.from_numpy(golden[f"{name}_mask"].astype(np.int64)).to(dev)


# ------------------------------------------------------------------------------------------------ split-K GEMM, exact
# (name, mode, cin, cout, hin) of every layer the GEMM serves
GEMM_LAYERS = ([(f"enc{i}", 1, cin, cout, 256 >> i) for i, (cin, cout) in
                enumerate(zip([32, 64, 128, 256, 512, 1024], [64, 128, 256, 512, 1024, 2048]), start=1)] +
               [("enc_fc_face", 0, 8192, 1024, 1), ("enc_fc_hair", 0, 8192, 16, 1),
                ("dec_in_hair", 0, 1040, 8192, 1), ("dec_in_face", 0, 1024, 8192, 1),
                ("dec0", 2, 2048, 2048, 2), ("dec1", 2, 2048, 1024, 4), ("dec2", 2, 1024, 512, 8)])


@pytest.mark.parametrize("name,mode,cin,cout,hin", GEMM_LAYERS, ids=[g[0] for g in GEMM_LAYERS])
def test_gemm_bit_exact(dev, dt, name, mode, cin, cout, hin):
    """Integer operands (every partial sum exact in fp32) against the float64 gather; impulses at the image corners,
    the last row / column and the stride-2 / upsample seams; the split count the plan picks is reported."""
    from hairfastgan_b200 import _lib, shape_adaptor as S
    g = torch.Generator().manual_seed(cin + cout + hin)
    x = torch.randint(-2, 3, (hin, hin, cin), generator=g).double()
    x[0, 0] = 9.0
    x[-1, -1] = -9.0
    x[-1, 0] = 7.0
    if hin > 2:
        x[hin // 2 - 1, hin // 2] = 5.0
    kk = {0: 1, 1: 4, 2: 3}[mode]
    w = torch.randint(-2, 3, (cout, kk, kk, cin), generator=g).double()
    b = torch.randint(-8, 9, (cout,), generator=g).double()
    ref = O.gather_gemm(mode, x, w, b) if mode else x.reshape(1, -1) @ w.reshape(cout, -1).t() + b
    pl = (C.c_int * 5)()
    assert _lib.lib().hf_shape_gemm_plan(mode, cin, cout, hin, hin, _lib.lib().hf_sm_count(), pl) == 0
    y16, y32 = S.gemm(mode, w.reshape(cout, -1).to(dt[1]).to(dev), x.to(dt[1]).to(dev), b.float().to(dev), hin, hin,
                      dt[0], want_y32=True)
    record(f"shape_gemm_{name}", splits=pl[1], pixel_tile=pl[0], k_tiles=pl[2])
    assert torch.equal(y32.cpu().double(), ref), (name, float((y32.cpu().double() - ref).abs().max()))
    assert torch.equal(y16.cpu(), ref.float().to(dt[1]))


# ------------------------------------------------------------------------------------------------ glue kernels
def test_layer0_lookup_vs_oracle(dev, dt, golden, params):
    from hairfastgan_b200 import shape_adaptor as S
    m = gen_model(params)
    for hair in (True, False):
        pk = S.PackedEncoder(m.hair_encoder if hair else m.face_encoder, hair, dt[0])
        mask = mask_of(golden, "some_255", dev)
        L, bad = S.labels(mask.clone())
        assert int(bad) == 0
        y = torch.empty(128, 128, 32, dtype=dt[1], device=dev)
        from hairfastgan_b200 import _lib
        _lib.check(_lib.lib().hf_shape_onehot_s2(L.data_ptr(), pk.table.data_ptr(), pk.cmap.data_ptr(), y.data_ptr(),
                                                 128, 32, dt[0], _lib.stream_ptr()))
        ref = O.layer0_lookup(mask.cpu(), pk.table.cpu(), pk.cmap.cpu())
        err = (y.cpu().double() - ref).abs()
        assert float((err - ref.abs() * 2.0 ** -7 - 1e-5).max()) <= 0, float(err.max())


@pytest.mark.parametrize("shape,offset", [((128, 128, 32), 0.0), ((256, 256, 32), 3.0), ((2, 2, 2048), 0.0),
                                          ((1, 8192), 40.0)])
def test_layer_norm_vs_oracle(dev, dt, shape, offset):
    from hairfastgan_b200 import shape_adaptor as S
    g = torch.Generator().manual_seed(shape[-1])
    x = (torch.randn(*shape, generator=g) * 2 + offset).to(dt[1])
    c = shape[-1]
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    y = S.layer_norm_lrelu(x.to(dev), gamma.to(dev), beta.to(dev), dt[0]).cpu().double()
    ref = O.layer_norm_lrelu(x.double(), gamma, beta)
    ulp = 2.0 ** (-10 if dt[1] == torch.float16 else -7)
    assert bool(((y - ref).abs() <= ref.abs() * ulp + 1e-4).all()), float((y - ref).abs().max())


# ------------------------------------------------------------------------------------------------ drop-ins vs golden
def test_codes_and_labels_vs_golden(dev, golden, params):
    from hairfastgan_b200 import shape_adaptor as S
    m = gen_model(params)
    names = [str(n) for n in golden["names"]]
    codes = {n: S.get_hair_face_code(m, mask_of(golden, n, dev)) for n in names}
    res = {}
    for n in names:
        fe, _ = rel_err(codes[n][0], torch.from_numpy(golden[f"{n}_face_code"]))
        he, _ = rel_err(codes[n][1], torch.from_numpy(golden[f"{n}_hair_code"]))
        hair_from = str(golden[f"{n}_hair_from"])
        labels = S.get_new_shape(m, codes[n][0], codes[hair_from][1])
        assert labels.shape == (256, 256) and labels.dtype == torch.int64 and labels.is_cuda
        ref = torch.from_numpy(golden[f"{n}_labels"].astype(np.int64))
        margin = torch.from_numpy(golden[f"{n}_margin"].astype(np.float32))
        flip = labels.cpu() != ref
        rate = float(flip.float().mean())
        bound = MAX_FLIP_MARGIN[enc_dtype_name()]
        worst = float(margin[flip].max()) if bool(flip.any()) else 0.0
        res[n] = (fe, he, rate, worst, bound)
        record(f"shape_adaptor_{n}", enc_dtype=enc_dtype_name(), face_code_rel_err=fe, hair_code_rel_err=he,
               label_flip_rate=rate, worst_flipped_margin=worst, median_margin=float(margin.median()))
    for n, (fe, he, rate, worst, bound) in res.items():
        assert fe < TOL_CODES[enc_dtype_name()] and he < TOL_CODES[enc_dtype_name()], (n, fe, he)
        assert rate <= MAX_FLIP_RATE[enc_dtype_name()] and worst <= bound, (n, rate, worst, bound)


def test_deterministic_rng_and_syncs(dev, golden, params):
    from hairfastgan_b200 import shape_adaptor as S
    m = gen_model(params)
    mask = mask_of(golden, "face", dev)
    f0, h0 = S.get_hair_face_code(m, mask)
    l0 = S.get_new_shape(m, f0, h0)
    torch.manual_seed(11)
    torch.randn([1, 16])
    want_state = torch.get_rng_state()
    torch.manual_seed(11)
    torch.cuda.synchronize()
    counts = []
    for fn in (lambda: S.get_hair_face_code(m, mask), lambda: S.get_new_shape(m, f0, h0)):
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                out = fn()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        counts.append(len([w for w in caught if str(w.message).startswith("called a synchronizing")]))
        if len(counts) == 1:
            assert torch.equal(torch.get_rng_state(), want_state)        # the hair encoder's one CPU draw
            assert torch.equal(out[0], f0) and torch.equal(out[1], h0)
        else:
            assert torch.equal(out, l0)
    assert counts == [1, 0], counts


def test_mask_rewrite_and_errors(dev, golden, params):
    from hairfastgan_b200 import shape_adaptor as S
    m = gen_model(params)
    mask = mask_of(golden, "some_255", dev)
    n255 = int((mask == 255).sum())
    assert n255 > 0
    a = S.get_hair_face_code(m, mask)
    assert int((mask == 255).sum()) == 0 and int((mask == 19).sum()) == n255      # rewritten in place, as stock
    b = S.get_hair_face_code(m, mask)                                              # 19 is the same all-zero one-hot
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    as_float = mask_of(golden, "some_255", dev).float()
    S.get_hair_face_code(m, as_float)
    assert int((as_float == 255).sum()) == n255                                    # .long() copied: no rewrite
    for bad in (20, -1, 254):
        x = mask_of(golden, "face", dev)
        x[100, 3] = bad
        with pytest.raises(ValueError, match="outside"):
            S.get_hair_face_code(m, x)
    with pytest.raises(NotImplementedError):
        S.get_hair_face_code(m, torch.zeros(128, 128, dtype=torch.int64, device=dev))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.get_hair_face_code(m, torch.zeros(256, 256, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.get_new_shape(m, a[0].cpu(), a[1].cpu())
    other = dict(params)
    other["face_decoder.out_layer.conv.weight"] = torch.zeros(17, 32, 3, 3)
    other["face_decoder.out_layer.conv.bias"] = torch.zeros(17)
    with pytest.raises(NotImplementedError, match="config 054"):
        S.get_new_shape(gen_model(other), a[0], a[1])


def test_repack_on_load_state_dict(dev, golden, params):
    from hairfastgan_b200 import shape_adaptor as S
    m = gen_model(params)
    mask = mask_of(golden, "face", dev)
    f, h = S.get_hair_face_code(m, mask)
    la = S.get_new_shape(m, f, h)
    sd = m.state_dict()
    sd["face_encoder.out_layer.fc.bias"] = sd["face_encoder.out_layer.fc.bias"] + 1.0
    sd["face_decoder.out_layer.conv.bias"] = sd["face_decoder.out_layer.conv.bias"] + torch.arange(18, device=dev)
    m.load_state_dict(sd)
    f2, _ = S.get_hair_face_code(m, mask)
    assert torch.allclose(f2, f + 1.0, atol=1e-5)
    assert not torch.equal(S.get_new_shape(m, f, h), la)


# ------------------------------------------------------------------------------------------------ whole swap
@pytest.mark.skipif(not refenv.available(), reason="reference not built (oracle/build_ref.py)")
def test_overlay_all_swap_matches_stock_reference(tmp_path, hf_dtype):
    """baseline/run_swap.py --mode overlay_all (SEAN and the shape adaptor on our kernels) against the stock reference,
    at the final-image tolerance tests/test_gpu_swap.py states for the default dtypes (run once)."""
    from tests import test_gpu_swap as SW
    if hf_dtype not in (None, "default", "bf16"):
        pytest.skip("the swap arms run once, with the default dtypes")
    work = os.environ.get("HAIRFAST_WORK", "/tmp/hairfast_work")
    env = {k: v for k, v in os.environ.items() if k not in ("HAIRFAST_DTYPE", "HAIRFAST_ENC_DTYPE")}

    def run(mode):
        out = str(tmp_path / f"{mode}.pt")
        cmd = [sys.executable, os.path.join(ROOT, "baseline", "run_swap.py"), "--mode", mode, "--work", work, "--out",
               out, "--reps", "2", "--warmup", "1"]
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env)
        assert p.returncode == 0, (mode, p.stdout[-2000:], p.stderr[-4000:])
        return torch.load(out, weights_only=False)

    ref, got = run("reference"), run("overlay_all")
    assert got["summary"]["deterministic"] and got["summary"]["finite"]
    d = (got["finals"][-1] - ref["finals"][-1]).abs()
    mean, q99, mx = float(d.mean()), float(torch.quantile(d.flatten()[::7], 0.99)), float(d.max())
    record("swap_overlay_all_vs_stock_reference", mean_abs=mean, q99_abs=q99, max_abs=mx,
           full_swap_ms=got["summary"]["timings"][-1]["gpu_ms"],
           reference_full_swap_ms=ref["summary"]["timings"][-1]["gpu_ms"])
    assert (mean <= SW.TOL_FINAL_MEAN["default"] and q99 <= SW.TOL_FINAL_Q99["default"]
            and mx <= SW.TOL_FINAL_MAX["default"]), (mean, q99, mx)

"""SEAN encode_sean on the GPU (hairfastgan_b200/sean.py): the two new forms of the wgmma convolution bit for bit, the
reflection pad, the InstanceNorm and the class means against the oracle, and the whole encode against the golden of
the unmodified reference (tests/golden/sean_encode.npz, oracle/gen_golden_sean_encode.py).  The SEAN model is a
stand-in module tree carrying the seeded golden parameters under the reference's attribute names."""
import ctypes as C
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from baseline import refenv
from oracle import sean_encode_oracle as EO
from oracle import sean_oracle as SO
from tests import conv_exact_cases as T
from tests.gpu_util import ROOT, enc_dtype_name, record, rel_err
from tests.test_gpu_conv_exact import assert_equal, ints, nchw64, nhwc16, ulp16

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

# Stated tolerances of the whole encode against the reference golden, max-abs error relative to the RMS of the
# reference (16-bit activations, fp32 accumulation and statistics).  Measured on an H100 80GB HBM3 over the two
# golden cases: codes 9.9e-4 fp16 / 7.2e-3 bf16; InstanceNorm outputs up to 4.4e-3 fp16 / 4.2e-2 bf16; pre-tanh conv
# up to 3.7e-3 fp16 / 2.7e-2 bf16.  The bounds leave about 2x.
TOL_CODES = {"fp16": 2e-3, "bf16": 1.5e-2}
TOL_TAPS = {"fp16": 1e-2, "bf16": 8e-2}


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
    return np.load(os.path.join(ROOT, "tests", "golden", "sean_encode.npz"))


@pytest.fixture(scope="module")
def zparams(golden):
    return {k: v for k, v in SO.synth_sean_params(int(golden["seed"])).items() if k.startswith("Zencoder.")}


def zencoder_model(zparams):
    return SO.stand_in_model(zparams, torch.device("cuda:0"))


def golden_case(golden, case):
    labels = torch.from_numpy(golden[f"c{case}_labels"].astype(np.int64))
    return EO.golden_images(int(golden[f"c{case}_image_seed"]), labels.shape[0]), labels


def plan(desc, batch, h, w):
    from hairfastgan_b200 import _lib
    out = (C.c_int * 12)()
    assert _lib.lib().hf_conv2d_plan_query(C.byref(desc), batch, h, w, out) == 0, _lib.lib().hf_last_error()
    return T._as_dict(out)


# ------------------------------------------------------------------------------------------------ conv forms, exact
# (name, cin, cout, stored H, W, batch, (kchunk, mainloop))
PREPADDED = [("shift_kc64", 64, 64, 18, 34, 2, (64, T.SHIFT)), ("shift_kc32_stem", 3, 32, 34, 18, 2, (32, T.SHIFT)),
             ("tap_kc64_8x8", 64, 32, 10, 10, 3, (64, T.TAP))]


@pytest.mark.parametrize("name,cin,cout,h,w,batch,loop", PREPADDED)
def test_prepadded_conv_bit_exact(dev, dt, name, cin, cout, h, w, batch, loop):
    """Reflection-padded integer inputs (impulses at the corners and edges of the unpadded image, where reflection and
    zero padding differ) through hf_reflect_pad1_nhwc16 and the prepadded conv against float64 conv2d."""
    import hairfastgan_b200.nn16 as N
    cin_pad = max(32, cin)
    g = torch.Generator().manual_seed(cin + h)
    x = ints(g, (batch, cin, h - 2, w - 2), -3, 3)
    for b, (y, xx) in enumerate([(0, 0), (h - 3, w - 3), (0, w - 3)][:batch]):
        x[b, :, y, xx] = 40.0                                           # border impulses
    wt = ints(g, (cout, cin, 3, 3), -2, 2)
    ref = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), wt)
    pc = N.PackedConv2d(wt.float().to(dev), cin_pad=cin_pad, prepadded=True, dtype=dt[0])
    p = plan(pc.desc, batch, h, w)
    assert (p["kchunk"], p["a_slots"]) == loop, (name, p)
    xp = N.reflect_pad1(nhwc16(x, dt[1], dev, cin_pad), dt[0])
    assert_equal(nchw64(xp), F.pad(F.pad(x, (0, 0, 0, 0, 0, cin_pad - cin)), (1, 1, 1, 1), mode="reflect"), "pad")
    y16, _, y32 = pc(xp, want_y32=True)
    assert_equal(y32.cpu().double(), ref, name + " y32")
    assert_equal(nchw64(y16), ref.float().to(dt[1]).double(), name + " y16")


# (name, cin, cout, input H = W, batch, (kchunk, mainloop))
TRANSPOSED = [("shift_64x64", 64, 64, 64, 1, (64, T.SHIFT)), ("shift_16x16_kc32", 32, 96, 16, 2, (32, T.SHIFT)),
              ("tap_8x8", 128, 64, 8, 3, (64, T.TAP))]


@pytest.mark.parametrize("name,cin,cout,h,batch,loop", TRANSPOSED)
def test_transposed_conv_bit_exact(dev, dt, name, cin, cout, h, batch, loop):
    """ConvTranspose2d(3, 2, 1, output_padding 1) on integers against float64 conv_transpose2d, with impulses at the
    last row / column (whose odd outputs read the zero fill below / right of the image) and at the first."""
    import hairfastgan_b200.nn16 as N
    g = torch.Generator().manual_seed(cin + cout + h)
    x = ints(g, (batch, cin, h, h), -3, 3)
    x[0, :, h - 1, :] = 40.0
    x[-1, :, :, 0] = 40.0
    wt = ints(g, (cin, cout, 3, 3), -2, 2)
    ref = F.conv_transpose2d(x, wt, None, stride=2, padding=1, output_padding=1)
    pc = N.PackedConv2d(wt.float().to(dev), stride=2, transposed=True, dtype=dt[0])
    p = plan(pc.desc, batch, h, h)
    assert (p["kchunk"], p["a_slots"]) == loop, (name, p)
    shift = ints(g, (cout,), -4, 4)
    y16, _, y32 = pc(nhwc16(x, dt[1], dev), shift=shift.float().to(dev), want_y32=True)
    assert_equal(y32.cpu().double(), ref + shift.view(1, -1, 1, 1), name + " y32")
    assert_equal(nchw64(y16), (ref + shift.view(1, -1, 1, 1)).float().to(dt[1]).double(), name + " y16")


# ------------------------------------------------------------------------------------------------ glue kernels
def test_reflect_pad_bit_exact(dev, dt):
    import hairfastgan_b200.nn16 as N
    x = torch.randn(2, 24, 40, 8 * 5, generator=torch.Generator().manual_seed(4)).to(dt[1])
    y = N.reflect_pad1(x.to(dev), dt[0])
    ref = F.pad(x.permute(0, 3, 1, 2).float(), (1, 1, 1, 1), mode="reflect").permute(0, 2, 3, 1).to(dt[1])
    assert torch.equal(y.cpu(), ref)


@pytest.mark.parametrize("shape,offset", [((2, 256, 256, 32), 0.0), ((2, 64, 64, 128), 0.0), ((1, 32, 32, 256), 60.0)])
def test_instance_norm_vs_oracle(dev, dt, shape, offset):
    """Against EO.instance_norm_lrelu of the same 16-bit values: one rounding of the 16-bit output plus fp32 statistics;
    the offset case has mean >> std (a one-pass E[x^2] - E[x]^2 would lose the variance)."""
    import hairfastgan_b200.nn16 as N
    x = (torch.randn(*shape, generator=torch.Generator().manual_seed(shape[3])) * 2 + offset).to(dt[1])
    y = N.instance_norm_lrelu(x.to(dev), 0.2, dt[0]).cpu().double()
    ref = EO.instance_norm_lrelu(x.double().permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    err = (y - ref).abs()
    bound = ulp16(ref, dt[1]) + 1e-4 * ref.abs() + 1e-5
    assert bool((err <= bound).all()), float((err - bound).max())


def test_class_means_vs_oracle(dev, golden):
    """tanh + class means over the 128^2 nearest map, including the zero rows of absent and odd-only classes."""
    from hairfastgan_b200 import sean as S
    labels = torch.cat([golden_case(golden, 0)[1], golden_case(golden, 1)[1]])
    y = torch.randn(3, 512, 128, 128, generator=torch.Generator().manual_seed(6)) * 1.5
    maps, bad = S.batch_label_maps(labels.to(dev))
    got = S.class_means(y.to(dev), maps).cpu()
    assert int(bad.sum()) == 0
    ref = EO.class_means(torch.tanh(y.double()), labels)
    assert float((got.double() - ref).abs().max()) < 2e-6
    assert torch.equal(got == 0, ref == 0)
    assert int((ref.abs().sum(2) == 0).sum()) >= 6


# ------------------------------------------------------------------------------------------------ whole encode
@pytest.mark.parametrize("case", [0, 1])
def test_encode_vs_golden(dev, golden, zparams, case):
    from hairfastgan_b200 import nn16, sean as S
    images, labels = golden_case(golden, case)
    m = zencoder_model(zparams)
    codes = S.encode_sean(m, images.to(dev), labels.float().to(dev))
    assert codes.shape == (labels.shape[0], 19, 512) and codes.dtype == torch.float32 and codes.is_cuda
    ref = torch.from_numpy(golden[f"c{case}_codes"])
    assert torch.equal(codes.cpu() == 0, ref == 0)                  # exactly the reference's zero rows
    err, _ = rel_err(codes, ref)
    taps = {}
    maps, _ = S.batch_label_maps(labels.to(dev))
    again = S.run_zencoder(S._pack_zencoder(m.netG.Zencoder), images.to(dev), maps, taps)
    assert torch.equal(again, codes)
    tap_err = {}
    for name, t in taps.items():
        t = t if t.dtype == torch.float32 else nn16.to_nchw32(t)
        tap_err[name], _ = rel_err(EO.golden_sample_enc(t), torch.from_numpy(golden[f"c{case}_{name}"]))
    record(f"sean_encode_case{case}", enc_dtype=enc_dtype_name(), codes_rel_err=err, **tap_err)
    assert err < TOL_CODES[enc_dtype_name()], err
    for name, e in tap_err.items():
        assert e < TOL_TAPS[enc_dtype_name()], (name, e)


def test_encode_deterministic_rng_and_one_sync(dev, golden, zparams):
    from hairfastgan_b200 import sean as S
    images, labels = golden_case(golden, 0)
    m = zencoder_model(zparams)
    args = (m, images.to(dev), labels.float().to(dev))
    a = S.encode_sean(*args)
    state = torch.cuda.get_rng_state()
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            b = S.encode_sean(*args)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if str(w.message).startswith("called a synchronizing")]
    assert len(syncs) == 1, [str(w.message) for w in syncs]
    assert torch.equal(a, b)
    assert torch.equal(torch.cuda.get_rng_state(), state)


def test_encode_error_paths(dev, golden, zparams):
    from hairfastgan_b200 import sean as S
    m = zencoder_model(zparams)
    images = torch.zeros(2, 3, 256, 256, device=dev)
    for bad in (19, -1):
        L = torch.zeros(2, 1, 256, 256, device=dev)
        L[1, 0, 200, 3] = bad
        with pytest.raises(ValueError, match="outside 0..18"):
            S.encode_sean(m, images, L)
    with pytest.raises(NotImplementedError):
        S.encode_sean(m, torch.zeros(2, 3, 128, 128, device=dev), torch.zeros(2, 1, 128, 128, device=dev))
    with pytest.raises(NotImplementedError):
        S.encode_sean(m, images, torch.zeros(1, 1, 256, 256, device=dev))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.encode_sean(m, images.cpu(), torch.zeros(2, 1, 256, 256))
    other = dict(zparams)
    other["Zencoder.model.14.weight"] = torch.zeros(256, 256, 3, 3)
    other["Zencoder.model.14.bias"] = torch.zeros(256)
    with pytest.raises(NotImplementedError, match="Zencoder"):
        S.encode_sean(zencoder_model(other), images, torch.zeros(2, 1, 256, 256, device=dev))


def test_repack_on_parameter_change(dev, golden, zparams):
    from hairfastgan_b200 import sean as S
    m = zencoder_model(zparams)
    images, labels = golden_case(golden, 1)
    args = (m, images.to(dev), labels.float().to(dev))
    a = S.encode_sean(*args)
    m.netG.Zencoder.model[14].bias.add_(0.5)
    b = S.encode_sean(*args)
    assert not torch.equal(a, b)
    assert torch.equal(a == 0, b == 0)


# ------------------------------------------------------------------------------------------------ whole swap
@pytest.mark.skipif(not refenv.available(), reason="reference not built (oracle/build_ref.py)")
def test_overlay_sean_full_swap_matches_stock_reference(tmp_path, hf_dtype):
    """baseline/run_swap.py --mode overlay_sean_full (install(sean=True, sean_encode=True)) against the stock reference,
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

    ref, got = run("reference"), run("overlay_sean_full")
    assert got["summary"]["deterministic"] and got["summary"]["finite"]
    d = (got["finals"][-1] - ref["finals"][-1]).abs()
    mean, q99, mx = float(d.mean()), float(torch.quantile(d.flatten()[::7], 0.99)), float(d.max())
    record("swap_overlay_sean_full_vs_stock_reference", mean_abs=mean, q99_abs=q99, max_abs=mx,
           full_swap_ms=got["summary"]["timings"][-1]["gpu_ms"],
           reference_full_swap_ms=ref["summary"]["timings"][-1]["gpu_ms"])
    assert (mean <= SW.TOL_FINAL_MEAN["default"] and q99 <= SW.TOL_FINAL_Q99["default"]
            and mx <= SW.TOL_FINAL_MAX["default"]), (mean, q99, mx)

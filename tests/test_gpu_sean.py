"""SEAN decode_sean on the GPU (hairfastgan_b200/sean.py) against the CPU oracle and the golden of the unmodified
reference (tests/golden/sean.npz, oracle/gen_golden_sean.py).  The SEAN model is a stand-in module tree carrying the
seeded golden parameters under the reference's attribute names (the reference tree is not needed)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from baseline import refenv
from oracle import sean_oracle as SO
from tests.gpu_util import ROOT, enc_dtype_name, record, rel_err

pytestmark = pytest.mark.gpu

# Stated tolerances, max-abs error relative to the RMS of the reference (16-bit activations, fp32 accumulate):
# (measured on an H100: blocks up to 0.038 bf16 / 0.0045 fp16, image up to 0.093 bf16 / 0.012 fp16)
TOL_TABLE = 1e-4                                  # fp32 style tables
ULP16 = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}  # one-hot lookups: fp32 sums, then one rounding to the 16-bit type
TOL_BLOCK = {"bf16": 5e-2, "fp16": 6e-3}          # one SPADEResnetBlock (3 ACEs, 3 convolutions) from the same input
TOL_IMAGE = {"bf16": 1.5e-1, "fp16": 2e-2}        # final image after 7 chained blocks and tanh


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "sean.npz"))


@pytest.fixture(scope="module")
def params(golden):
    return SO.synth_sean_params(int(golden["seed"]))


@pytest.fixture(scope="module")
def model(params):
    return SO.stand_in_model(params, torch.device("cuda:0"))


def _case(golden, case):
    labels = torch.from_numpy(golden[f"c{case}_labels"].astype(np.int64))
    code = torch.from_numpy(golden[f"c{case}_code"])
    noise = SO.golden_noise(int(golden[f"c{case}_noise_seed"]))
    assert np.array_equal(np.stack([d.reshape(-1)[:16].numpy() for d in noise]), golden[f"c{case}_noise_head"])
    return labels, code, noise


def test_label_maps_and_onehot_lut(params):
    from hairfastgan_b200 import nn16, sean as S
    dev = torch.device("cuda:0")
    L = torch.randint(0, 19, (1, 1, 256, 256), generator=torch.Generator().manual_seed(1))
    maps = S.label_maps(L.to(dev))
    for r, m in zip(S.LEVELS, maps):
        assert torch.equal(m.long().cpu(), SO.label_map(L, r)), r
    for r, key, relu in [(8, "fc.", False), (32, "up_0.ace_s.Spade.mlp_shared.0.", True),
                         (256, "up_3.ace_1.Spade.mlp_shared.0.", True)]:
        w, b = params[key + "weight"], params[key + "bias"]
        ref = SO.onehot_conv_lut(SO.label_map(L, r), w, b)
        ref = torch.relu(ref) if relu else ref
        y = S.onehot_conv(maps[S.LEVELS.index(r)], S._onehot_table(w.to(dev)), b.to(dev), relu, nn16.default_dtype())
        d = (y[0].permute(2, 0, 1).float().cpu() - ref).abs()
        assert bool((d <= ref.abs() * ULP16[enc_dtype_name()] + 1e-6).all()), (r, float(d.max()))


def test_out_of_range_labels_raise(model):
    from hairfastgan_b200 import sean as S
    for bad in (19, -1):
        L = torch.zeros(1, 1, 256, 256, dtype=torch.int64)
        L[0, 0, 100, 37] = bad
        with pytest.raises(ValueError, match="outside 0..18"):
            S.decode_sean(model, torch.zeros(1, 19, 512, device="cuda:0"), L.cuda(),
                          noise=[torch.zeros(s, device="cuda:0") for s in SO.noise_shapes()],
                          mean_codes=torch.zeros(19, 512))


def test_style_tables_vs_oracle(golden, params, model):
    from hairfastgan_b200 import sean as S
    pk = S._pack(model.netG)
    code = torch.from_numpy(golden["c0_code"])
    mean = torch.from_numpy(golden["mean_codes"])
    tables = S.style_tables(pk.rgb_aces, code.cuda(), mean.cuda())
    codes = SO.style_codes(code, mean)
    names = [(n, a) for n, fin, fout, _, rgb in SO.BLOCKS if rgb for a, _ in SO.block_aces(fin, fout)]
    assert len(names) == len(tables) == 15
    for (n, a), t in zip(names, tables):
        pre = f"{n}.{a}."
        mu = torch.relu(torch.stack([codes[j] @ params[pre + f"fc_mu{j}.weight"].T + params[pre + f"fc_mu{j}.bias"]
                                     for j in range(19)]))
        ag, ab = torch.sigmoid(params[pre + "blending_gamma"]), torch.sigmoid(params[pre + "blending_beta"])
        w = torch.cat([params[pre + "conv_gamma.weight"] * ag, params[pre + "conv_beta.weight"] * ab])
        ref = SO.style_tables(w, mu)
        err, _ = rel_err(t, ref)
        assert err < TOL_TABLE, (pre, err)


@pytest.mark.parametrize("name", [b[0] for b in SO.BLOCKS])
def test_block_vs_oracle(golden, params, model, name):
    """One full SPADEResnetBlock per resolution, from the oracle's input of that block."""
    from hairfastgan_b200 import nn16, sean as S
    labels, code, noise = _case(golden, 0)
    mean = torch.from_numpy(golden["mean_codes"])
    p = dict(params)
    codes = SO.style_codes(code, mean)
    seg = SO.one_hot(labels)
    x = torch.nn.functional.conv2d(torch.nn.functional.interpolate(seg, size=(8, 8)), p["fc.weight"], p["fc.bias"],
                                   padding=1)
    it = iter(noise)
    bi = [b[0] for b in SO.BLOCKS].index(name)
    start = sum(len(SO.block_aces(b[1], b[2])) for b in SO.BLOCKS[:bi])         # first noise tensor of the block
    for n, fin, fout, _, rgb in SO.BLOCKS[:bi + 1]:
        if n in SO.UPSAMPLE_BEFORE:
            x = torch.nn.functional.interpolate(x, scale_factor=2, mode="nearest")
        x_in = x
        x = SO.block_ref(p, n, fin, fout, rgb, x, seg, codes, it)
    pk = S._pack(model.netG)
    dev = torch.device("cuda:0")
    blk = pk.blocks[bi]
    all_tables = S.style_tables(pk.rgb_aces, code.to(dev), mean.to(dev))
    t0 = sum(len(b.aces()) for b in pk.blocks[:bi] if b.ace_0.use_rgb)
    x16 = nn16.to_nhwc16(x_in.to(dev))
    maps = dict(zip(S.LEVELS, S.label_maps(labels.to(dev))))
    y = S.run_block(pk, blk, x16, maps[blk.res], iter([n.to(dev) for n in noise[start:]]), iter(all_tables[t0:]))
    err, rms = rel_err(nn16.to_nchw32(y), x)
    record(f"sean_block_{name}", enc_dtype=enc_dtype_name(), rel_err=err, max_abs_ref=float(x.abs().max()))
    assert err < TOL_BLOCK[enc_dtype_name()], (name, err)


@pytest.mark.parametrize("case", [0, 1])
def test_decode_vs_golden(golden, model, case):
    from hairfastgan_b200 import nn16, sean as S
    labels, code, noise = _case(golden, case)
    taps = {}
    pk = S._pack(model.netG)
    img = S.run_packed(pk, code.cuda(), labels.cuda(), torch.from_numpy(golden["mean_codes"]).cuda(),
                       [n.cuda() for n in noise], taps)
    out = S.decode_sean(model, code.cuda(), labels.cuda(), noise=[n.cuda() for n in noise],
                        mean_codes=torch.from_numpy(golden["mean_codes"]))
    assert out.shape == (3, 256, 256) and out.dtype == torch.float32 and out.is_cuda
    assert torch.equal(out, img)
    err, _ = rel_err(SO.golden_sample_image(img), torch.from_numpy(golden[f"c{case}_image"]))
    max_act = max(float(nn16.to_nchw32(t).abs().max()) for t in taps.values())
    record(f"sean_decode_case{case}", enc_dtype=enc_dtype_name(), rel_err=err, max_abs_residual=max_act)
    assert max_act < 6e4                                   # the fp16 residual stream stays far from overflow
    assert err < TOL_IMAGE[enc_dtype_name()], err


def test_decode_deterministic_and_rng_contract(golden, model):
    """Same inputs and noise -> the same bits; with noise=None the 18 draws are the reference's torch.randn(1, W, H, 1)
    sequence (normalization.py:111), so the generator state afterwards is the one the reference leaves."""
    from hairfastgan_b200 import sean as S
    labels, code, _ = _case(golden, 1)
    mean = torch.from_numpy(golden["mean_codes"])
    torch.manual_seed(123)
    state0 = torch.cuda.get_rng_state()
    draws = [torch.randn(*s, device="cuda") for s in SO.noise_shapes()]     # the reference's draws, in its order
    state_ref = torch.cuda.get_rng_state()
    torch.cuda.set_rng_state(state0)
    a = S.decode_sean(model, code.cuda(), labels.cuda(), mean_codes=mean)
    assert torch.equal(torch.cuda.get_rng_state(), state_ref)
    b = S.decode_sean(model, code.cuda(), labels.cuda(), noise=draws, mean_codes=mean)
    c = S.decode_sean(model, code.cuda(), labels.cuda(), noise=draws, mean_codes=mean)
    assert torch.equal(a, b) and torch.equal(b, c)


def test_unsupported_config_raises(params):
    from hairfastgan_b200 import sean as S
    m = SO.stand_in_model({k: v for k, v in params.items() if k.startswith("fc.")}, torch.device("cuda:0"))
    m.opt.ngf = 32
    with pytest.raises(NotImplementedError, match="ngf"):
        S.decode_sean(m, torch.zeros(1, 19, 512, device="cuda:0"), torch.zeros(1, 1, 256, 256, device="cuda:0"))


def test_repack_on_parameter_change(golden, params):
    from hairfastgan_b200 import sean as S
    m = SO.stand_in_model(params, torch.device("cuda:0"))
    labels, code, noise = _case(golden, 0)
    args = (m, code.cuda(), labels.cuda())
    kw = dict(noise=[n.cuda() for n in noise], mean_codes=torch.from_numpy(golden["mean_codes"]))
    a = S.decode_sean(*args, **kw)
    with torch.no_grad():
        m.netG.conv_img.bias.add_(0.5)
    b = S.decode_sean(*args, **kw)
    assert not torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ whole swap
@pytest.mark.skipif(not refenv.available(), reason="reference not built (oracle/build_ref.py)")
def test_overlay_sean_swap_matches_stock_reference(tmp_path, hf_dtype):
    """baseline/run_swap.py --mode overlay_sean (install(sean=True)) against the stock reference, at the final-image
    tolerance tests/test_gpu_swap.py states for the default dtypes (what a user of install() gets; run once)."""
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

    ref, got = run("reference"), run("overlay_sean")
    assert got["summary"]["deterministic"] and got["summary"]["finite"]
    d = (got["finals"][-1] - ref["finals"][-1]).abs()
    mean, q99, mx = float(d.mean()), float(torch.quantile(d.flatten()[::7], 0.99)), float(d.max())
    record("swap_overlay_sean_vs_stock_reference", mean_abs=mean, q99_abs=q99, max_abs=mx,
           full_swap_ms=got["summary"]["timings"][-1]["gpu_ms"],
           reference_full_swap_ms=ref["summary"]["timings"][-1]["gpu_ms"])
    assert (mean <= SW.TOL_FINAL_MEAN["default"] and q99 <= SW.TOL_FINAL_Q99["default"]
            and mx <= SW.TOL_FINAL_MAX["default"]), (mean, q99, mx)

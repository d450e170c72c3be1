"""HairFast's latent modulation nets on the GPU (hairfastgan_b200/modulation.py, csrc/hf_modulation.cu): the grouped
split-K GEMM bit for bit on integer operands for every shape it serves, the fused layer-1 reduction and the cluster
chain against the float64 oracle, and the three drop-ins against the golden of the unmodified reference
(tests/golden/modulation.npz, oracle/gen_golden_modulation.py), on stand-in modules carrying the seeded parameters
under the reference's names."""
import ctypes as C
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from baseline import refenv
from oracle import modulation_oracle as O
from tests.gpu_util import ROOT, enc_dtype_name, record

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

# Drop-ins against the golden: max-abs error of base + 0.1 dt relative to the RMS of the reference's 0.1 dt (16-bit
# operands, fp32 accumulation and statistics).  Measured on an H100 80GB HBM3 over the four golden cases and the
# batched oracle cases (B = 2 and 18): up to 5.9e-3 fp16 / 4.5e-2 bf16.
TOL_DROP_IN = {"fp16": 1.2e-2, "bf16": 9e-2}
# The chain against the operand-rounded oracle, same measure.  Summation order alone gives about 1e-6, but once one
# operand rounds the other way (an fp32 instead of a float64 value next to a 16-bit rounding boundary) the next
# modules' roundings follow, and the difference settles at the 16-bit rounding level.  A wrong cluster rank, output
# slice or K chunk gives O(1).  Measured up to 1.8e-3 fp16 / 6.7e-3 bf16 over L in {6, 12, 18} and B in {1, 2, 5}.
TOL_CHAIN = {"fp16": 4e-3, "bf16": 1.5e-2}
# embed16, hidden (GEMM + reduce / LayerNorm), gamma-beta (GEMM + reduce), chain; PostProcess's two stacks add one
# cudaMemsetAsync of the chain's completion counters, which is not a kernel launch
LAUNCHES_PER_CALL = 6


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
    return np.load(os.path.join(ROOT, "tests", "golden", "modulation.npz"))


def g64(golden, key, dev=None):
    x = torch.from_numpy(golden[key])
    return x.to(dev) if dev is not None else x.double()


def lib():
    from hairfastgan_b200 import _lib
    return _lib


def workspace(d, batch, dev):
    n = lib().lib().hf_mod_workspace_bytes(C.byref(d), batch)
    assert n > 0, lib().lib().hf_last_error()
    return torch.empty(n, dtype=torch.uint8, device=dev)


# ------------------------------------------------------------------------------------------------ grouped GEMM, exact
# (name, layers, inp, middle, stacks, layer): Rotate and PostProcess 512 -> 5120 and 10 x (512 -> 512), Blending
# 1536 -> 10240 and 10 x (1024 -> 512), PostProcess's two groups in layer 1 and twenty in layer 2
GEMMS = [("rotate_l1", 6, 512, 512, 1, 1), ("rotate_l2", 6, 512, 512, 1, 2),
         ("blending_l1", 12, 1536, 1024, 1, 1), ("blending_l2", 12, 1536, 1024, 1, 2),
         ("post_l1", 18, 512, 512, 2, 1), ("post_l2", 18, 512, 512, 2, 2)]


@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("name,layers,inp,middle,stacks,layer", GEMMS, ids=[g[0] for g in GEMMS])
def test_grouped_gemm_bit_exact(dev, dt, name, layers, inp, middle, stacks, layer, batch):
    """Integer operands (every partial sum exact in fp32) against float64; one impulse per group."""
    L = lib()
    rows = batch * layers
    g = torch.Generator().manual_seed(layers * 10 + layer + batch)
    if layer == 1:
        w = torch.randint(-2, 3, (stacks, 10 * middle, inp), generator=g).double()
        x = torch.randint(-2, 3, (stacks, rows, inp), generator=g).double()
        b = torch.randint(-8, 9, (stacks, 10 * middle), generator=g).double()
        x[:, -1, -1] = 9.0
        ref = torch.einsum("srk,snk->srn", x, w) + b[:, None]
    else:
        w = torch.randint(-2, 3, (10 * stacks, 512, middle), generator=g).double()
        x = torch.randint(-2, 3, (rows, 10 * stacks * middle), generator=g).double()
        b = torch.randint(-8, 9, (10 * stacks, 512), generator=g).double()
        x[-1, middle - 1::middle] = 7.0
        ref = torch.einsum("rgk,gnk->grn", x.view(rows, 10 * stacks, middle), w) + b[:, None]
    d = L.hf_mod_desc(layers, inp, middle, stacks, dt[0])
    y = torch.empty(ref.shape, dtype=torch.float32, device=dev)
    ws = workspace(d, batch, dev)
    wd, xd, bd = w.to(dt[1]).to(dev), x.to(dt[1]).to(dev), b.float().to(dev)
    L.check(L.lib().hf_mod_gemm(C.byref(d), batch, layer, wd.data_ptr(), xd.data_ptr(), bd.data_ptr(), y.data_ptr(),
                                ws.data_ptr(), L.stream_ptr()), "hf_mod_gemm")
    pl = (C.c_int * 5)()
    assert L.lib().hf_mod_gemm_plan(C.byref(d), batch, layer, L.lib().hf_sm_count(), pl) == 0
    record(f"mod_gemm_{name}_b{batch}", splits=pl[1], row_tile=pl[0], k_tiles=pl[2])
    assert torch.equal(y.cpu().double(), ref), (name, float((y.cpu().double() - ref).abs().max()))


# ------------------------------------------------------------------------------------------------ layer 1 + LayerNorm
@pytest.mark.parametrize("layers,inp,middle,stacks", [(6, 512, 512, 1), (12, 1536, 1024, 1), (18, 512, 512, 2)])
def test_hidden_layer_norm_vs_oracle(dev, dt, layers, inp, middle, stacks):
    """Against float64 from the same 16-bit operands, within half a 16-bit ulp of the result plus 1e-4.  Branch 0 of
    stack 0 gets its first Linear (weight and bias) scaled by 1e-3, so its pre-norm variance (about 1e-6) is below
    eps: a wrong eps moves it by a large factor.  In fp16 the unbiased variance would move every output by
    1 / (2 middle) relative, more than the bound."""
    L = lib()
    batch = 2
    rows = batch * layers
    params = [O.synth_params(40 + s, layers) for s in range(stacks)]
    g = torch.Generator().manual_seed(layers)
    e = torch.randn(stacks, rows, inp, generator=g).to(dt[1])
    keys = [(i, f) for i in range(5) for f in O.FNS]
    w1 = torch.stack([torch.cat([p[i][f"{f}.0.weight"] for i, f in keys]) for p in params])
    b1 = torch.stack([torch.cat([p[i][f"{f}.0.bias"] for i, f in keys]) for p in params])
    lw = torch.stack([torch.cat([p[i][f"{f}.1.weight"] for i, f in keys]) for p in params])
    lb = torch.stack([torch.cat([p[i][f"{f}.1.bias"] for i, f in keys]) for p in params])
    for k in ("weight", "bias"):
        params[0][0][f"gamma_function.0.{k}"] = params[0][0][f"gamma_function.0.{k}"] * 1e-3
    w1[0, :middle] *= 1e-3
    b1[0, :middle] *= 1e-3
    d = L.hf_mod_desc(layers, inp, middle, stacks, dt[0])
    h = torch.empty(rows, stacks * 10 * middle, dtype=dt[1], device=dev)
    ws = workspace(d, batch, dev)
    args = [t.to(dev).contiguous() for t in (w1.to(dt[1]), e, b1, lw, lb)]
    L.check(L.lib().hf_mod_hidden(C.byref(d), batch, *[t.data_ptr() for t in args], h.data_ptr(), ws.data_ptr(),
                                  L.stream_ptr()), "hf_mod_hidden")
    ref = torch.cat([O.hidden(e[s], params[s][i], f, dt[1]) for s in range(stacks) for i, f in keys], 1)
    y = h.cpu().double()
    half_ulp = 2.0 ** (-11 if dt[1] == torch.float16 else -8)
    excess = (y - ref).abs() - ref.abs() * half_ulp
    low_var = (ref[:, :middle].std() / ref[:, middle:2 * middle].std()).item()
    record(f"mod_hidden_L{layers}", enc_dtype=enc_dtype_name(), max_excess_over_half_ulp=float(excess.max()),
           low_variance_branch_std_ratio=low_var)
    assert low_var < 0.5                                   # eps 1e-5 dominates branch 0's variance
    assert float(excess.max()) <= 1e-4, float(excess.max())


# ------------------------------------------------------------------------------------------------ the cluster chain
def run_chain(dev, dt, layers, stacks, batch, x0, base, gb, fc_w, fc_b, out=None):
    L = lib()
    inp, middle = O.CONFIGS[layers]
    d = L.hf_mod_desc(layers, inp, middle, stacks, dt[0])
    from hairfastgan_b200 import modulation as M
    x0r = [M.rows(x, batch, layers, M.ROWS, "x0")[0] for x in x0]
    out = torch.empty(batch, layers, 512, device=dev) if out is None else out
    ws = workspace(d, batch, dev)
    L.check(L.lib().hf_mod_chain(C.byref(d), batch, fc_w.data_ptr(), fc_b.data_ptr(), gb.data_ptr(),
                                 (L.hf_mod_rows * 2)(*(x0r + x0r)[:2]),
                                 C.byref(M.rows(base, batch, layers, M.ROWS, "base")[0]), out.data_ptr(), ws.data_ptr(),
                                 L.stream_ptr()), "hf_mod_chain")
    return out


@pytest.mark.parametrize("batch", [1, 2, 5])
@pytest.mark.parametrize("layers", [6, 12, 18])
def test_chain_vs_operand_rounded_oracle(dev, dt, layers, batch):
    """Given gamma / beta, the chain against the oracle with the kernel's 16-bit operands: a wrong cluster rank, output
    slice or K chunk moves whole columns.  PostProcess's L = 18 runs two stacks.  Repeated calls are bit-identical."""
    stacks = 2 if layers == 18 else 1
    rows = batch * layers
    g = torch.Generator().manual_seed(100 * layers + batch)
    x0 = [torch.randn(batch, 18, 512, generator=g)[:, 18 - layers:] * torch.linspace(0.5, 2, layers)[None, :, None]
          for _ in range(stacks)]                                                  # strided row views
    base = torch.randn(batch, layers, 512, generator=g)
    gb = 0.3 * torch.randn(10 * stacks, rows, 512, generator=g)
    fc_w = torch.randn(stacks, 5, 512, 512, generator=g) / 512 ** 0.5
    fc_b = 0.1 * torch.randn(stacks, 5, 512, generator=g)
    dev_args = dict(x0=[x.to(dev) for x in x0], base=base.to(dev), gb=gb.to(dev), fc_w=fc_w.to(dt[1]).to(dev),
                    fc_b=fc_b.to(dev))
    out = run_chain(dev, dt, layers, stacks, batch, **dev_args)
    dts = []
    for s in range(stacks):
        params = [{"fc.weight": fc_w[s, i], "fc.bias": fc_b[s, i]} for i in range(5)]
        gbs = [(gb[s * 10 + 2 * i].view(batch, layers, 512), gb[s * 10 + 2 * i + 1].view(batch, layers, 512))
               for i in range(5)]
        dts.append(O.stack(x0[s], None, params, dt[1], gbs))
    dt_ref = sum(dts)
    err = float((out.cpu().double() - base.double() - 0.1 * dt_ref).abs().max() / (0.1 * dt_ref).pow(2).mean().sqrt())
    record(f"mod_chain_L{layers}_b{batch}", enc_dtype=enc_dtype_name(), max_abs_over_rms=err)
    assert err < TOL_CHAIN[enc_dtype_name()], err
    again = run_chain(dev, dt, layers, stacks, batch, **dev_args)
    assert torch.equal(again, out)


# ------------------------------------------------------------------------------------------------ drop-ins vs golden
def models(golden, dev):
    rot = O.StandInRotate(O.synth_params(int(golden["seed_rotate"]), 6), dev)
    bl = O.StandInBlending(O.synth_params(int(golden["seed_blending"]), 12), dev)
    pp = O.StandInPostProcess(O.synth_params(int(golden["seed_post_1"]), 18),
                              O.synth_params(int(golden["seed_post_2"]), 18), g64(golden, "post_latent_avg", dev),
                              dev)
    return rot, bl, pp


def drop_in_cases(golden, dev):
    """(name, call, reference output, reference base)"""
    from hairfastgan_b200 import modulation as M
    rot, bl, pp = models(golden, dev)
    out = []
    for b in (1, 2):
        wf, wt = g64(golden, f"rotate_b{b}_from", dev), g64(golden, f"rotate_b{b}_to", dev)
        out.append((f"rotate_b{b}", lambda wf=wf, wt=wt: M.rotate_forward(rot, wf[:, :6], wt[:, :6]),
                    g64(golden, f"rotate_b{b}_out"), g64(golden, f"rotate_b{b}_from")[:, :6]))
    bl_in = [g64(golden, f"blending_{k}", dev) for k in ("latent_face", "latent_color", "embed_face", "embed_color")]
    out.append(("blending", lambda: M.blending_forward(bl, *bl_in), g64(golden, "blending_out"),
                g64(golden, "blending_latent_face")))
    pp_in = [g64(golden, f"post_s_{k}", dev) for k in ("face", "hair")]
    out.append(("postprocess", lambda: M.postprocess_forward(pp, *pp_in)[0], g64(golden, "post_out"),
                g64(golden, "post_latent_avg")))
    return out


def test_drop_ins_vs_golden(dev, golden):
    res = {}
    for name, call, ref, base in drop_in_cases(golden, dev):
        y = call()
        assert y.shape == ref.shape and y.dtype == torch.float32 and y.is_cuda
        err = float((y.cpu().double() - ref).abs().max() / (ref - base).pow(2).mean().sqrt())
        res[name] = err
        record(f"modulation_{name}", enc_dtype=enc_dtype_name(), max_abs_over_rms_dt=err)
    assert all(e < TOL_DROP_IN[enc_dtype_name()] for e in res.values()), res


@pytest.mark.parametrize("batch", [2, 18])
def test_batched_drop_ins_vs_oracle(dev, golden, batch):
    """Every drop-in at B > 1 against the float64 oracle.  B = 18 equals PostProcess's L, where latent_avg [18, 512]
    has the shape of a per-sample [B, 512] row: it must still be added row by row."""
    from hairfastgan_b200 import modulation as M
    rot, bl, pp = models(golden, dev)
    g = torch.Generator().manual_seed(batch)
    lat = [torch.randn(batch, 18, 512, generator=g) * torch.linspace(0.25, 2, 18)[None, :, None] for _ in range(4)]
    emb = [torch.randn(batch, 512, generator=g) for _ in range(2)]
    rot_p = O.synth_params(int(golden["seed_rotate"]), 6)
    bl_p = O.synth_params(int(golden["seed_blending"]), 12)
    pp_p = [O.synth_params(int(golden[f"seed_post_{i}"]), 18) for i in (1, 2)]
    avg = g64(golden, "post_latent_avg")
    d = [x.to(dev) for x in lat + emb]
    cases = {"rotate": (M.rotate_forward(rot, d[0][:, :6], d[1][:, :6]),
                        O.rotate(rot_p, lat[0][:, :6], lat[1][:, :6]), lat[0][:, :6]),
             "blending": (M.blending_forward(bl, d[2][:, 6:], d[3][:, 6:], d[4], d[5]),
                          O.blending(bl_p, lat[2][:, 6:], lat[3][:, 6:], emb[0], emb[1]), lat[2][:, 6:]),
             "postprocess": (M.postprocess_forward(pp, d[0], d[1])[0],
                             O.postprocess(*pp_p, lat[0], lat[1], avg), avg.expand(batch, -1, -1))}
    res = {}
    for name, (y, ref, base) in cases.items():
        assert y.shape == ref.shape, name
        res[name] = float((y.cpu().double() - ref).abs().max() / (ref - base.double()).pow(2).mean().sqrt())
        record(f"modulation_{name}_b{batch}_vs_oracle", enc_dtype=enc_dtype_name(), max_abs_over_rms_dt=res[name])
    assert all(e < TOL_DROP_IN[enc_dtype_name()] for e in res.values()), res


def test_no_sync_no_rng_launch_count_and_determinism(dev, golden):
    L = lib()
    cases = drop_in_cases(golden, dev)
    first = [c[1]() for c in cases]                     # packs
    torch.cuda.synchronize()
    cpu_rng, cuda_rng = torch.get_rng_state(), torch.cuda.get_rng_state()
    for (name, call, _, _), y0 in zip(cases, first):
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                n0 = L.lib().hf_total_launch_count()
                y = call()
                n = L.lib().hf_total_launch_count() - n0
            finally:
                torch.cuda.set_sync_debug_mode(0)
        assert not [w for w in caught if str(w.message).startswith("called a synchronizing")], name
        assert n == LAUNCHES_PER_CALL, (name, n)
        assert torch.equal(y, y0), name
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(torch.cuda.get_rng_state(), cuda_rng)


def test_repack_on_load_state_dict(dev, golden):
    from hairfastgan_b200 import modulation as M
    rot, _, pp = models(golden, dev)
    wf = g64(golden, "rotate_b1_from", dev)[:, :6]
    wt = g64(golden, "rotate_b1_to", dev)[:, :6]
    a = M.rotate_forward(rot, wf, wt)
    sd = rot.state_dict()
    sd["modulation_module_list.4.beta_function.3.bias"] += 1.0        # beta of the last module: dt + 1
    rot.load_state_dict(sd)
    b = M.rotate_forward(rot, wf, wt)
    assert torch.allclose(b, a + 0.1, atol=1e-4)
    old = rot.modulation_module_list[4].beta_function._modules["3"]
    new = torch.nn.Linear(512, 512).to(dev)                           # a replaced submodule: beta + 1 again
    new.weight.data.copy_(old.weight)
    new.bias.data.copy_(old.bias + 1.0)
    setattr(rot.modulation_module_list[4].beta_function, "3", new)
    assert torch.allclose(M.rotate_forward(rot, wf, wt), a + 0.2, atol=1e-4)
    s = g64(golden, "post_s_face", dev)
    p0 = M.postprocess_forward(pp, s, s)[0]
    sd = pp.to_latent_2.state_dict()
    sd["4.fc.bias"] += 1.0                                            # before the last LayerNorm: no change
    sd["4.gamma_function.3.bias"] += 1.0                              # dt_hair scaled
    pp.to_latent_2.load_state_dict(sd)
    assert not torch.allclose(M.postprocess_forward(pp, s, s)[0], p0, atol=1e-3)


def test_errors(dev, golden):
    from hairfastgan_b200 import modulation as M
    rot, bl, pp = models(golden, dev)
    x = torch.randn(1, 6, 512, device=dev)
    with pytest.raises(RuntimeError, match="CUDA"):
        M.rotate_forward(rot, x, x.cpu())
    with pytest.raises(NotImplementedError):
        M.rotate_forward(rot, torch.randn(1, 7, 512, device=dev), x)
    with pytest.raises(NotImplementedError):
        M.rotate_forward(rot, x, torch.randn(2, 6, 512, device=dev))
    with pytest.raises(NotImplementedError):
        M.blending_forward(bl, torch.randn(1, 12, 512, device=dev), torch.randn(1, 12, 512, device=dev),
                           torch.randn(1, 256, device=dev), torch.randn(1, 512, device=dev))
    with pytest.raises(NotImplementedError):                          # the reference's expand / cat would raise
        M.blending_forward(bl, torch.randn(2, 12, 512, device=dev), torch.randn(2, 12, 512, device=dev),
                           torch.randn(12, 512, device=dev)[:2], torch.randn(12, 512, device=dev))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        M.rotate_forward(O.StandInRotate(O.synth_params(1, 6)), x.cpu(), x.cpu())
    wrong = O.StandInRotate(O.synth_params(1, 6), dev)
    wrong.modulation_module_list[2].last = True
    with pytest.raises(NotImplementedError):
        M.rotate_forward(wrong, x, x)


# ------------------------------------------------------------------------------------------------ whole swap
@pytest.mark.skipif(not refenv.available(), reason="reference not built (oracle/build_ref.py)")
def test_overlay_modulation_swap_matches_stock_reference(tmp_path, hf_dtype):
    """baseline/run_swap.py --mode overlay_modulation against the stock reference, at the final-image tolerance
    tests/test_gpu_swap.py states for the default dtypes (run once)."""
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

    ref, got = run("reference"), run("overlay_modulation")
    assert got["summary"]["deterministic"] and got["summary"]["finite"]
    d = (got["finals"][-1] - ref["finals"][-1]).abs()
    mean, q99, mx = float(d.mean()), float(torch.quantile(d.flatten()[::7], 0.99)), float(d.max())
    record("swap_overlay_modulation_vs_stock_reference", mean_abs=mean, q99_abs=q99, max_abs=mx,
           full_swap_ms=got["summary"]["timings"][-1]["gpu_ms"],
           reference_full_swap_ms=ref["summary"]["timings"][-1]["gpu_ms"])
    assert (mean <= SW.TOL_FINAL_MEAN["default"] and q99 <= SW.TOL_FINAL_Q99["default"]
            and mx <= SW.TOL_FINAL_MAX["default"]), (mean, q99, mx)

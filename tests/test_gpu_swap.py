"""The unmodified `HairFast(get_parser().parse_args([])).swap(face, shape, color)` of the unmodified reference
(hair_swap.py:27-105), end to end on the GPU, three ways: the stock reference (cuDNN + its JIT kernels), the same
checkout under hairfastgan_b200.install(), and under install(skip_fse_reconstruction=True).  BASELINE configs[2] /
SURVEY 8d config 3: three `torch.rand(3,1024,1024)` images (seeds 0,1,2), synthetic checkpoints
(baseline/synth_checkpoints.py), default seed 3407.

Each arm is its own process (the reference's modules are cached in sys.modules; one process = one mode).  The reference
is what oracle/build_ref.py built under oracle/_ref (git-ignored); the test skips when it is absent.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from baseline import refenv
from tests.gpu_util import ROOT, record

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not refenv.available(), reason="reference not built (oracle/build_ref.py)")]

WORK = os.environ.get("HAIRFAST_WORK", "/tmp/hairfast_work")
# "default" = nothing set in the environment: generator bf16, encoder family fp16 (what a user of install() gets)
# (HAIRFAST_SWAP_DTYPES=default,fp16,bf16 adds the forced modes: each costs two more 20 s process start-ups)
HF_DTYPES = os.environ.get("HAIRFAST_SWAP_DTYPES", "default").split(",")

# Stated tolerance of the FINAL 1024^2 image (values in [0,1]) against the stock reference run on the same GPU, same
# seeds.  The pipeline has discrete decisions (BiSeNet arg-max labels -> 256^2 masks -> F-space blends), so a small set
# of pixels near label boundaries can move by more than the arithmetic error; the bound is therefore on the mean and on
# a high quantile, with the max reported.
TOL_FINAL_MEAN = {"default": 4e-4, "bf16": 8e-4, "fp16": 1.5e-4}
TOL_FINAL_Q99 = {"default": 1.5e-3, "bf16": 2.5e-3, "fp16": 5e-4}
TOL_FINAL_MAX = {"default": 5e-3, "bf16": 8e-3, "fp16": 2e-3}
_reference_arm = {}


def _run(mode, out, extra=()):
    cmd = [sys.executable, os.path.join(ROOT, "baseline", "run_swap.py"), "--mode", mode, "--work", WORK, "--out", out,
           "--reps", "2", "--warmup", "1", *extra]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    assert p.returncode == 0, (mode, p.stdout[-2000:], p.stderr[-4000:])
    return torch.load(out, weights_only=False)


@pytest.fixture(scope="module")
def arms(tmp_path_factory, hf_dtype):
    d = tmp_path_factory.mktemp("swap")
    if "reference" not in _reference_arm:                             # the stock arm does not depend on our dtype
        _reference_arm["reference"] = _run("reference", str(d / "reference.pt"))
    res = {"reference": _reference_arm["reference"], "dtype": hf_dtype or "default"}
    res.update({m: _run(m, str(d / f"{m}.pt")) for m in ("overlay", "overlay_fast")})
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", f"swap_arms_{res['dtype']}.json"), "w") as f:
        json.dump({m: r["summary"] for m, r in res.items() if isinstance(r, dict)}, f, indent=1)
    return res


def test_swap_runs_under_overlay(arms):
    s = arms["overlay"]["summary"]
    assert s["generator_class"] == "hairfastgan_b200.model"          # the overlay really is what ran
    assert arms["reference"]["summary"]["generator_class"] == "models.stylegan2.model"
    final = arms["overlay"]["finals"][-1]
    assert final.shape == (3, 1024, 1024) and s["finite"]
    assert 0.0 <= s["final_min"] and s["final_max"] <= 1.0 and s["final_max"] - s["final_min"] > 0.05
    assert s["deterministic"], "same seed (3407) must give the same image bit for bit"


def test_swap_matches_stock_reference(arms):
    ref = arms["reference"]["finals"][-1]
    got = arms["overlay"]["finals"][-1]
    d = (got - ref).abs()
    mean, q99, mx = float(d.mean()), float(torch.quantile(d.flatten()[::7], 0.99)), float(d.max())
    emb = {}
    for k, v in arms["reference"]["embed"].items():
        w = arms["overlay"]["embed"][k]
        if v.is_floating_point():
            emb[k] = float((w - v).abs().max()) / (float(v.pow(2).mean().sqrt()) + 1e-12)
        else:
            emb[k] = float((w != v).float().mean())                   # label disagreement rate of the 256^2 masks
    dt = arms["dtype"]
    record("swap_final_vs_stock_reference", mode=dt, mean_abs=mean, q99_abs=q99, max_abs=mx,
           embed={k: round(x, 5) for k, x in emb.items()})
    assert mean <= TOL_FINAL_MEAN[dt] and q99 <= TOL_FINAL_Q99[dt] and mx <= TOL_FINAL_MAX[dt], (mean, q99, mx, emb)


def test_skip_fse_reconstruction_gives_the_same_image(arms):
    """hairfastgan_b200/fse_fast.py against the real FeatureStyleEncoder/trainer.py:357-365 (not a stand-in): the
    discarded reconstruction is skipped, its RNG draws are consumed, so the final image is bit-identical."""
    a, b = arms["overlay"], arms["overlay_fast"]
    assert torch.equal(a["finals"][-1], b["finals"][-1])
    for k, v in a["embed"].items():
        assert torch.equal(v, b["embed"][k]), k
    ta = a["summary"]["timings"][-1]["per_module_ms"].get("fse_generator", 0.0)
    tb = b["summary"]["timings"][-1]["per_module_ms"].get("fse_generator", 0.0)
    assert tb == 0.0 and ta > 0.0                                     # the forward really was skipped

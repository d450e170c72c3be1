"""The FFHQ face alignment on the GPU (hairfastgan_b200/face_align.py, csrc/hf_align.cu) against the library calls it
replaces (oracle/align_oracle.py) and the unmodified reference's outputs (tests/golden/align.npz).

Every stage is bit-exact by construction (DESIGN.md, "Face alignment"): the Lanczos passes and the QUAD transform
against Pillow, the median against np.median, the padding chain against numpy / scipy, and the whole warp against
the golden.  The blur is held to scipy bit for bit as well: the same float64 operations in the same order.
"""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from baseline import refenv
from oracle import align_oracle as O
from tests.gpu_util import ROOT, record

pytestmark = pytest.mark.gpu
HF_DTYPES = ["default"]          # nothing here depends on the 16-bit operand type
GOLD = os.path.join(os.path.dirname(__file__), "golden", "align.npz")
NAMES = list(O.CASES)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def FA():
    from hairfastgan_b200 import face_align
    return face_align


def _u8(rng, h, w):
    return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)


def _mismatch(got: np.ndarray, ref: np.ndarray):
    d = np.abs(got.astype(np.int16) - ref.astype(np.int16))
    return int(d.max()), float((d > 0).mean())


@pytest.mark.parametrize("h,w,oh,ow", [(301, 250, 150, 125), (301, 250, 100, 83), (97, 1203, 32, 401),
                                       (1024, 768, 1024, 384), (640, 480, 213, 480), (4096, 4096, 1024, 1024)])
def test_lanczos_bit_exact(dev, FA, h, w, oh, ow):
    """Shrink by 2 and 3 (the shrink branch rounds the size), one axis only, and 4096 -> 1024, on random uint8."""
    img = _u8(np.random.default_rng(h * 7 + w), h, w)
    got = FA.resample(torch.from_numpy(img).to(dev), ow, oh).cpu().numpy()
    assert np.array_equal(got, O.resample(img, ow, oh))


def test_lanczos_reads_a_crop_window(dev, FA):
    img = _u8(np.random.default_rng(5), 300, 400)
    t = torch.from_numpy(img).to(dev)
    got = FA.resample(t[17:271, 33:390], 119, 127).cpu().numpy()
    assert np.array_equal(got, O.resample(np.ascontiguousarray(img[17:271, 33:390]), 119, 127))


def _quads():
    rng = np.random.default_rng(11)
    base = np.array([[10.0, 12.0], [14.0, 230.0], [250.0, 226.0], [246.0, 8.0]])
    yield "inside", base + rng.normal(0, 0.3, base.shape), (256, 256)
    th = np.deg2rad(33.0)
    c, r = np.array([128.0, 120.0]), 150.0
    corners = [c + r * np.array([np.cos(th + a), np.sin(th + a)]) for a in np.deg2rad([225, 135, 45, 315])]
    yield "tilted_fill0", np.array(corners), (300, 300)             # corners well outside the 256^2 source
    yield "skewed_fill0", np.array([[-40.3, -20.7], [5.1, 290.2], [300.6, 240.9], [230.2, -35.5]]), (173, 411)
    yield "edges", np.array([[-0.5, -0.5], [-0.5, 255.5], [255.5, 255.5], [255.5, -0.5]]), (512, 512)


@pytest.mark.parametrize("name,quad,size", list(_quads()), ids=[q[0] for q in _quads()])
def test_quad_bit_exact(dev, FA, name, quad, size):
    img = _u8(np.random.default_rng(13), 256, 256)
    data = (quad + 0.5).flatten()
    got = FA.quad_transform(torch.from_numpy(img).to(dev), data, *size).cpu().numpy()
    ref = O.quad(img, data, *size)
    assert np.array_equal(got, ref)
    if "fill0" in name:
        assert (ref == 0).all(axis=2).mean() > 0.02                  # the fill really is exercised


def test_quad_transform_size(dev, FA):
    img = _u8(np.random.default_rng(17), 900, 700)
    quad = np.array([[60.2, 40.7], [20.9, 850.1], [690.4, 880.3], [650.8, 30.2]])
    got = FA.quad_transform(torch.from_numpy(img).to(dev), (quad + 0.5).flatten(), 4096, 4096).cpu().numpy()
    assert np.array_equal(got, O.quad(img, quad + 0.5, 4096, 4096))


@pytest.mark.parametrize("shape", [(1, 1), (7, 5), (64, 64), (513, 1001), (2100, 2100)])
def test_median_equals_numpy(dev, FA, shape):
    rng = np.random.default_rng(shape[0])
    x = (rng.random(shape + (3,)) * 255).astype(np.float32)
    x[..., 1] = np.round(x[..., 1])                                  # many ties
    x[..., 2] -= 128.0                                               # negative values
    got = FA.median(torch.from_numpy(x).to(dev)).cpu().numpy()
    ref = np.median(x, axis=(0, 1))
    assert got.dtype == ref.dtype == np.float32 and np.array_equal(got, ref), (got, ref)


@pytest.mark.parametrize("shape,sigma", [((61, 47), 0.7), ((300, 200), 3.3), ((512, 700), 16.0), ((90, 80), 30.0)])
def test_gaussian_vs_scipy(dev, FA, shape, sigma):
    """Stated bound: 0 ulp.  Summation order is scipy's symmetric order, so any difference is a defect."""
    x = (np.random.default_rng(int(sigma * 10)).random(shape + (3,)) * 255).astype(np.float32)
    got = FA.gaussian(torch.from_numpy(x).to(dev), sigma).cpu().numpy()
    ref = O.gaussian(x, sigma)
    record("align_gaussian_vs_scipy", shape=list(shape), sigma=sigma, max_abs=float(np.abs(got - ref).max()))
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("h,w,pad,blur", [(200, 180, (60, 70, 61, 59), 4.1), (964, 963, (504, 528, 504, 504), 33.6),
                                          (31, 29, (40, 12, 9, 33), 2.2)])
def test_pad_blend_bit_exact(dev, FA, h, w, pad, blur):
    """Including pads wider than the image (numpy's repeated reflection)."""
    img = _u8(np.random.default_rng(h), h, w)
    got = FA.pad_blend(torch.from_numpy(img).to(dev), pad, blur).cpu().numpy()
    assert np.array_equal(got, O.pad_blend(img, pad, blur))


@pytest.mark.parametrize("name", NAMES)
def test_align_from_landmarks_vs_golden(dev, FA, gold, name):
    data, _, _ = O.case_input(name)
    img = np.array(O.pil_input(data))
    ref = O.golden_output(gold, name)
    out = FA.align_from_landmarks(torch.from_numpy(img).to(dev), gold[f"{name}_lm"])
    assert out.dtype == torch.uint8 and out.shape == (1024, 1024, 3) and out.device == dev
    got = out.cpu().numpy()
    mx, frac = _mismatch(got, ref)
    record("align_from_landmarks_vs_golden", case=name, max_abs=mx, frac_differing=frac)
    assert np.array_equal(got, ref), (mx, frac)
    again = FA.align_from_landmarks(torch.from_numpy(img).to(dev), gold[f"{name}_lm"])
    assert torch.equal(out, again)                                   # identical run to run


@pytest.fixture(scope="module")
def shape_predictor():
    if not refenv.available():
        pytest.skip("reference not built (oracle/build_ref.py)")
    refenv.activate(overlay=False, chdir=False)
    import utils.shape_predictor as sp
    saved = sp.dlib
    yield sp
    sp.dlib = saved


@pytest.mark.parametrize("name", NAMES)
def test_drop_in_align_face_vs_golden(dev, FA, gold, shape_predictor, name):
    from torchvision import transforms as T
    data, _, _ = O.case_input(name)
    fake = O.FakeDlib([gold[f"{name}_lm"]])
    shape_predictor.dlib = fake
    ref = O.golden_output(gold, name)
    imgs = FA.align_face([data], fake.predictor, return_tensors=False)
    assert len(imgs) == 1 and imgs[0].mode == "RGB" and imgs[0].size == (1024, 1024)
    assert np.array_equal(np.asarray(imgs[0]), ref)
    tens = FA.align_face(data, fake.predictor)                       # a single input is wrapped in a list
    assert len(tens) == 1 and tens[0].device.type == "cpu" and tens[0].dtype == torch.float32
    assert torch.equal(tens[0], T.ToTensor()(imgs[0]).clamp(0, 1))


def test_align_from_landmarks_accepts_any_layout(dev, FA, gold):
    """A channels-first tensor permuted to HWC (not packed along rows) is copied, not rejected."""
    data, _, img = O.case_input("odd")
    chw = torch.from_numpy(img).permute(2, 0, 1).contiguous().to(dev)
    out = FA.align_from_landmarks(chw.permute(1, 2, 0), gold["odd_lm"])
    assert np.array_equal(out.cpu().numpy(), O.golden_output(gold, "odd"))


def test_non_rgb_inputs_raise(dev, FA, gold, shape_predictor):
    import PIL.Image
    fake = O.FakeDlib([gold["crop_lm"]])
    shape_predictor.dlib = fake
    gray = PIL.Image.fromarray(np.zeros((64, 64), np.uint8))
    with pytest.raises(NotImplementedError):
        FA.align_face([gray], fake.predictor)
    with pytest.raises(NotImplementedError):
        FA.align_face([torch.rand(1, 64, 64)], fake.predictor)      # ToPILImage gives mode 'L'
    with pytest.raises(NotImplementedError):
        FA.align_from_landmarks(torch.zeros(64, 64, 4, dtype=torch.uint8, device=dev), gold["crop_lm"])
    with pytest.raises(NotImplementedError):
        FA.align_from_landmarks(torch.zeros(64, 64, 3, device=dev), gold["crop_lm"])
    with pytest.raises(RuntimeError):
        FA.align_from_landmarks(torch.zeros(64, 64, 3, dtype=torch.uint8), gold["crop_lm"])


def test_aligned_swap_matches_stock_reference(tmp_path):
    """baseline/run_swap.py --mode overlay_align (overlay_all + install(face_align=True)) against the stock reference's
    swap(face, shape, color, align=True), at tests/test_gpu_swap.py's final-image tolerance; the three aligned inputs
    swap() returns must be identical."""
    if not refenv.available():
        pytest.skip("reference not built (oracle/build_ref.py)")
    from tests.test_gpu_swap import TOL_FINAL_MAX, TOL_FINAL_MEAN, TOL_FINAL_Q99
    work = os.environ.get("HAIRFAST_WORK", "/tmp/hairfast_work")

    def run(mode):
        out = str(tmp_path / f"{mode}.pt")
        cmd = [sys.executable, os.path.join(ROOT, "baseline", "run_swap.py"), "--mode", mode, "--work", work,
               "--out", out, "--reps", "1", "--warmup", "1"]
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
        assert p.returncode == 0, (mode, p.stdout[-2000:], p.stderr[-4000:])
        return torch.load(out, weights_only=False)
    ref, got = run("reference_align"), run("overlay_align")
    assert len(ref["aligned"]) == len(got["aligned"]) == 3
    for a, b in zip(ref["aligned"], got["aligned"]):
        assert a.shape == (3, 1024, 1024) and torch.equal(a, b)
    d = (got["finals"][-1] - ref["finals"][-1]).abs()
    mean, q99, mx = float(d.mean()), float(torch.quantile(d.flatten()[::7], 0.99)), float(d.max())
    record("swap_overlay_align_vs_stock_reference", mean_abs=mean, q99_abs=q99, max_abs=mx)
    assert mean <= TOL_FINAL_MEAN["default"] and q99 <= TOL_FINAL_Q99["default"] and mx <= TOL_FINAL_MAX["default"]

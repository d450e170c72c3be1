"""The CPU oracle of the face alignment (oracle/align_oracle.py) against tests/golden/align.npz, which the unmodified
reference align_face made (oracle/gen_golden_align.py): every case bit for bit, and the host geometry of
hairfastgan_b200.face_align gives the reference's integer shrink, crop and pad boxes."""
from __future__ import annotations

import os

import numpy as np
import pytest

from oracle import align_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden", "align.npz")
NAMES = list(O.CASES)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _case(gold, name):
    data, lm, img = O.case_input(name)
    assert np.array_equal(lm, gold[f"{name}_lm"]), "landmark template changed since the golden was made"
    return np.asarray(O.pil_input(data)), gold[f"{name}_lm"]


def test_golden_covers_every_branch(gold):
    names = [str(n) for n in gold["case_names"]]
    assert names == NAMES
    assert any((gold[f"{n}_rsize"] >= 0).all() for n in names), "no shrink case"
    assert any((gold[f"{n}_pad"] >= 0).all() for n in names), "no padding case"
    assert any((gold[f"{n}_crop"] >= 0).all() and (gold[f"{n}_pad"] < 0).all() for n in names), "no crop-only case"
    assert any(gold[f"{n}_params"][0] != gold[f"{n}_params"][1] and gold[f"{n}_params"][0] % 2 for n in names)


@pytest.mark.parametrize("name", NAMES)
def test_geometry_gives_reference_boxes(gold, name):
    from hairfastgan_b200 import face_align as FA
    img, lm = _case(gold, name)
    g = FA.geometry(lm, (img.shape[1], img.shape[0]))
    b = O.boxes(lm, (img.shape[1], img.shape[0]))
    assert tuple(gold[f"{name}_rsize"]) == (g.rsize or (-1, -1)) == (b["rsize"] or (-1, -1))
    assert tuple(gold[f"{name}_crop"]) == (g.crop or (-1,) * 4) == (b["crop"] or (-1,) * 4)
    assert tuple(gold[f"{name}_pad"]) == (g.pad or (-1,) * 4) == (b["pad"] or (-1,) * 4)
    assert np.array_equal(g.quad, b["quad"]) and g.blur == b["blur"]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_golden(gold, name):
    img, lm = _case(gold, name)
    out = O.align(img, lm)
    assert out.dtype == np.uint8 and out.shape == (1024, 1024, 3)
    assert np.array_equal(out, O.golden_output(gold, name))


def test_float_case_is_truncated_by_to_pil(gold):
    """ToPILImage's mul(255).byte() truncates: the float case's pixels are the uint8 levels it was made from, where
    rounding would have moved about half of them up by one."""
    data, _, img = O.case_input("float_tensor")
    assert np.array_equal(np.asarray(O.pil_input(data)), img)
    rounded = np.clip(np.rint(data.permute(1, 2, 0).numpy().astype(np.float64) * 255), 0, 255).astype(np.uint8)
    assert (rounded != img).mean() > 0.3


def test_geometry_restatement_matches_numpy_on_random_faces():
    """Random landmark sets (rolls, scales, positions, image sizes): the host geometry equals the oracle's boxes."""
    from hairfastgan_b200 import face_align as FA
    rng = np.random.default_rng(7)
    for _ in range(200):
        w, h = int(rng.integers(200, 5000)), int(rng.integers(200, 5000))
        io = float(rng.uniform(20, 0.6 * min(w, h)))
        lm = O.synth_landmarks((rng.uniform(0, w), rng.uniform(0, h)), io, rng.uniform(-60, 60))
        g, b = FA.geometry(lm, (w, h)), O.boxes(lm, (w, h))
        assert (g.rsize, g.crop, g.pad) == (b["rsize"], b["crop"], b["pad"])
        assert np.array_equal(g.quad, b["quad"]) and g.blur == b["blur"]


def test_numpy_reflect_pad_beyond_one_period():
    """np.pad 'reflect' wider than the image repeats the mirror with period 2 (n - 1): what hf_align.cu's
    numpy_reflect computes (pads wider than the crop only occur for faces near tiny images, but must not differ)."""
    x = np.arange(5)
    padded = np.pad(x, (13, 11), "reflect")
    period = 2 * (len(x) - 1)
    idx = np.mod(np.arange(-13, 5 + 11), period)
    assert np.array_equal(padded, x[np.where(idx < len(x), idx, period - idx)])


def test_gaussian_is_the_symmetric_double_sum():
    """scipy's gaussian_filter equals the float64 sum w0 x_i + sum_{j=r..1} w_j (x_{i-j} + x_{i+j}) per axis in that
    order, rounded to float32 after each axis -- what hf_align.cu's blur computes, so the GPU may match bit for bit."""
    from hairfastgan_b200 import face_align as FA
    rng = np.random.default_rng(3)
    x = (rng.random((61, 47, 3)) * 255).astype(np.float32)
    for sigma in (0.7, 3.3, 9.1):
        w = FA.gaussian_half_kernel(sigma)
        r = len(w) - 1

        def axis(a, ax):
            a = np.moveaxis(a, ax, 0).astype(np.float64)
            n = a.shape[0]
            i = np.arange(n)

            def refl(k):
                k = np.mod(k, 2 * n)
                return np.where(k < n, k, 2 * n - 1 - k)
            o = a * w[0]
            for j in range(r, 0, -1):
                o = o + (a[refl(i - j)] + a[refl(i + j)]) * w[j]
            return np.moveaxis(o.astype(np.float32), 0, ax)
        assert np.array_equal(O.gaussian(x, sigma), axis(axis(x, 0), 1)), sigma

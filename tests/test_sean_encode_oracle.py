"""SEAN encode_sean: the CPU oracle against the golden of the unmodified reference, the forms the CUDA path runs (in
float64), the plans of the five Zencoder convolutions, and the opt-in overlay binding (no GPU needed)."""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sean_encode_oracle as EO
from oracle import sean_oracle as SO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sean_encode.npz")
TAPS = ("in1", "in2", "in3", "in4", "pre_tanh")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def params(golden):
    p = SO.synth_sean_params(int(golden["seed"]))
    assert len(p) == int(golden["n_keys"])
    return p


def golden_case(golden, case):
    labels = torch.from_numpy(golden[f"c{case}_labels"].astype(np.int64))
    images = EO.golden_images(int(golden[f"c{case}_image_seed"]), labels.shape[0])
    return images, labels


@pytest.mark.parametrize("case", [0, 1])
def test_encode_ref_matches_reference_golden(golden, params, case):
    images, labels = golden_case(golden, case)
    codes, taps = EO.encode_ref(params, images, labels)
    ref = torch.from_numpy(golden[f"c{case}_codes"])
    assert codes.shape == ref.shape == (labels.shape[0], 19, 512)
    assert float((codes - ref).abs().max()) < 1e-5
    assert torch.equal(codes == 0, ref == 0)                       # the zero rows are the reference's
    for name in TAPS:
        g = torch.from_numpy(golden[f"c{case}_{name}"])
        assert float((EO.golden_sample_enc(taps[name]) - g).abs().max()) <= 1e-4 * float(g.abs().max()) + 1e-5, name


def test_golden_label_cases(golden):
    l0, l1 = golden["c0_labels"], golden["c1_labels"]
    assert len(np.unique(l0[0])) == 19 and len(np.unique(l0[1])) < 19
    codes0, codes1 = golden["c0_codes"], golden["c1_codes"]
    absent = sorted(set(range(19)) - set(np.unique(l0[1]).tolist()))
    assert absent and (np.abs(codes0[1, absent]).sum(1) == 0).all() and (np.abs(codes0[0]).sum(1) > 0).all()
    j = int(golden["odd_only_class"])
    assert (l1[0, 0] == j).any() and not (l1[0, 0, ::2, ::2] == j).any()      # present at 256^2, absent at 128^2
    assert np.abs(codes1[0, j]).sum() == 0


def test_instance_norm_cancels_the_conv_bias():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 64, 16, 16, generator=g, dtype=torch.float64) * 3 + 1
    b = torch.randn(1, 64, 1, 1, generator=g, dtype=torch.float64) * 5
    ref = F.leaky_relu(F.instance_norm(x + b, eps=1e-5), 0.2)
    torch.testing.assert_close(EO.instance_norm_lrelu(x), ref, rtol=1e-12, atol=1e-12)
    # the variance of the centred values, not E[x^2] - E[x]^2: same result on a large offset
    torch.testing.assert_close(EO.instance_norm_lrelu(x + 1e4), ref, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("cin,cout,h,w", [(128, 256, 8, 8), (32, 64, 5, 7)])
def test_four_parity_form_is_conv_transpose(cin, cout, h, w):
    g = torch.Generator().manual_seed(cin + h)
    x = torch.randn(2, cin, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(cin, cout, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, wt, None, stride=2, padding=1, output_padding=1)
    torch.testing.assert_close(EO.conv_transpose_four_parity(x, wt), ref, rtol=1e-12, atol=1e-12)


def test_class_means_equal_the_reference_loop(golden):
    """EO.class_means over label_map(labels, 128) against Zencoder.forward's loop (architecture.py:178-205)."""
    _, labels = golden_case(golden, 0)
    _, l1 = golden_case(golden, 1)
    labels = torch.cat([labels, l1])
    g = torch.Generator().manual_seed(3)
    codes = torch.tanh(torch.randn(3, 64, 128, 128, generator=g, dtype=torch.float64))
    seg = F.interpolate(SO.one_hot(labels).double(), size=codes.shape[2:], mode="nearest")
    ref = torch.zeros(3, 19, 64, dtype=torch.float64)
    for i in range(3):
        for j in range(19):
            area = int(seg.bool()[i, j].sum())
            if area > 0:
                ref[i, j] = codes[i].masked_select(seg.bool()[i, j]).reshape(64, area).mean(1)
    got = EO.class_means(codes, labels)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    assert torch.equal(got == 0, ref == 0)


# ------------------------------------------------------------------------------------------------ plans
@pytest.fixture(scope="module")
def lib():
    from hairfastgan_b200 import build
    build.build()
    from hairfastgan_b200 import _lib
    return _lib


SHIFT, TAP = 2, 0          # plan out[4]: activation ring slots of the column-shift mainloop, 0 on the per-tap one
# (name, cin, cout, cin_pad, stride, prepadded, transposed, stored input H = W, kchunk, mainloop, output H = W)
ZENCODER = [("model.1", 3, 32, 32, 1, 1, 0, 258, 32, SHIFT, 256), ("model.4", 32, 64, 32, 2, 0, 0, 256, 32, TAP, 128),
            ("model.7", 64, 128, 64, 2, 0, 0, 128, 64, TAP, 64), ("model.10", 128, 256, 128, 2, 0, 1, 64, 64, SHIFT, 128),
            ("model.14", 256, 512, 256, 1, 1, 0, 130, 64, SHIFT, 128)]


@pytest.mark.parametrize("batch", [1, 2])
def test_zencoder_convolutions_are_planned(lib, batch):
    for name, cin, cout, cin_pad, stride, pre, tr, h, kchunk, loop, ho in ZENCODER:
        d = lib.hf_conv2d_desc(cin, cout, cin_pad, 3, stride, 1, lib.HF_F16, pre, tr)
        out = (C.c_int * 12)()
        assert lib.lib().hf_conv2d_plan_query(C.byref(d), batch, h, h, out) == 0, (name, lib.lib().hf_last_error())
        n_tile, n_n, a_slots, work, kc = out[1], out[2], out[4], out[9], out[11]
        assert (kc, a_slots) == (kchunk, loop), (name, list(out))
        ntot = 4 * cout if tr else cout
        assert n_tile * n_n == ntot, (name, list(out))
        m_pixels = (h if tr else ho) ** 2 * batch          # GEMM rows: input pixels of the transposed form
        assert work * n_tile == m_pixels // 128 * ntot, (name, list(out))
        if tr:
            assert n_tile == 128, name                         # four parities of 32 channels per N tile


def test_new_descriptor_fields_are_checked(lib):
    out = (C.c_int * 12)()
    for args in [(64, 64, 64, 1, 1, 1, 1, 0), (64, 64, 64, 3, 2, 1, 1, 0), (64, 64, 64, 3, 1, 1, 0, 1),
                 (64, 64, 64, 3, 2, 2, 0, 1), (64, 64, 64, 3, 2, 1, 1, 1), (64, 64, 64, 3, 1, 1, 2, 0)]:
        cin, cout, pad, k, stride, groups, pre, tr = args
        d = lib.hf_conv2d_desc(cin, cout, pad, k, stride, groups, lib.HF_F16, pre, tr)
        assert lib.lib().hf_conv2d_plan_query(C.byref(d), 1, 16, 16, out) != 0, args
    d = lib.hf_conv2d_desc(64, 64, 64, 3, 1, 1, lib.HF_F16, 1, 0)
    assert lib.lib().hf_conv2d_plan_query(C.byref(d), 1, 2, 18, out) != 0          # nothing left after the border
    assert "prepadded" in lib.lib().hf_last_error().decode()
    # the packed operand of the transposed form holds the four parities
    d = lib.hf_conv2d_desc(128, 256, 128, 3, 2, 1, lib.HF_F16, 0, 1)
    assert lib.lib().hf_conv2d_packed_bytes(C.byref(d)) == 4 * 256 * 9 * 128 * 2


# ------------------------------------------------------------------------------------------------ overlay binding
def _fake_reference(tmp_path):
    pkg = tmp_path / "models"
    (pkg / "sean_codes" / "models").mkdir(parents=True)
    for d in (pkg, pkg / "sean_codes", pkg / "sean_codes" / "models"):
        (d / "__init__.py").write_text("")
    (pkg / "sean_codes" / "models" / "pix2pix_model.py").write_text(
        "def decode_sean(sean_model, image_code, target_mask): return 'reference'\n"
        "def encode_sean(sean_model, images, labels): return 'reference'\n")
    (pkg / "Alignment.py").write_text(
        "from models.sean_codes.models.pix2pix_model import encode_sean, decode_sean\n")


@pytest.mark.parametrize("flags", [{"sean_encode": True}, {"sean": True}, {"sean": True, "sean_encode": True}])
@pytest.mark.parametrize("order", ["pix2pix_first", "alignment_first"])
def test_install_binds_only_the_chosen_names(tmp_path, flags, order):
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.sean as S
    _fake_reference(tmp_path)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.")}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install(**flags)
        names = ["models.sean_codes.models.pix2pix_model", "models.Alignment"]
        for n in (names if order == "pix2pix_first" else names[::-1]):
            importlib.import_module(n)
        mods = [sys.modules[n] for n in names]
        for fn in ("encode_sean", "decode_sean"):
            want = flags.get("sean_encode" if fn == "encode_sean" else "sean", False)
            for m in mods:
                assert (getattr(m, fn) is getattr(S, fn)) == want, (m.__name__, fn)
        inst.uninstall()
        for m in mods:
            assert m.encode_sean(None, None, None) == "reference" and m.decode_sean(None, None, None) == "reference"
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_encode_sean_rejects_cpu_tensors(params):
    from hairfastgan_b200 import sean as S
    m = SO.stand_in_model({k: v for k, v in params.items() if k.startswith("Zencoder.")}, torch.device("cpu"))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.encode_sean(m, torch.zeros(2, 3, 256, 256), torch.zeros(2, 1, 256, 256))

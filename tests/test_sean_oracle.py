"""SEAN decode_sean: the CPU oracle against the golden of the unmodified reference, the lookup-table algebra the CUDA
path implements, and the opt-in overlay binding (no GPU needed)."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sean_oracle as SO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sean.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def params(golden):
    p = SO.synth_sean_params(int(golden["seed"]))
    assert len(p) == int(golden["n_keys"])
    return p


@pytest.mark.parametrize("case", [0, 1])
def test_oracle_matches_reference_golden(golden, params, case):
    labels = torch.from_numpy(golden[f"c{case}_labels"].astype(np.int64))
    noise = SO.golden_noise(int(golden[f"c{case}_noise_seed"]))
    head = np.stack([d.reshape(-1)[:16].numpy() for d in noise])
    assert np.array_equal(head, golden[f"c{case}_noise_head"])          # the draws the reference consumed
    img, taps = SO.decode_ref(dict(params), torch.from_numpy(golden[f"c{case}_code"]), labels,
                              torch.from_numpy(golden["mean_codes"]), noise)
    ref = torch.from_numpy(golden[f"c{case}_image"])
    assert float((SO.golden_sample_image(img) - ref).abs().max()) < 1e-4
    for name, t in taps.items():
        sub = SO.golden_sample_block(t)
        g = torch.from_numpy(golden[f"c{case}_{name}"])
        assert float((sub - g).abs().max()) <= 1e-4 * float(g.abs().max()) + 1e-5, name


def test_golden_exercises_every_term(golden, params):
    # all 19 classes in case 0, some absent in case 1; all-zero code rows select the mean codes
    assert len(np.unique(golden["c0_labels"])) == 19 and len(np.unique(golden["c1_labels"])) < 19
    assert (np.abs(golden["c0_code"][0]).sum(1) == 0).any()
    for k, v in params.items():
        if k.endswith(("noise_var", "blending_gamma", "blending_beta")):
            assert float(v.abs().min()) > 0, k
    img = golden["c0_image"]
    assert 0.1 < float(np.sqrt((img ** 2).mean())) < 0.9       # tanh not saturated


def _random_labels(res, classes, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.tensor(classes)[torch.randint(0, len(classes), (res, res), generator=g)]


@pytest.mark.parametrize("res", [8, 16])
def test_onehot_conv_is_table_lookup(res):
    g = torch.Generator().manual_seed(res)
    w, b = torch.randn(64, 19, 3, 3, generator=g), torch.randn(64, generator=g)
    L = _random_labels(res, list(range(19)), res)
    plain = F.conv2d(F.one_hot(L, 19).permute(2, 0, 1)[None].float(), w, b, padding=1)[0]
    np.testing.assert_allclose(SO.onehot_conv_lut(L, w, b).numpy(), plain.numpy(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("classes", [list(range(19)), [0, 1, 4, 13, 17]])
def test_style_conv_is_table_gather(classes):
    """conv2d(middle_avg) with middle_avg[:, p] = mu[L(p)] (zero padding at the borders) equals the 9-tap gather of
    T[j][tap] = W[:, :, tap] . mu_j; classes absent from the map are never gathered."""
    g = torch.Generator().manual_seed(len(classes))
    w, b = torch.randn(32, 512, 3, 3, generator=g) / 48, torch.randn(32, generator=g)
    mu = torch.relu(torch.randn(19, 512, generator=g))
    L = _random_labels(16, classes, 3)
    middle_avg = mu[L].permute(2, 0, 1)[None]
    plain = F.conv2d(middle_avg, w, b, padding=1)[0]
    mu_absent_poisoned = mu.clone()
    for j in set(range(19)) - set(classes):
        mu_absent_poisoned[j] = float("nan")
    lut = SO.style_conv_lut(L, w, b, mu_absent_poisoned)
    np.testing.assert_allclose(lut.numpy(), plain.numpy(), rtol=1e-4, atol=1e-4)


def test_label_map_is_nearest_interpolation():
    L = _random_labels(256, list(range(19)), 9)[None, None]
    oh = F.one_hot(L[0, 0], 19).permute(2, 0, 1)[None].float()
    for r in (8, 32, 256):
        ref = F.interpolate(oh, size=(r, r), mode="nearest")[0].argmax(0)
        assert torch.equal(SO.label_map(L, r), ref)


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


@pytest.mark.parametrize("order", ["pix2pix_first", "alignment_first"])
def test_install_sean_rebinds_and_uninstall_restores(tmp_path, order):
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.sean as S
    _fake_reference(tmp_path)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.")}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install(sean=True)
        names = ["models.sean_codes.models.pix2pix_model", "models.Alignment"]
        mods = [importlib.import_module(n) for n in (names if order == "pix2pix_first" else names[::-1])]
        p2p, al = sys.modules[names[0]], sys.modules[names[1]]
        assert p2p.decode_sean is S.decode_sean and al.decode_sean is S.decode_sean
        assert p2p.encode_sean(None, None, None) == "reference" and al.encode_sean is p2p.encode_sean
        inst.uninstall()
        assert p2p.decode_sean(None, None, None) == "reference"
        assert al.decode_sean(None, None, None) == "reference"
        assert len(mods) == 2
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_install_without_sean_keeps_reference_decode(tmp_path):
    import hairfastgan_b200.install as inst
    _fake_reference(tmp_path)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.")}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install()
        al = importlib.import_module("models.Alignment")
        p2p = sys.modules["models.sean_codes.models.pix2pix_model"]
        assert al.decode_sean(None, None, None) == "reference"
        assert p2p.decode_sean(None, None, None) == "reference"
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_unsupported_sean_options_raise():
    import types
    from hairfastgan_b200 import sean as S
    opt = types.SimpleNamespace(**S.SUPPORTED_OPT)
    S.check_opt(opt)
    for k, v in [("ngf", 32), ("num_upsampling_layers", "more"), ("norm_G", "spectralspadeinstance3x3"),
                 ("no_instance", False), ("label_nc", 18)]:
        bad = types.SimpleNamespace(**{**S.SUPPORTED_OPT, k: v})
        with pytest.raises(NotImplementedError):
            S.check_opt(bad)

"""HairFast's latent modulation nets without a GPU: the float64 oracle against the golden of the unmodified reference
(tests/golden/modulation.npz, oracle/gen_golden_modulation.py), PixelNorm's dimension, the split-K plans of every
style GEMM shape, the descriptor's dtype check, and the install bindings."""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from oracle import modulation_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "modulation.npz")
H100_SMS = 132


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def t(golden, key):
    return torch.from_numpy(golden[key]).double()


def max_rel(a, b):
    return float((a - b).abs().max() / b.pow(2).mean().sqrt())


def oracle_cases(golden, pixel_dim=1):
    """(name, oracle result, golden result) of every case."""
    rot = O.synth_params(int(golden["seed_rotate"]), 6)
    out = []
    for b in (1, 2):
        wf, wt = t(golden, f"rotate_b{b}_from"), t(golden, f"rotate_b{b}_to")
        out.append((f"rotate_b{b}", O.rotate(rot, wf[:, :6], wt[:, :6], pixel_dim=pixel_dim),
                    t(golden, f"rotate_b{b}_out")))
    if pixel_dim == 1:
        bl = O.synth_params(int(golden["seed_blending"]), 12)
        out.append(("blending", O.blending(bl, t(golden, "blending_latent_face"), t(golden, "blending_latent_color"),
                                           t(golden, "blending_embed_face"), t(golden, "blending_embed_color")),
                    t(golden, "blending_out")))
        p1, p2 = (O.synth_params(int(golden[f"seed_post_{i}"]), 18) for i in (1, 2))
        out.append(("postprocess", O.postprocess(p1, p2, t(golden, "post_s_face"), t(golden, "post_s_hair"),
                                                 t(golden, "post_latent_avg")), t(golden, "post_out")))
    return out


def test_golden_is_small_and_complete(golden):
    assert os.path.getsize(GOLDEN) < 1 << 20
    assert golden["rotate_b2_from"].shape == (2, 18, 512) and golden["rotate_b1_out"].shape == (1, 6, 512)
    assert golden["blending_out"].shape == (1, 12, 512) and golden["blending_embed_face"].shape == (1, 512)
    assert golden["post_out"].shape == (1, 18, 512) and golden["post_latent_avg"].shape == (18, 512)


def test_oracle_matches_golden(golden):
    for name, got, ref in oracle_cases(golden):
        assert got.shape == ref.shape, name
        assert max_rel(got, ref) < 1e-5, (name, max_rel(got, ref))


def test_pixel_norm_over_the_wrong_dimension_is_caught(golden):
    """The golden latents have rows of different scales: PixelNorm over the 512 channels instead of the L rows
    (models/stylegan2/model.py:21 normalises dim 1) moves the result far outside the oracle's agreement."""
    for name, got, ref in oracle_cases(golden, pixel_dim=2):
        assert max_rel(got, ref) > 1e-2, (name, max_rel(got, ref))


def test_operand_rounded_mode_is_close(golden):
    """The operand-rounded oracle stays within 16-bit rounding of the exact one (a sanity bound for the GPU tests)."""
    rot = O.synth_params(int(golden["seed_rotate"]), 6)
    wf, wt = t(golden, "rotate_b2_from")[:, :6], t(golden, "rotate_b2_to")[:, :6]
    exact = O.rotate(rot, wf, wt)
    for rnd, bound in ((torch.float16, 1e-2), (torch.bfloat16, 5e-2)):
        err = max_rel(O.rotate(rot, wf, wt, rnd=rnd), exact)
        assert 0 < err < bound, (rnd, err)


@pytest.fixture(scope="module")
def lib():
    from hairfastgan_b200 import build
    build.build()
    from hairfastgan_b200 import _lib
    return _lib


CONFIGS = [(6, 512, 512, 1), (12, 1536, 1024, 1), (18, 512, 512, 2)]


@pytest.mark.parametrize("batch", [1, 2, 5, 32])
@pytest.mark.parametrize("layers,inp,middle,stacks", CONFIGS)
def test_gemm_plans_without_device(lib, layers, inp, middle, stacks, batch):
    """Layer 1: stacks groups of [10 middle, inp]; layer 2: 10 stacks groups of [512, middle].  Row tile 8 when the
    rows fit, splits within the K tiles (at least 4 per split) and about two CTAs per SM over all groups."""
    h = lib.lib()
    d = lib.hf_mod_desc(layers, inp, middle, stacks, lib.HF_F16)
    rows = batch * layers
    for layer, groups, k, cout in ((1, stacks, inp, 10 * middle), (2, 10 * stacks, middle, 512)):
        out = (C.c_int * 5)()
        assert h.hf_mod_gemm_plan(C.byref(d), batch, layer, H100_SMS, out) == 0, h.hf_last_error()
        bn, splits, kt, gm, gn = list(out)
        assert bn == (8 if rows <= 8 else 64) and kt == k // 64 and gm == cout // 128 and gn == -(-rows // bn)
        assert 1 <= splits and (splits == 1 or kt // splits >= 4)
        assert splits == 1 or groups * gm * gn * (splits - 1) < 2 * H100_SMS
    assert h.hf_mod_gemm_plan(C.byref(d), batch, 3, H100_SMS, out) == -1 and b"layer 3" in h.hf_last_error()


def test_descriptor_checks_without_device(lib):
    h = lib.lib()
    out = (C.c_int * 5)()
    for bad, msg in (((7, 512, 512, 1), b"layers"), ((25, 512, 512, 1), b"layers"), ((6, 1536, 512, 2), b"inp"),
                     ((6, 512, 768 + 1, 1), b"middle"), ((6, 512, 512, 3), b"stacks")):
        d = lib.hf_mod_desc(*bad, lib.HF_BF16)
        rc = h.hf_mod_gemm_plan(C.byref(d), 1, 1, H100_SMS, out)
        if bad[0] == 7:
            assert rc == 0                     # the kernels take any L up to 24; the Python drop-ins take 6, 12, 18
            continue
        assert rc == -1 and msg in h.hf_last_error(), (bad, h.hf_last_error())


def test_every_descriptor_dtype_is_checked_first(lib):
    """The hf_mod_* calls carry the dtype in hf_mod_desc; each rejects a bad one before its other argument checks."""
    h = lib.lib()
    calls = {"hf_mod_gemm_plan": (1, 1, H100_SMS, (C.c_int * 5)()),
             "hf_mod_embed16": (1, None, None, None),
             "hf_mod_gemm": (1, 1) + (None,) * 6,
             "hf_mod_hidden": (1,) + (None,) * 8,
             "hf_mod_chain": (1,) + (None,) * 8}
    for bad in (2, -1):
        d = lib.hf_mod_desc(6, 512, 512, 1, bad)
        for name, args in calls.items():
            assert getattr(h, name)(C.byref(d), *args) == -1, name
            assert h.hf_last_error() == f"{name}: bad dtype {bad}".encode(), (name, h.hf_last_error())
        assert h.hf_mod_workspace_bytes(C.byref(d), 1) == 0


def test_cpu_module_and_unsupported_shapes_raise(golden):
    from hairfastgan_b200 import modulation as M
    rot = O.StandInRotate(O.synth_params(1, 6))
    x = torch.randn(1, 6, 512)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        M.rotate_forward(rot, x, x)
    with pytest.raises(NotImplementedError):
        M.rotate_forward(rot, torch.randn(1, 7, 512), x)
    other = O.StandInRotate(O.synth_params(1, 6))
    other.modulation_module_list[0].fc = torch.nn.Linear(512, 256)
    with pytest.raises(NotImplementedError, match="ModulationModule"):
        M.rotate_forward(other, x, x)
    assert set(M.stack_shapes(12)) == set(O.stack_state_dict(O.synth_params(2, 12)))
    # each caller names the broadcast it means: a [12, 512] CLIP embedding at B = 2, or a per-sample row passed as
    # latent_avg, is rejected rather than read in the other form
    with pytest.raises(NotImplementedError):
        M.rows(torch.zeros(12, 512), 2, 12, M.PER_SAMPLE, "embedding")
    with pytest.raises(NotImplementedError):
        M.rows(torch.zeros(2, 512), 2, 18, M.PER_LAYER, "latent_avg")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        M.rows(torch.zeros(18, 512), 18, 18, M.PER_LAYER, "latent_avg")


_ENCODERS_STUB = '''
import torch
from torch import nn
class FeatureiResnet: pass
class ModulationModule(nn.Module):
    def __init__(self, layernum, last=False, inp=512, middle=512):
        super().__init__()
        self.fc = nn.Linear(4, 4)
class RotateModel(nn.Module):
    def __init__(self):
        super().__init__()
        self.modulation_module_list = nn.ModuleList([ModulationModule(6, i == 4) for i in range(5)])
    def forward(self, latent_from, latent_to):
        return "reference rotate"
class ClipBlendingModel(nn.Module):
    def forward(self, latent_face, latent_color, target_face, hair_color):
        return "reference blending"
class PostProcessModel(nn.Module):
    def forward(self, source, target):
        return "reference postprocess"
'''


@pytest.mark.parametrize("postprocess", [True, False])
def test_install_wraps_the_three_forwards(tmp_path, postprocess):
    """install(modulation=True) wraps the three forwards of models.Encoders after import (the module stays the
    reference's; a stand-in package plays it here), independently of install(postprocess=...); uninstall() restores
    them; the state-dict keys are unchanged."""
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.modulation as M
    import hairfastgan_b200.postprocess as P
    pkg = tmp_path / "models"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "Net.py").write_text("class FeatureEncoder: pass\nclass FeatureEncoderMult(FeatureEncoder): pass\n")
    (pkg / "Encoders.py").write_text("from models.Net import FeatureEncoderMult\n" + _ENCODERS_STUB)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.")}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install(postprocess=postprocess)
        enc = importlib.import_module("models.Encoders")
        keys = list(enc.RotateModel().state_dict())
        assert enc.RotateModel.forward.__module__ == "models.Encoders"         # off by default
        inst.uninstall()
        inst.install(postprocess=postprocess, modulation=True)                  # already imported: wrapped in place
        for cls, fn in ((enc.RotateModel, M.rotate_forward), (enc.ClipBlendingModel, M.blending_forward),
                        (enc.PostProcessModel, M.postprocess_forward)):
            assert cls.forward.__module__ == "hairfastgan_b200.modulation" and cls.forward.__doc__ == fn.__doc__
            assert cls.forward.__wrapped__.__module__ == "models.Encoders"
        assert (enc.FeatureiResnet is P.FeatureiResnet) == postprocess
        assert list(enc.RotateModel().state_dict()) == keys
        inst.uninstall()
        assert enc.RotateModel().forward(None, None) == "reference rotate"
        assert enc.ClipBlendingModel().forward(None, None, None, None) == "reference blending"
        assert enc.PostProcessModel().forward(None, None) == "reference postprocess"
        assert enc.FeatureiResnet.__module__ == "models.Encoders"
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        inst.install(postprocess=postprocess, modulation=True)                  # imported later: wrapped on import
        enc = importlib.import_module("models.Encoders")
        assert hasattr(enc.ClipBlendingModel.forward, "__wrapped__")
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)

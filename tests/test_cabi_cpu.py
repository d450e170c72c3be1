"""CPU-side checks (no GPU): the C-ABI library builds for sm_90a, loads, exports every symbol that
include/hairfast_b200.h declares, validates arguments without touching a device, and the host-side
mirrors of the reference interface keep the reference's names / signatures / state_dict layout."""
import ctypes as C
import inspect
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from hairfastgan_b200 import build
    build.build()
    from hairfastgan_b200 import _lib
    return _lib


def test_header_symbols_all_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "hairfast_b200.h")).read()
    declared = set(re.findall(r"\b(hf_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(lib.SYMBOLS), declared ^ set(lib.SYMBOLS)
    handle = lib.lib()
    for name in declared:
        assert hasattr(handle, name), name
    assert handle.hf_version() == 90


def test_library_contains_hopper_sass(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    for mnemonic in ("HGMMA", "UTMALDG", "SYNCS"):      # wgmma, TMA load, mbarrier
        assert mnemonic in out, mnemonic


def test_argument_validation_without_device(lib):
    h = lib.lib()
    d = lib.hf_conv_desc(64, 48, 3, 0, lib.HF_BF16)       # Cout % 32 != 0
    assert h.hf_conv_packed_bytes(C.byref(d)) == 0
    assert b"multiples of 32" in h.hf_last_error()
    d = lib.hf_conv_desc(64, 64, 3, 0, lib.HF_BF16)
    assert h.hf_conv_packed_bytes(C.byref(d)) == 64 * 9 * 64 * 2 + 64 * 64 * 4
    d = lib.hf_conv_desc(64, 32, 3, 1, lib.HF_F16)
    assert h.hf_conv_packed_bytes(C.byref(d)) == 4 * 32 * 9 * 64 * 2 + 32 * 64 * 4
    cfg = lib.hf_gen_config(1024, 512, 2, lib.HF_BF16)
    nbytes = h.hf_generator_packed_bytes(C.byref(cfg))
    assert 100e6 < nbytes < 260e6          # 16-bit GEMM operands (4x for the polyphase up-convs) + fp32 tables
    ws1, ws4 = h.hf_generator_workspace_bytes(C.byref(cfg), 1), h.hf_generator_workspace_bytes(C.byref(cfg), 4)
    assert 100e6 < ws1 < 400e6 and 3.5 * ws1 < ws4 < 4.5 * ws1
    bad = lib.hf_gen_config(1000, 512, 2, lib.HF_BF16)
    assert h.hf_generator_packed_bytes(C.byref(bad)) == 0 and b"size 1000" in h.hf_last_error()
    assert h.hf_upfirdn2d_f32(None, None, None, 1, 4, 4, 4, 4, 1, 1, 1, 1, 0, 0, 0, 0, None) != 0
    assert h.hf_upfirdn2d_f32(None, None, None, 0, 4, 4, 4, 4, 1, 1, 1, 1, 0, 0, 0, 0, None) == 0   # empty input


def test_module_surface_matches_reference_signatures():
    """Same ctor / forward parameter names and defaults as models/stylegan2/model.py (SURVEY 8b)."""
    import hairfastgan_b200.model as M
    import hairfastgan_b200.op as op
    assert list(inspect.signature(op.upfirdn2d).parameters) == ["input", "kernel", "up", "down", "pad"]
    assert list(inspect.signature(op.fused_leaky_relu).parameters) == ["input", "bias", "negative_slope", "scale"]
    assert list(inspect.signature(op.FusedLeakyReLU.__init__).parameters) == ["self", "channel", "negative_slope", "scale"]
    fwd = inspect.signature(M.Generator.forward)
    assert list(fwd.parameters) == ["self", "styles", "return_latents", "inject_index", "truncation",
                                    "truncation_latent", "input_is_latent", "noise", "randomize_noise", "layer_in",
                                    "skip", "start_layer", "end_layer", "return_rgb"]
    assert fwd.parameters["end_layer"].default == 8 and fwd.parameters["randomize_noise"].default is True
    assert list(inspect.signature(M.ModulatedConv2d.__init__).parameters) == [
        "self", "in_channel", "out_channel", "kernel_size", "style_dim", "demodulate", "upsample", "downsample",
        "blur_kernel"]
    assert list(inspect.signature(M.StyledConv.forward).parameters) == ["self", "input", "style", "noise"]
    assert list(inspect.signature(M.ToRGB.forward).parameters) == ["self", "input", "style", "skip"]


def test_state_dict_layout_matches_reference_keys():
    import hairfastgan_b200.model as M
    from oracle import stylegan2_oracle as O
    for size, nkeys in [(256, 135), (1024, 171)]:
        g = M.Generator(size, 512, 8)
        p = O.synth_generator_params(size=size, seed=0)    # keys/shapes pinned against the reference (gen_golden.py)
        assert len(p) == nkeys
        g.load_state_dict(p, strict=True)
        assert g.n_latent == 2 * g.log_size - 2 and g.num_layers == 2 * (g.log_size - 2) + 1
    up, blur = M.Upsample([1, 3, 3, 1]), g.convs[0].conv.blur
    assert up.pad == (2, 1) and blur.pad == (1, 1)
    assert torch.allclose(up.kernel, O.make_kernel([1, 3, 3, 1]) * 4)


def test_cpu_inputs_fail_loudly():
    """No CPU fallback: a CPU tensor must raise, not silently compute somewhere else."""
    import hairfastgan_b200.model as M
    g = M.Generator(256, 512, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        g([torch.randn(1, 14, 512)], input_is_latent=True)
    m = M.StyledConv(64, 64, 3, 512)
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 64, 8, 8), torch.randn(1, 512))


def test_install_overlay_redirects_reference_imports():
    import sys
    import hairfastgan_b200.install as inst
    inst.install()
    try:
        import importlib
        assert importlib.import_module("models.stylegan2.op").__name__ == "hairfastgan_b200.op"
        assert importlib.import_module("models.stylegan2.model").Generator.__module__ == "hairfastgan_b200.model"
        fse = importlib.import_module("pixel2style2pixel.models.stylegan2.model")
        assert fse.Generator.__module__ == "hairfastgan_b200.fse_model" and callable(fse.get_keys)
        psp = importlib.import_module("models.encoder4editing.models.encoders.psp_encoders")
        assert psp.Encoder4Editing.__module__ == "hairfastgan_b200.encoders"
        seg = importlib.import_module("models.CtrlHair.external_code.face_parsing.model")     # my_parsing_util.py:15
        assert seg.BiSeNet.__module__ == "hairfastgan_b200.bisenet"
        bic = importlib.import_module("utils.bicubic")                                          # Embedding.py:13
        assert bic.BicubicDownSample.__module__ == "hairfastgan_b200.bicubic"
        ns = {}
        exec("from nets.feature_style_encoder import *", ns)          # trainer.py:20
        assert ns["fs_encoder_v2"].__module__ == "hairfastgan_b200.encoders"
    finally:
        inst.uninstall()
    assert "models.stylegan2.op" not in sys.modules and "nets" not in sys.modules


def test_install_rebinds_postprocess_classes(tmp_path):
    """models.Net / models.Encoders stay the reference's modules; only the PostProcess class names are rebound,
    right after import (a stand-in package with the same module layout plays the reference here)."""
    import sys
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.postprocess as P
    pkg = tmp_path / "models"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "Net.py").write_text("class FeatureEncoder: pass\nclass FeatureEncoderMult(FeatureEncoder): pass\n"
                                "class Net: pass\n")
    (pkg / "Encoders.py").write_text("from models.Net import FeatureEncoderMult\nclass FeatureiResnet: pass\n"
                                     "class PostProcessModel:\n    def build(self):\n"
                                     "        return FeatureEncoderMult, FeatureiResnet\n")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.")}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install()
        import importlib
        enc = importlib.import_module("models.Encoders")
        net = importlib.import_module("models.Net")
        assert enc.PostProcessModel().build() == (P.FeatureEncoderMult, P.FeatureiResnet)
        assert net.FeatureEncoderMult is P.FeatureEncoderMult and net.FeatureEncoder is P.FeatureEncoder
        assert net.Net.__module__ == "models.Net"                       # everything else untouched
        inst.uninstall()
        assert net.FeatureEncoderMult.__module__ == "models.Net" and enc.FeatureiResnet.__module__ == "models.Encoders"
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_install_rebinds_dilate_erosion(tmp_path):
    """utils/image_utils.py stays the reference's module (Poisson blending helpers, ...); only DilateErosion is
    rebound after import (a stand-in package plays the reference)."""
    import sys
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.masks as MK
    pkg = tmp_path / "utils"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "image_utils.py").write_text("class DilateErosion: pass\ndef poisson_image_blending(): return 'reference'\n")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "utils" or k.startswith("utils.")}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install()
        import importlib
        iu = importlib.import_module("utils.image_utils")
        assert iu.DilateErosion is MK.DilateErosion and iu.poisson_image_blending() == "reference"
        assert importlib.import_module("utils.bicubic").BicubicDownSample.__module__ == "hairfastgan_b200.bicubic"
        inst.uninstall()
        assert iu.DilateErosion.__module__ == "utils.image_utils"
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "utils" or k.startswith("utils.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_fse_reconstruction_skip_is_opt_in_and_results_identical(tmp_path):
    """SURVEY 8f-2: install(skip_fse_reconstruction=True) rebinds Trainer.test of the FeatureStyleEncoder `trainer`
    module; the fast path returns the same (w_recon, fea), None for the unused image, and asks the generator for the
    RNG draws of the skipped forward.  A stand-in trainer module plays the reference here."""
    import sys
    import hairfastgan_b200.install as inst
    (tmp_path / "trainer.py").write_text(
        "class Trainer:\n"
        "    def test(self, w=None, img=None, noise=None, zero_noise_input=True, return_latent=False, training_mode=False):\n"
        "        return ['original', return_latent]\n")
    saved = sys.modules.pop("trainer", None)
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install()                                   # default: not patched
        import importlib
        mod = importlib.import_module("trainer")
        assert not hasattr(mod.Trainer.test, "__wrapped__")
        inst.uninstall()
        inst.install(skip_fse_reconstruction=True)       # already imported: patched in place
        assert hasattr(mod.Trainer.test, "__wrapped__")

        class Gen:
            drawn = []

            def consume_noise(self, batch, device=None):
                self.drawn.append(batch)

        t = mod.Trainer()
        t.config, t.scale, t.scale_mode = {"use_fs_encoder": True}, 1, "bilinear"
        t.dlatent_avg = torch.ones(18, 512)
        t.enc = lambda x: (torch.full((x.shape[0], 18, 512), 2.0), x.mean((2, 3)))
        t.StyleGAN = Gen()
        img = torch.rand(3, 4, 16, 16)
        out = t.test(img=img, return_latent=True)
        assert out[1] is None and torch.equal(out[0], img[:, :3]) and torch.equal(out[2], torch.full((3, 18, 512), 3.0))
        assert torch.allclose(out[3], F_interp_mean(img)) and Gen.drawn == [3] and t.n_iter == 1e5
        assert t.test(img=img, return_latent=False) == ["original", False]         # every other call: the reference
        t.StyleGAN = object()                                                       # not our generator: the reference
        assert t.test(img=img, return_latent=True) == ["original", True]
        inst.uninstall()
        assert not hasattr(mod.Trainer.test, "__wrapped__")
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        sys.modules.pop("trainer", None)
        if saved is not None:
            sys.modules["trainer"] = saved


def F_interp_mean(img):
    import torch.nn.functional as F
    return F.interpolate(img, scale_factor=0.5, mode="bilinear").mean((2, 3))


def test_conv_plans_for_every_generator_layer(lib):
    """Tiling decisions for the 17 StyledConvs of the 1024^2 generator (no device needed): shared memory
    fits the 227 KB opt-in limit of sm_90, the grid never exceeds the 132 SMs of an H100, the N tile fits the
    m64 x n128 wgmma register accumulator, and every up-conv runs its four parities in one 128-column tile."""
    h = lib.lib()
    layers = [(512, 512, 4, 0), (512, 512, 4, 1), (512, 512, 8, 0), (512, 512, 8, 1), (512, 512, 16, 0),
              (512, 512, 16, 1), (512, 512, 32, 0), (512, 512, 32, 1), (512, 512, 64, 0), (512, 256, 64, 1),
              (256, 256, 128, 0), (256, 128, 128, 1), (128, 128, 256, 0), (128, 64, 256, 1), (64, 64, 512, 0),
              (64, 32, 512, 1), (32, 32, 1024, 0)]
    for batch in (1, 3, 4, 12):
        for i, (cin, cout, r, up) in enumerate(layers):
            d = lib.hf_conv_desc(cin, cout, 3, up, lib.HF_BF16)
            out = (C.c_int * 12)()
            assert h.hf_conv_plan_query(C.byref(d), batch, r, r, out) == 0, h.hf_last_error()
            halo, n_tile, n_n, G, na, pitch, res, stages, smem, work, grid, kchunk = list(out)
            assert smem <= 232448 and stages >= 2 and grid <= 132 and work >= 1
            assert (halo, G, na, pitch, res) == (0, 1, 0, 0, 0)
            assert n_tile * n_n == (4 * cout if up else cout) and n_tile in (32, 64, 128)
            assert kchunk == (32 if cin == 32 else 64)
            assert work == n_n * -(-batch * r * r // 128) if r >= 16 else work >= n_n
            if up:
                assert n_tile == 128

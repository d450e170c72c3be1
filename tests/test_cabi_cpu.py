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


no_device_only = pytest.mark.skipif(torch.cuda.is_available(),
                                    reason="hands the library fake pointers: only where no CUDA device could run them")


@no_device_only
@pytest.mark.parametrize("dt", ["HF_BF16", "HF_F16"])
def test_unaligned_16bit_tensors_rejected_without_device(lib, dt):
    """Every SIMT entry point whose kernel moves 16 bytes at a time rejects a pointer that is only 8-byte aligned
    (0x...8), before any launch, on either path (vec8 or scalar)."""
    h, d = lib.lib(), getattr(lib, dt)
    A, B_, C_, D_, U = 0x10000, 0x20000, 0x30000, 0x40000, 0x50008       # U: 8-byte aligned, not 16
    part = b"channel_partial: the 16-bit tensor must be 16-byte aligned"
    cases = [
        (h.hf_channel_mean_nhwc16, (U, A, B_, 1, 4, 8, d, None), part),
        (h.hf_se_gate_nhwc16, (U, A, B_, C_, D_, 1, 4, 8, 2, d, None), part),
        (h.hf_pooled_fc_nhwc16, (U, A, None, None, 0, B_, C_, 1, 4, 8, 3, d, None), part),
        (h.hf_instance_norm_lrelu_nhwc16, (U, A, B_, 1, 4, 8, 0.2, d, None), b"instance_norm: 16-bit tensors"),
        (h.hf_instance_norm_lrelu_nhwc16, (A, U, B_, 1, 4, 8, 0.2, d, None), b"instance_norm: 16-bit tensors"),
        (h.hf_scale_add_nhwc16, (U, None, None, 1, None, None, A, None, 1, 2, 2, 8, d, None), b"scale_add: 16-bit"),
        (h.hf_scale_add_nhwc16, (A, U, None, 1, None, None, B_, None, 1, 2, 2, 8, d, None), b"scale_add: 16-bit"),
        (h.hf_scale_add_nhwc16, (A, None, U, 2, None, None, B_, None, 1, 2, 2, 8, d, None), b"scale_add: 16-bit"),
        (h.hf_scale_add_nhwc16, (A, None, None, 1, B_, C_, None, U, 1, 2, 2, 8, d, None), b"scale_add: 16-bit"),
        (h.hf_scale_add_nhwc16, (U, None, None, 1, None, None, A, None, 1, 2, 2, 6, d, None), b"scale_add: 16-bit"),
        (h.hf_upsample_add_nhwc16, (U, A, B_, 1, 2, 2, 4, 4, 8, d, None), b"upsample_add: 16-bit"),
        (h.hf_upsample_add_nhwc16, (A, B_, U, 1, 2, 2, 4, 4, 6, d, None), b"upsample_add: 16-bit"),
        (h.hf_adaptive_avgpool_nhwc16, (U, A, 1, 4, 4, 8, 2, 2, d, None), b"adaptive_avgpool: the 16-bit tensor"),
        (h.hf_adaptive_avgpool_nhwc16, (U, A, 1, 4, 4, 6, 2, 2, d, None), b"adaptive_avgpool: the 16-bit tensor"),
        (h.hf_maxpool3x3s2_nhwc16, (U, A, 1, 4, 4, 8, d, None), b"maxpool: 16-bit tensors"),
        (h.hf_maxpool3x3s2_nhwc16, (A, U, 1, 4, 4, 8, d, None), b"maxpool: 16-bit tensors"),
        (h.hf_gate_add_up_nhwc16, (U, None, None, None, A, 1, 2, 2, 8, 2, d, None), b"gate_add_up: 16-bit"),
        (h.hf_gate_add_up_nhwc16, (A, None, None, U, B_, 1, 2, 2, 8, 1, d, None), b"gate_add_up: 16-bit"),
        (h.hf_gate_add_up_nhwc16, (A, B_, C_, None, U, 1, 2, 2, 8, 2, d, None), b"gate_add_up: 16-bit"),
    ]
    for fn, args, msg in cases:
        assert fn(*args) == -1, (fn.__name__, args)                   # HF_ERR_INVALID
        assert h.hf_last_error().startswith(msg), (fn.__name__, args, h.hf_last_error())


@no_device_only
@pytest.mark.parametrize("dt", ["HF_BF16", "HF_F16"])
def test_sean_and_shape_unaligned_operands_rejected_without_device(lib, dt):
    """The SEAN and shape adaptor entry points check every operand their kernels read or write 16 bytes at a time
    (uint4 for 16-bit tensors, float4 for fp32 rows) before any device call: an fp32 pointer that is only 4-byte
    aligned (0x...4) or a 16-bit one that is only 8-byte aligned (0x...8) is an error, not a launch."""
    h, d = lib.lib(), getattr(lib, dt)
    A, B_, C_, D_, E, U4, U8 = 0x10000, 0x20000, 0x30000, 0x40000, 0x60000, 0x50004, 0x50008

    def aces(fc_w, tw):
        arr = (lib.hf_sean_ace_tables * 2)()
        arr[0] = lib.hf_sean_ace_tables(A, B_, C_, D_, 64)
        arr[1] = lib.hf_sean_ace_tables(fc_w, B_, tw, D_, 64)
        return arr

    tables = b"hf_sean_style_tables: image_code, mean_code and mu_workspace must be 16-byte aligned"
    ace_rows = b"hf_sean_style_tables: fc_w and tw of ACE 1 must be 16-byte aligned"
    cases = [
        (h.hf_sean_conv_img, (U8, A, B_, C_, 4, 8, d, None), b"hf_sean_conv_img: x16 must be 16-byte aligned"),
        (h.hf_sean_style_tables, (U4, A, aces(A, A), 2, B_, None), tables),
        (h.hf_sean_style_tables, (A, U4, aces(A, A), 2, B_, None), tables),
        (h.hf_sean_style_tables, (A, B_, aces(A, A), 2, U4, None), tables),
        (h.hf_sean_style_tables, (A, B_, aces(U4, A), 2, C_, None), ace_rows),
        (h.hf_sean_style_tables, (A, B_, aces(A, U4), 2, C_, None), ace_rows),
        (h.hf_sean_onehot_conv, (A, U4, None, 0, B_, 8, 8, d, None), b"hf_sean_onehot_conv: unaligned pointer"),
        (h.hf_sean_onehot_conv, (A, B_, None, 0, U8, 8, 8, d, None), b"hf_sean_onehot_conv: unaligned pointer"),
        (h.hf_sean_ace_apply, (U8, A, A, A, A, A, None, None, 0, B_, 8, 64, d, None), b"hf_sean_ace_apply: unaligned"),
        (h.hf_sean_ace_apply, (A, A, A, A, A, A, None, None, 0, U8, 8, 64, d, None), b"hf_sean_ace_apply: unaligned"),
        (h.hf_sean_ace_apply, (A, A, A, A, A, A, U4, B_, 0, C_, 8, 64, d, None), b"hf_sean_ace_apply: unaligned"),
        (h.hf_shape_onehot_s2, (A, U4, B_, C_, 4, 8, d, None), b"hf_shape_onehot_s2: unaligned pointer"),
        (h.hf_shape_onehot_s2, (A, B_, U4, C_, 4, 8, d, None), b"hf_shape_onehot_s2: unaligned pointer"),
        (h.hf_shape_onehot_s2, (A, B_, C_, U8, 4, 8, d, None), b"hf_shape_onehot_s2: unaligned pointer"),
        (h.hf_shape_layer_norm_lrelu, (U8, A, A, B_, C_, 4, 8, 0.2, d, None), b"hf_shape_layer_norm_lrelu: unaligned"),
        (h.hf_shape_layer_norm_lrelu, (A, B_, B_, U8, C_, 4, 8, 0.2, d, None), b"hf_shape_layer_norm_lrelu: unaligned"),
        (h.hf_shape_logits_argmax, (U8, A, B_, C_, D_, 4, d, None), b"hf_shape_logits_argmax: unaligned input"),
        (h.hf_shape_logits_argmax, (A, U8, B_, C_, D_, 4, d, None), b"hf_shape_logits_argmax: unaligned input"),
        (h.hf_shape_gemm, (0, U8, A, None, B_, None, C_, 8, 8, 4, 4, d, None), b"hf_shape_gemm: unaligned operand"),
        (h.hf_shape_gemm, (0, A, U8, None, B_, None, C_, 8, 8, 4, 4, d, None), b"hf_shape_gemm: unaligned operand"),
    ]
    for fn, args, msg in cases:
        assert fn(*args) == -1, (fn.__name__, args)                   # HF_ERR_INVALID
        assert h.hf_last_error().startswith(msg), (fn.__name__, args, h.hf_last_error())
    for n_ace in (0, 17):                                                 # 1..16 ACE layers per call
        assert h.hf_sean_style_tables(A, B_, aces(A, A), n_ace, C_, None) == -1
        assert b"ACE layers (1..16)" in h.hf_last_error(), h.hf_last_error()


@no_device_only
def test_unaligned_style_rows_rejected_without_device(lib):
    """The style affine reads latent rows and modulation weights with float4 loads: hf_torgb_forward,
    hf_conv_forward and hf_generator_forward reject a pointer that is only 4-byte aligned (0x...4), before any
    launch."""
    h = lib.lib()
    A, B_, U = 0x10000, 0x20000, 0x50004                                # U: 4-byte aligned, not 16
    msg = b"hf_torgb_forward: style and mod_weight must be 16-byte aligned"
    for style, mw in ((U, A), (A, U)):
        assert h.hf_torgb_forward(A, style, 512, 512, A, mw, B_, B_, None, None, A, 1, 64, 4, 4, A, None) == -1
        assert h.hf_last_error() == msg, h.hf_last_error()
    d = lib.hf_conv_desc(64, 64, 3, 0, lib.HF_BF16)
    for style, mw in ((U, A), (A, U)):
        io = lib.hf_conv_io()
        io.batch, io.height, io.width, io.x, io.style, io.style_dim, io.style_stride = 1, 4, 4, A, style, 512, 512
        io.mod_weight, io.mod_bias, io.y, io.workspace = mw, B_, A, A
        assert h.hf_conv_forward(C.byref(d), A, C.byref(io), None) == -1
        assert h.hf_last_error() == b"hf_conv_forward: style and mod_weight must be 16-byte aligned", h.hf_last_error()
    cfg = lib.hf_gen_config(64, 512, 2, lib.HF_BF16)
    io = lib.hf_gen_io()
    io.batch, io.latent, io.out_rgb = 1, U, A
    assert h.hf_generator_forward(C.byref(cfg), A, C.byref(io), A, None, None) == -1
    assert h.hf_last_error() == b"hf_generator_forward: latent must be 16-byte aligned", h.hf_last_error()


@no_device_only
def test_scale_add_rejects_a_shortcut_of_the_wrong_shape():
    """MaxPool2d(1, 2) of an odd (2H-1) x (2W-1) map also has H x W pixels, but the kernel reads its stride-2
    shortcut as [B, 2H, 2W, C]: the wrapper refuses any other shape before the library sees it."""
    import hairfastgan_b200.nn16 as N
    res = torch.zeros(2, 4, 5, 8, dtype=torch.float16)
    for sc, stride in (((2, 7, 9, 8), 2), ((2, 8, 9, 8), 2), ((2, 8, 10, 8), 1), ((1, 8, 10, 8), 2),
                       ((2, 8, 10, 16), 2)):
        with pytest.raises(ValueError, match="scale_add: shortcut of shape"):
            N.scale_add(res, shortcut16=torch.zeros(sc, dtype=torch.float16), shortcut_stride=stride)


def test_every_dtype_argument_is_checked_first(lib):
    """Every call with an `int dtype` parameter rejects a value other than HF_BF16 / HF_F16 before its other
    argument checks: with every other argument zero / NULL the error names the dtype."""
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hairfast_b200.h")).read(), flags=re.S)
    dtype_pos = {}
    for name, params in re.findall(r"\b(hf_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr):
        if re.search(r"\bint\s+dtype\b", params):
            dtype_pos[name] = [re.findall(r"\w+", p)[-1] for p in params.split(",")].index("dtype")
    assert len(dtype_pos) == 21, sorted(dtype_pos)
    h = lib.lib()
    for name, pos in sorted(dtype_pos.items()):
        argtypes = lib.SYMBOLS[name][1]
        for bad in (2, -1):
            args = [None if t is C.c_void_p or issubclass(t, C._Pointer) else t(0) for t in argtypes]
            args[pos] = bad
            assert getattr(h, name)(*args) == -1, name               # HF_ERR_INVALID
            assert h.hf_last_error() == f"{name}: bad dtype {bad}".encode(), (name, h.hf_last_error())


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
            # out[4]: the 2-slot activation ring of the column-shift mainloop (16-pixel-wide tiles), 0 on the per-tap one
            assert (halo, G, na, pitch, res) == (0, 1, 2 if r >= 16 else 0, 0, 0)
            assert n_tile * n_n == (4 * cout if up else cout) and n_tile in (32, 64, 128)
            assert kchunk == (32 if cin == 32 else 64)
            assert work == n_n * -(-batch * r * r // 128) if r >= 16 else work >= n_n
            if up:
                assert n_tile == 128


@no_device_only
@pytest.mark.parametrize("dt", ["HF_BF16", "HF_F16"])
def test_modulation_arguments_checked_without_device(lib, dt):
    """hf_mod_embed16, hf_mod_gemm, hf_mod_hidden and hf_mod_chain check the descriptor, NULL pointers and the
    alignment of every pointer their kernels reach wider than its type (16-byte cp.async / uint4 operands, the 2-byte
    hidden rows) before they select a device or launch."""
    h, d16 = lib.lib(), getattr(lib, dt)
    A, B_, C_, D_, E, U8, U1 = 0x10000, 0x20000, 0x30000, 0x40000, 0x60000, 0x50008, 0x50001
    d = lib.hf_mod_desc(6, 512, 512, 1, d16)
    bad = lib.hf_mod_desc(25, 512, 512, 1, d16)
    src = (lib.hf_mod_rows * 1)(lib.hf_mod_rows(A, 6 * 512, 512))
    nul = (lib.hf_mod_rows * 1)(lib.hf_mod_rows(None, 0, 0))
    x0 = (lib.hf_mod_rows * 2)(lib.hf_mod_rows(A, 6 * 512, 512), lib.hf_mod_rows(A, 6 * 512, 512))
    x0n = (lib.hf_mod_rows * 2)(lib.hf_mod_rows(None, 0, 0), lib.hf_mod_rows(None, 0, 0))
    base = lib.hf_mod_rows(B_, 0, 512)
    r = C.byref
    cases = [
        (h.hf_mod_embed16, (r(bad), 1, src, A, None), b"hf_mod_embed16: layers 25"),
        (h.hf_mod_embed16, (r(d), 0, src, A, None), b"hf_mod_embed16: batch 0"),
        (h.hf_mod_embed16, (r(d), 1, src, U8, None), b"hf_mod_embed16: null or unaligned pointer"),
        (h.hf_mod_embed16, (r(d), 1, nul, A, None), b"hf_mod_embed16: source 0 is null"),
        (h.hf_mod_gemm, (r(d), 1, 3, A, B_, None, C_, D_, None), b"hf_mod_gemm: layer 3"),
        (h.hf_mod_gemm, (r(d), 1, 2, A, B_, None, None, D_, None), b"hf_mod_gemm: null pointer"),
        (h.hf_mod_gemm, (r(d), 1, 1, U8, B_, None, C_, D_, None), b"hf_mod_gemm: unaligned operand"),
        (h.hf_mod_gemm, (r(d), 1, 2, A, U8, None, C_, D_, None), b"hf_mod_gemm: unaligned operand"),
        (h.hf_mod_hidden, (r(bad), 1, A, B_, C_, C_, C_, D_, E, None), b"hf_mod_hidden: layers 25"),
        (h.hf_mod_hidden, (r(d), 1, A, B_, None, C_, C_, D_, E, None), b"hf_mod_hidden: null pointer"),
        (h.hf_mod_hidden, (r(d), 1, U8, B_, C_, C_, C_, D_, E, None), b"hf_mod_hidden: unaligned operand"),
        (h.hf_mod_hidden, (r(d), 1, A, U8, C_, C_, C_, D_, E, None), b"hf_mod_hidden: unaligned operand"),
        (h.hf_mod_hidden, (r(d), 1, A, B_, C_, C_, C_, U1, E, None), b"hf_mod_hidden: h16 must be 2-byte aligned"),
        (h.hf_mod_chain, (r(bad), 1, A, B_, C_, x0, r(base), D_, E, None), b"hf_mod_chain: layers 25"),
        (h.hf_mod_chain, (r(d), 1, A, B_, C_, x0, r(base), None, E, None), b"hf_mod_chain: null pointer"),
        (h.hf_mod_chain, (r(d), 1, U8, B_, C_, x0, r(base), D_, E, None), b"hf_mod_chain: unaligned weights"),
        (h.hf_mod_chain, (r(d), 1, A, B_, C_, x0n, r(base), D_, E, None), b"hf_mod_chain: x0[0] is null"),
    ]
    for fn, args, msg in cases:
        assert fn(*args) == -1, (fn.__name__, args)                   # HF_ERR_INVALID
        assert h.hf_last_error().startswith(msg), (fn.__name__, args, h.hf_last_error())


@no_device_only
def test_stylegan2_op_and_glue_arguments_checked_without_device(lib):
    """hf_upfirdn2d_f32, hf_bias_act_f32, hf_bicubic_downsample_f32, hf_dilate_erode_f32, hf_align_masks_f32 and
    hf_fspace_blend_f32 check their arguments before they select a device; empty inputs are no-ops."""
    h = lib.lib()
    A, B_, C_ = 0x10000, 0x20000, 0x30000
    two = lambda *v: (C.c_void_p * 2)(*v)
    f2 = (C.c_float * 2)(1.0, -1.0)
    cases = [
        (h.hf_upfirdn2d_f32, (A, B_, None, 1, 4, 4, 4, 4, 1, 1, 1, 1, 0, 0, 0, 0, None), b"upfirdn2d: null pointer"),
        (h.hf_upfirdn2d_f32, (A, B_, C_, 1, 0, 4, 4, 4, 1, 1, 1, 1, 0, 0, 0, 0, None), b"upfirdn2d: bad shape"),
        (h.hf_upfirdn2d_f32, (A, B_, C_, 1, 4, 4, 4, 4, 1, 0, 1, 1, 0, 0, 0, 0, None), b"upfirdn2d: up/down must be"),
        (h.hf_upfirdn2d_f32, (A, B_, C_, 1, 2, 2, 4, 4, 1, 1, 1, 1, 0, 0, 0, 0, None), b"upfirdn2d: output would be"),
        (h.hf_bias_act_f32, (None, None, B_, 8, 0, 4, 3, 0.2, 1.0, None), b"bias_act: null pointer"),
        (h.hf_bias_act_f32, (A, None, B_, 8, 0, 4, 2, 0.2, 1.0, None), b"bias_act: act must be 1"),
        (h.hf_bias_act_f32, (A, None, B_, 8, 0, 0, 3, 0.2, 1.0, None), b"bias_act: bad sizes"),
        (h.hf_bias_act_f32, (A, None, B_, 8, 2, 4, 3, 0.2, 1.0, None), b"bias_act: bias pointer is null"),
        (h.hf_bicubic_downsample_f32, (A, None, B_, 1, 64, 64, 4, 0, None), b"bicubic_down: null pointer"),
        (h.hf_bicubic_downsample_f32, (A, B_, C_, 1, 64, 64, 9, 0, None), b"bicubic_down: factor 9 unsupported"),
        (h.hf_bicubic_downsample_f32, (A, B_, C_, 0, 64, 64, 4, 0, None), b"bicubic_down: bad shape"),
        (h.hf_bicubic_downsample_f32, (A, B_, C_, 1, 6, 64, 4, 0, None), b"bicubic_down: image smaller than"),
        (h.hf_dilate_erode_f32, (A, None, C_, None, 1, 4, 4, 1, None), b"dilate_erode: null pointer"),
        (h.hf_dilate_erode_f32, (A, B_, C_, None, 1, 4, 4, -1, None), b"dilate_erode: bad arguments"),
        (h.hf_dilate_erode_f32, (A, B_, C_, None, 1, 4, 4, 2, None), b"dilate_erode: workspace"),
        (h.hf_dilate_erode_f32, (A, B_, C_, None, 50000, 200, 200, 1, None), b"dilate_erode: tensor too large"),
        (h.hf_align_masks_f32, (A, B_, None, C_, 16, None), b"align_masks: bad arguments"),
        (h.hf_align_masks_f32, (A, B_, C_, A, 0, None), b"align_masks: bad arguments"),
        (h.hf_fspace_blend_f32, (A, two(B_, B_), two(C_, C_), None, f2, A, 2, 4, 8, 8, 8, 8, None),
         b"fspace_blend: null pointer"),
        (h.hf_fspace_blend_f32, (A, two(B_, B_), two(C_, C_), f2, None, A, 2, 4, 8, 8, 8, 8, None),
         b"fspace_blend: null pointer"),
        (h.hf_fspace_blend_f32, (A, two(B_, B_), two(C_, C_), f2, f2, A, 5, 4, 8, 8, 8, 8, None),
         b"fspace_blend: 1..4 stages"),
        (h.hf_fspace_blend_f32, (A, two(B_, B_), two(C_, C_), f2, f2, A, 2, 4, 0, 8, 8, 8, None),
         b"fspace_blend: bad shape"),
        (h.hf_fspace_blend_f32, (A, two(B_, None), two(C_, C_), f2, f2, A, 2, 4, 8, 8, 8, 8, None),
         b"fspace_blend: null stage pointer"),
    ]
    for fn, args, msg in cases:
        assert fn(*args) == -1, (fn.__name__, args)                   # HF_ERR_INVALID
        assert h.hf_last_error().startswith(msg), (fn.__name__, args, h.hf_last_error())
    assert h.hf_bias_act_f32(None, None, None, 0, 0, 1, 3, 0.2, 1.0, None) == 0          # empty input

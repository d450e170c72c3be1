"""CtrlHair's shape adaptor without a GPU: the oracle against the golden of the unmodified reference, the algebra of
the kernels' forms in float64 (layer-0 lookup, stride-2 4x4 and nearest-up 3x3 gathers, LayerNorm, logits order), the
plans of the wgmma-routed decoder layers and of the split-K GEMM, and the install bindings."""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from baseline import refenv
from oracle import shape_adaptor_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "shape_adaptor.npz")
needs_ref = pytest.mark.skipif(not refenv.available(), reason="reference not built (oracle/build_ref.py)")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def params(golden):
    return O.synth_params(int(golden["seed"]))


@pytest.fixture(scope="module")
def lib():
    from hairfastgan_b200 import _lib
    _lib.lib()
    return _lib


def test_golden_is_small_and_complete(golden):
    assert os.path.getsize(GOLDEN) < 1 << 20
    names = [str(n) for n in golden["names"]]
    assert names == list(O.label_cases())
    cases = O.label_cases()
    for n in names:
        assert np.array_equal(golden[f"{n}_mask"].astype(np.int64), cases[n].numpy())
    assert (golden["no_hair_mask"] != O.HAIR_IDX).all() and (golden["hair_only_mask"] != O.HAIR_IDX).any()
    assert (golden["some_255_mask"] == 255).any()


_REF_CHECK = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
from baseline import refenv
refenv.activate(overlay=False, chdir=False)
from models.CtrlHair.shape_branch import solver
from oracle import shape_adaptor_oracle as O
g = np.load(sys.argv[2])
gen = O.reference_generator()
assert [(k, tuple(v.shape)) for k, v in gen.state_dict().items()] == list(O.config054_shapes().items())
gen.load_state_dict(O.synth_params(int(g["seed"])))
torch.set_grad_enabled(False)
mask = torch.from_numpy(g["some_255_mask"].astype(np.int64))
torch.manual_seed(3)
face, hair = solver.get_hair_face_code(gen, mask)
assert int((mask == 255).sum()) == 0 and int((mask == 19).sum()) > 0
assert np.allclose(face.numpy(), g["some_255_face_code"], rtol=1e-4, atol=1e-5)
assert np.allclose(hair.numpy(), g["some_255_hair_code"], rtol=1e-4, atol=1e-5)
print("ok")
"""


@needs_ref
def test_reference_reproduces_golden_and_rewrites_mask(golden):
    p = subprocess.run([sys.executable, "-c", _REF_CHECK, ROOT, GOLDEN], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and p.stdout.strip().endswith("ok"), p.stderr[-3000:]


# ------------------------------------------------------------------------------------------------ forms, float64
@pytest.mark.parametrize("hair", [True, False])
def test_layer0_lookup_equals_conv(golden, params, hair):
    """Positional constant + one-hot gather == ZeroPad 1 + Conv 4x4 s2 over cat[one-hot, positional channels]."""
    from hairfastgan_b200 import shape_adaptor as S
    pre = "hair_encoder" if hair else "face_encoder"
    w0, b0 = params[f"{pre}.layers.0.conv.weight"], params[f"{pre}.layers.0.conv.bias"]
    n_mask = 1 if hair else 18
    table = S.onehot_table(w0, hair)
    cmap = S.positional_map(w0, b0, O.pos_embedding(), n_mask)
    for name in ("some_255", "odd_hair"):
        mask = torch.from_numpy(golden[f"{name}_mask"].astype(np.int64))
        x = torch.cat([O.one_hot_input(mask, hair), O.pos_embedding()[None].double()], 1)
        ref = F.conv2d(F.pad(x, (1, 1, 1, 1)), w0.double(), b0.double(), stride=2)[0].permute(1, 2, 0)
        got = O.layer0_lookup(mask, table, cmap)
        assert float((got - ref).abs().max()) < 2e-6 * float(ref.abs().max())     # cmap is stored in fp32


def test_stride2_gather_equals_conv():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 24, 16, 16, generator=g, dtype=torch.float64)
    w = torch.randn(40, 24, 4, 4, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.pad(x, (1, 1, 1, 1)), w, stride=2)[0].permute(1, 2, 0).reshape(-1, 40)
    got = O.gather_gemm(1, x[0].permute(1, 2, 0), w.permute(0, 2, 3, 1))
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)


def test_nearest_up_gather_equals_conv():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 16, 5, 7, generator=g, dtype=torch.float64)
    w = torch.randn(24, 16, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, padding=1)[0].permute(1, 2, 0).reshape(-1, 24)
    got = O.gather_gemm(2, x[0].permute(1, 2, 0), w.permute(0, 2, 3, 1))
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)


@needs_ref
def test_layer_norm_matches_reference_class():
    code = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from baseline import refenv
refenv.activate(overlay=False, chdir=False)
from models.CtrlHair.my_torchlib.module import LayerNorm
from oracle import shape_adaptor_oracle as O
ln = LayerNorm(24).double()
g = torch.Generator().manual_seed(3)
with torch.no_grad():
    ln.gamma.copy_(torch.rand(24, generator=g, dtype=torch.float64)); ln.beta.copy_(torch.randn(24, generator=g, dtype=torch.float64))
x = torch.randn(1, 24, 6, 5, generator=g, dtype=torch.float64) * 3 + 1
ref = torch.nn.functional.leaky_relu(ln(x), 0.2)[0].permute(1, 2, 0)
got = O.layer_norm_lrelu(x[0].permute(1, 2, 0), ln.gamma.detach(), ln.beta.detach())
assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)
print("ok")
"""
    p = subprocess.run([sys.executable, "-c", code, ROOT], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and p.stdout.strip().endswith("ok"), p.stderr[-3000:]


# ------------------------------------------------------------------------------------------------ plans
def test_wgmma_decoder_layers_plan(lib):
    """Decoder layers 3-6 (nearest 2x up, then a plain 3x3 conv) at B = 1 are accepted by the wgmma convolution."""
    from hairfastgan_b200 import shape_adaptor as S
    out = (C.c_int * 12)()
    for i in range(S.DEC_GEMM_LAYERS, len(S.DEC_CH)):
        cin, cout, r = S.DEC_CH[i - 1], S.DEC_CH[i], 4 << i
        d = lib.hf_conv2d_desc(cin, cout, cin, 3, 1, 1, lib.HF_F16, 0, 0)
        assert lib.lib().hf_conv2d_plan_query(C.byref(d), 1, r, r, out) == 0, (i, lib.lib().hf_last_error())


def test_gemm_plans_and_checks(lib):
    out = (C.c_int * 5)()
    L = lib.lib()
    assert L.hf_shape_gemm_plan(1, 1024, 2048, 4, 4, 132, out) == 0
    assert list(out) == [8, 17, 256, 16, 1]                  # enc layer 6: every SM streams weights
    assert L.hf_shape_gemm_plan(0, 8192, 1024, 1, 1, 132, out) == 0 and out[1] * out[3] >= 132
    assert L.hf_shape_gemm_plan(2, 1024, 512, 8, 8, 132, out) == 0 and out[0] == 64 and out[4] == 4
    for args in [(3, 64, 64, 4, 4), (1, 12, 64, 4, 4), (1, 64, 64, 5, 4), (0, 64, 0, 1, 1)]:
        assert L.hf_shape_gemm_plan(*args, 132, out) != 0, args


def test_shapes_table_rejects_other_configs(params):
    from hairfastgan_b200 import shape_adaptor as S
    m = O.stand_in_generator({k: v for k, v in params.items() if k.startswith("face_encoder.")
                              and not k.startswith("face_encoder.out_layer")}, torch.device("cpu"))
    with pytest.raises(NotImplementedError, match="config 054"):
        S.pack_encoder(m.face_encoder, False)


def test_cpu_tensors_raise(params):
    from hairfastgan_b200 import shape_adaptor as S
    with pytest.raises(RuntimeError, match="CUDA"):
        S.get_hair_face_code(None, torch.zeros(256, 256, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.get_new_shape(None, torch.zeros(1, 1024), torch.zeros(1, 16))


# ------------------------------------------------------------------------------------------------ overlay binding
def _fake_reference(tmp_path):
    pkg = tmp_path / "models"
    (pkg / "CtrlHair" / "shape_branch").mkdir(parents=True)
    (pkg / "sean_codes" / "models").mkdir(parents=True)
    for d in (pkg, pkg / "CtrlHair", pkg / "CtrlHair" / "shape_branch", pkg / "sean_codes", pkg / "sean_codes" / "models"):
        (d / "__init__.py").write_text("")
    (pkg / "CtrlHair" / "shape_branch" / "solver.py").write_text(
        "def get_hair_face_code(mask_generator, mask): return 'reference'\n"
        "def get_new_shape(mask_generator, face_code, new_hair_code): return 'reference'\n")
    (pkg / "sean_codes" / "models" / "pix2pix_model.py").write_text(
        "def decode_sean(sean_model, image_code, target_mask): return 'reference'\n"
        "def encode_sean(sean_model, images, labels): return 'reference'\n")
    (pkg / "Alignment.py").write_text(
        "from models.CtrlHair.shape_branch.solver import get_hair_face_code, get_new_shape\n"
        "from models.sean_codes.models.pix2pix_model import encode_sean, decode_sean\n")


@pytest.mark.parametrize("flags", [{}, {"shape_adaptor": True}, {"shape_adaptor": True, "sean": True}])
@pytest.mark.parametrize("order", ["solver_first", "alignment_first"])
def test_install_binds_the_shape_adaptor(tmp_path, flags, order):
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.sean as SE
    import hairfastgan_b200.shape_adaptor as S
    _fake_reference(tmp_path)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.")}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install(**flags)
        names = ["models.CtrlHair.shape_branch.solver", "models.Alignment"]
        for n in (names if order == "solver_first" else names[::-1]):
            importlib.import_module(n)
        solver, align = sys.modules[names[0]], sys.modules[names[1]]
        on = flags.get("shape_adaptor", False)
        for fn in ("get_hair_face_code", "get_new_shape"):
            for m in (solver, align):
                assert (getattr(m, fn) is getattr(S, fn)) == on, (m.__name__, fn)
        assert (align.decode_sean is SE.decode_sean) == flags.get("sean", False)
        assert align.encode_sean is not SE.encode_sean
        inst.uninstall()
        for m in (solver, align):
            assert m.get_hair_face_code(None, None) == "reference" and m.get_new_shape(None, None, None) == "reference"
        assert align.decode_sean(None, None, None) == "reference"
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)

"""Check against the reference built by oracle/build_ref.py (skipped where it was not built): with
``hairfastgan_b200.install.install()`` active, the UNMODIFIED reference modules that swap() imports resolve the hot-path
classes to this package.  Third-party packages the image lacks (dlib, clip, lpips, ...) are replaced by inert stubs;
nothing is constructed or run -- this is about import-time name resolution only.  Runs in a fresh interpreter."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from baseline import refenv  # noqa: E402

REF = refenv.REF_ROOT

PROBE = textwrap.dedent("""
    import importlib, sys, types
    sys.path.insert(0, %(root)r)
    import hairfastgan_b200.install as hfi
    hfi.install(skip_fse_reconstruction=True)
    sys.path.insert(0, %(ref)r)

    class Stub(types.ModuleType):
        __path__ = []
        def __getattr__(self, name):
            if name.startswith("__"):
                raise AttributeError(name)
            m = Stub(self.__name__ + "." + name); setattr(self, name, m); return m
        def __call__(self, *a, **k):
            return self
        def __iter__(self):
            return iter(())

    for name in ["gdown", "clip", "dlib", "face_alignment", "lpips", "addict", "matplotlib", "matplotlib.pyplot",
                 "cv2", "skimage", "skimage.io", "ranger", "tensorboard_logger", "yaml"]:
        try:
            importlib.import_module(name)
        except Exception:
            sys.modules[name] = Stub(name)

    import models.Net as net, models.Encoders as enc, models.Embedding as emb, models.Blending as blend
    import models.encoder4editing.models.psp as psp
    import models.FeatureStyleEncoder.FSencoder  # noqa: F401  (puts its directory on sys.path, imports `trainer`)
    import models.CtrlHair.external_code.face_parsing.my_parsing_util as parsing
    trainer = sys.modules["trainer"]
    got = {
        "Net.Generator": net.Generator.__module__,
        "Net.FeatureEncoderMult": net.FeatureEncoderMult.__module__,
        "Encoders.FeatureEncoderMult": enc.FeatureEncoderMult.__module__,
        "Encoders.FeatureiResnet": enc.FeatureiResnet.__module__,
        "Encoders.PixelNorm": enc.PixelNorm.__module__,
        "Embedding.BicubicDownSample": emb.BicubicDownSample.__module__,
        "Blending.BicubicDownSample": blend.BicubicDownSample.__module__,
        "Blending.DilateErosion": blend.DilateErosion.__module__,
        "psp.Encoder4Editing": psp.psp_encoders.Encoder4Editing.__module__,
        "trainer.Generator": trainer.Generator.__module__,
        "trainer.fs_encoder_v2": trainer.fs_encoder_v2.__module__,
        "trainer.Trainer.test": "patched" if hasattr(trainer.Trainer.test, "__wrapped__") else "reference",
        "parsing.BiSeNet": parsing.BiSeNet.__module__,
        "parsing.parsing_img": "patched" if hasattr(parsing.FaceParsing_tensor.parsing_img, "__wrapped__") else "reference",
        "Net.Net": net.Net.__module__,
    }
    for k, v in got.items():
        print(k, v)
""")

EXPECTED = {
    "Net.Generator": "hairfastgan_b200.model",
    "Net.FeatureEncoderMult": "hairfastgan_b200.postprocess",
    "Encoders.FeatureEncoderMult": "hairfastgan_b200.postprocess",
    "Encoders.FeatureiResnet": "hairfastgan_b200.postprocess",
    "Encoders.PixelNorm": "hairfastgan_b200.model",
    "Embedding.BicubicDownSample": "hairfastgan_b200.bicubic",
    "Blending.BicubicDownSample": "hairfastgan_b200.bicubic",
    "Blending.DilateErosion": "hairfastgan_b200.masks",
    "psp.Encoder4Editing": "hairfastgan_b200.encoders",
    "trainer.Generator": "hairfastgan_b200.fse_model",
    "trainer.fs_encoder_v2": "hairfastgan_b200.encoders",
    "trainer.Trainer.test": "patched",
    "parsing.BiSeNet": "hairfastgan_b200.bisenet",
    "parsing.parsing_img": "patched",
    "Net.Net": "models.Net",                      # the orchestration class stays the reference's
}


@pytest.mark.skipif(not refenv.available(), reason="reference not built (oracle/build_ref.py)")
def test_reference_imports_resolve_to_this_package(tmp_path):
    p = subprocess.run([sys.executable, "-c", PROBE % {"root": ROOT, "ref": REF}], capture_output=True, text=True,
                       timeout=600, cwd=str(tmp_path))
    assert p.returncode == 0, p.stderr[-3000:]
    got = dict(line.split(" ", 1) for line in p.stdout.strip().splitlines() if " " in line)
    assert got == EXPECTED, {k: (got.get(k), v) for k, v in EXPECTED.items() if got.get(k) != v}

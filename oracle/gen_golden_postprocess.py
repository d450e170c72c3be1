"""Golden vectors for the PostProcess conv stack (SURVEY 8f-1): run the UNMODIFIED reference classes
``FeatureEncoderMult(fs_layers=[9])`` (models/Net.py:396-477) and ``FeatureiResnet([[1024,2],[768,2],[512,2]])``
(models/Encoders.py:35-57) on CPU with seeded synthetic parameters and store small outputs in
tests/golden/postprocess.npz.  Build-container only; test infrastructure (see oracle/README.md).

models/Net.py and models/Encoders.py import packages this image lacks (gdown, clip); empty stub modules stand in for
them -- nothing of theirs is executed by the two classes."""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
REF = os.environ["HAIRFAST_REFERENCE"]          # path of an unmodified reference checkout


def main():
    torch.set_grad_enabled(False)
    import torch.utils.cpp_extension as ce
    ce.load = lambda *a, **k: None                      # the stylegan2 op JIT build is not needed here
    for name in ("gdown", "clip"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, REF)
    from oracle import encoders_oracle as EO
    import models.Net as RN
    import models.Encoders as RE
    out = {}

    # ---- FeatureEncoderMult(fs_layers=[9], opts) as PostProcessModel builds it (models/Encoders.py:109-110)
    tmp = "/tmp/_arcface_synth_pp.pth"
    torch.save(RN.iresnet50().state_dict(), tmp)
    enc = RN.FeatureEncoderMult(fs_layers=[9], opts=types.SimpleNamespace(arcface_model_path=tmp)).eval()
    params = EO.synth_params_like(enc, seed=31)
    enc.load_state_dict(params, strict=True)
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(32)) * 2 - 1
    lat, (content,) = enc(x)
    lo, (co,) = EO.feature_encoder_mult_ref(params, x)
    print("FeatureEncoderMult: ref vs oracle max abs", float((lat - lo).abs().max()), float((content - co).abs().max()),
          "rms", float(lat.pow(2).mean().sqrt()), float(content.pow(2).mean().sqrt()), "content", tuple(content.shape))
    out["mult_latent"] = lat.numpy()
    out["mult_content_sub"] = content[:, ::16, ::2, ::2].numpy()
    out["mult_n_keys"] = np.int64(len(params))
    # the 1024^2 -> 256^2 resize in front (transform_to_256, models/Net.py:12-14,447) with THIS torchvision
    xb = torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(33)) * 2 - 1
    r_ref = RN.transform_to_256(xb)
    r_or = EO.transform_to_256_ref(xb)
    # informational: torchvision >= 0.17 antialiases tensors by default, the reference's pinned 0.14 does not
    print("transform_to_256 (torchvision", __import__("torchvision").__version__, ") vs oracle (antialias off):",
          float((r_ref - r_or).abs().max()))

    # ---- FeatureiResnet([[1024, 2], [768, 2], [512, 2]]) (models/Encoders.py:113); fully convolutional, so the
    # pin uses a 16x16 map (the swap() call is 64x64)
    fr = RE.FeatureiResnet([[1024, 2], [768, 2], [512, 2]]).eval()
    fparams = EO.synth_params_like(fr, seed=41)
    fr.load_state_dict(fparams, strict=True)
    xf = torch.randn(2, 1024, 16, 16, generator=torch.Generator().manual_seed(42))
    y = fr(xf)
    yo = EO.feature_iresnet_ref(fparams, xf)
    print("FeatureiResnet: ref vs oracle max abs", float((y - yo).abs().max()), "rms", float(y.pow(2).mean().sqrt()))
    out["fres_out_sub"] = y[:, ::4].numpy()
    out["fres_n_keys"] = np.int64(len(fparams))
    np.savez_compressed(os.path.join(GOLD, "postprocess.npz"), **out)
    print("postprocess.npz", {k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()

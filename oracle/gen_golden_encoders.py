"""Golden vectors for the encoder rows (a13 / a14): run the UNMODIFIED reference classes
(Encoder4Editing, fs_encoder_v2) on CPU with seeded synthetic parameters and store small outputs in
tests/golden/encoders.npz.  Build-container only; test infrastructure (see oracle/README.md)."""
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
    ce.load = lambda *a, **k: None
    sys.path.insert(0, REF)
    from oracle import encoders_oracle as EO
    out = {}

    # ---- e4e: Encoder4Editing(50, 'ir_se', opts) as built by pSp (models/psp.py:24, opts from the ckpt)
    from models.encoder4editing.models.encoders.psp_encoders import Encoder4Editing
    ref = Encoder4Editing(50, "ir_se", types.SimpleNamespace(stylegan_size=1024)).eval()
    params = EO.synth_params_like(ref, seed=11)
    ref.load_state_dict(params, strict=True)
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(12)) * 2 - 1
    w = ref(x)
    out["e4e_w"] = w.numpy()
    out["e4e_n_keys"] = np.int64(len(params))
    # independent check of the oracle while the reference is at hand
    wo, taps = EO.e4e_ref(params, x, return_taps=True)
    print("e4e: ref vs oracle max abs", float((w - wo).abs().max()), "w rms", float(w.pow(2).mean().sqrt()))
    out["e4e_c3_sub"] = taps[23][:, ::32, ::2, ::2].numpy()

    # ---- FSE: fs_encoder_v2(n_styles=18, opts, stride=(2,2)) as built by Trainer (trainer.py:168-170)
    sys.path.insert(0, os.path.join(REF, "models", "FeatureStyleEncoder"))
    from arcface.iresnet import iresnet50
    from nets.feature_style_encoder import fs_encoder_v2
    tmp = "/tmp/_arcface_synth.pth"
    torch.save(iresnet50().state_dict(), tmp)
    fref = fs_encoder_v2(n_styles=18, opts=types.SimpleNamespace(arcface_model_path=tmp), stride=(2, 2)).eval()
    fparams = EO.synth_params_like(fref, seed=21)
    fref.load_state_dict(fparams, strict=True)
    xf = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(22)) * 2 - 1
    lat, content = fref(xf)
    out["fse_latent"] = lat.numpy()
    out["fse_content_sub"] = content[:, ::16].numpy()
    out["fse_n_keys"] = np.int64(len(fparams))
    lo, co = EO.fse_ref(fparams, xf, content_stride=2)
    print("fse: ref vs oracle max abs", float((lat - lo).abs().max()), float((content - co).abs().max()),
          "rms", float(lat.pow(2).mean().sqrt()), float(content.pow(2).mean().sqrt()))
    np.savez_compressed(os.path.join(GOLD, "encoders.npz"), **out)
    print("encoders.npz", {k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()

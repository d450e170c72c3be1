"""Golden vectors for BiSeNet (SURVEY 8f-3): run the UNMODIFIED reference class
``models/CtrlHair/external_code/face_parsing/model.py::BiSeNet`` (the one FaceParsing builds, my_parsing_util.py:42,77)
on CPU with seeded synthetic parameters and store small outputs in tests/golden/bisenet.npz.  Build-container only;
test infrastructure (see oracle/README.md).

``Resnet18.__init__`` downloads torchvision's ResNet-18 weights (face_parsing/resnet.py:71-77); there is no network
here, so ``model_zoo.load_url`` is stubbed with a randomly initialised torchvision resnet18 state_dict -- every value
is overwritten by the seeded parameters right after."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
REF = os.environ["HAIRFAST_REFERENCE"]          # path of an unmodified reference checkout


def main():
    torch.set_grad_enabled(False)
    import torch.utils.model_zoo as modelzoo
    import torchvision
    modelzoo.load_url = lambda *a, **k: torchvision.models.resnet18().state_dict()
    sys.path.insert(0, os.path.join(REF, "models", "CtrlHair", "external_code"))
    from face_parsing.model import BiSeNet                 # the package only needs torch / torchvision
    from oracle import bisenet_oracle as BO
    from oracle import encoders_oracle as EO
    out = {}
    net = BiSeNet(n_classes=19).eval()
    params = EO.synth_params_like(net, seed=51)
    net.load_state_dict(params, strict=True)
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(52)) * 2 - 1
    ref = net(x)
    mine = BO.bisenet_ref(params, x)
    for name, a, b in zip(("out", "out16", "out32"), ref, mine):
        print(f"bisenet {name}: ref vs oracle max abs", float((a - b).abs().max()), "rms", float(a.pow(2).mean().sqrt()),
              tuple(a.shape))
    low = BO.bisenet_ref(params, x, return_lowres=True)
    out["out_sub"] = ref[0][:, :, ::4, ::4].numpy()                  # [2,19,64,64]
    out["out16_sub"] = ref[1][:, :, ::8, ::8].numpy()
    out["out32_sub"] = ref[2][:, :, ::8, ::8].numpy()
    out["low_out"] = low[0].numpy()                                  # [2,19,32,32] before the bilinear upsample
    out["n_keys"] = np.int64(len(params))
    np.savez_compressed(os.path.join(GOLD, "bisenet.npz"), **out)
    print("bisenet.npz", {k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()

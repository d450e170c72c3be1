"""Golden vectors for SEAN's encode_sean: run the UNMODIFIED reference ``Pix2PixModel(SEAN_OPT)`` + ``encode_sean``
(models/sean_codes/models/pix2pix_model.py:299-306, the Zencoder of architecture.py:154-207) on CPU with the seeded
parameters of ``sean_oracle.synth_sean_params`` and store the codes and subsampled activations in
tests/golden/sean_encode.npz.  Build-container only; test infrastructure (see oracle/README.md).

The model is built the way oracle/gen_golden_sean.py builds it (``gpu_ids=[]``, a temporary checkpoint directory
holding the synthetic state_dict).  The images are regenerated from the stored seeds (``sean_encode_oracle.golden_images``); the file
stores the labels, the full codes, and subsampled outputs of the four InstanceNorm + LeakyReLU layers and of the
pre-tanh convolution -- no weights.

Label cases: case 0 (B = 2) has all 19 classes in sample 0 and five classes absent in sample 1; case 1 (B = 1) has
class 5 only at odd rows and columns of the 256^2 map, so its area at 128^2 is 0 and its code row must be zero."""
from __future__ import annotations

import copy
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
REF = os.environ["HAIRFAST_REFERENCE"]          # path of an unmodified reference checkout
SEED = 5
ODD_ONLY_CLASS = 5
TAPS = {"in1": 3, "in2": 6, "in3": 9, "in4": 12, "pre_tanh": 14}     # Zencoder.model index of each stored output


def label_cases():
    g = torch.Generator().manual_seed(23)
    full = torch.randint(0, 19, (1, 1, 16, 16), generator=g)
    full.view(-1)[:19] = torch.arange(19)
    full = full.repeat_interleave(16, 2).repeat_interleave(16, 3)
    stripes = torch.randint(0, 19, (1, 1, 64, 1), generator=g).repeat_interleave(4, 2).expand(1, 1, 256, 12)
    full[..., 100:112] = stripes                 # regions that meet inside the 2x2 cells of the 128^2 map
    part = full.clone()
    for j in (3, 7, 11, 15, 16):
        part[part == j] = 1
    odd = full.clone()
    odd[odd == ODD_ONLY_CLASS] = 0
    odd[0, 0, 33:97:2, 41:121:2] = ODD_ONLY_CLASS  # odd rows and columns only: nearest to 128^2 never picks them
    return [torch.cat([full, part]).long(), odd.long()]


def main():
    torch.set_grad_enabled(False)
    os.chdir(REF)
    sys.path.insert(0, REF)
    from oracle import sean_encode_oracle as EO
    from oracle import sean_oracle as SO
    import models.sean_codes.models.pix2pix_model as P

    params = SO.synth_sean_params(SEED)
    tmp = tempfile.mkdtemp()
    opt = copy.copy(P.SEAN_OPT)
    opt.gpu_ids, opt.checkpoints_dir = [], tmp
    os.makedirs(os.path.join(tmp, opt.name))
    torch.save(params, os.path.join(tmp, opt.name, "latest_net_G.pth"))
    torch.Tensor.cuda = lambda self, *a, **k: self
    model = P.Pix2PixModel(opt)           # util.load_network: strict load of the synthetic state_dict
    model.eval()
    zenc = model.netG.Zencoder
    out = {"n_keys": np.int64(len(params)), "seed": np.int64(SEED), "odd_only_class": np.int64(ODD_ONLY_CLASS)}
    for case, labels in enumerate(label_cases()):
        image_seed = 60 + case
        images = EO.golden_images(image_seed, labels.shape[0])
        taps = {}
        hooks = [zenc.model[i].register_forward_hook(lambda m, inp, o, name=name: taps.__setitem__(name, o.clone()))
                 for name, i in TAPS.items()]
        codes = P.encode_sean(model, images, labels.float())
        for h in hooks:
            h.remove()
        ours, otaps = EO.encode_ref(params, images, labels)
        print(f"case {case}: codes max abs {float(codes.abs().max()):.3g}, oracle max abs diff "
              f"{float((codes - ours).abs().max()):.3g}; " +
              ", ".join(f"{k} {float((taps[k] - otaps[k]).abs().max()):.3g}" for k in TAPS))
        out[f"c{case}_image_seed"] = np.int64(image_seed)
        out[f"c{case}_labels"] = labels.numpy().astype(np.int8)
        out[f"c{case}_codes"] = codes.numpy()
        for name, t in taps.items():
            out[f"c{case}_{name}"] = EO.golden_sample_enc(t).numpy()
    np.savez_compressed(os.path.join(GOLD, "sean_encode.npz"), **out)
    print("wrote", os.path.join(GOLD, "sean_encode.npz"))


if __name__ == "__main__":
    main()

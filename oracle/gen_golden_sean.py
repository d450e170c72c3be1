"""Golden vectors for SEAN's decode_sean: run the UNMODIFIED reference ``Pix2PixModel(SEAN_OPT)`` +
``decode_sean`` (models/sean_codes/models/pix2pix_model.py:309-325) on CPU with the seeded parameters of
``sean_oracle.synth_sean_params`` and store subsampled outputs in tests/golden/sean.npz.  Build-container only; test
infrastructure (see oracle/README.md).

Inside this script only: the model is built with ``gpu_ids=[]`` (CPU) from a temporary checkpoint directory holding
the synthetic state_dict; ``Tensor.cuda`` is the identity (load_average_feature, pix2pix_model.py:289); the ACE noise
``torch.randn(..., device='cuda')`` (normalization.py:111) is drawn on the CPU from a generator seeded per case.
The golden stores the noise seeds (with the first values of each draw), the mean style codes the reference loads, the
inputs and subsampled outputs -- no weights."""
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


def label_maps():
    """Two 256^2 label maps: blocky regions with all 19 classes, and one where classes 3, 7, 11, 15, 16 are absent."""
    g = torch.Generator().manual_seed(21)
    full = torch.randint(0, 19, (1, 1, 16, 16), generator=g)
    full.view(-1)[:19] = torch.arange(19)
    full = full.repeat_interleave(16, 2).repeat_interleave(16, 3)
    # finer structure: some 4-pixel-wide stripes so that regions also meet inside the 8^2 / 16^2 cells
    stripes = torch.randint(0, 19, (1, 1, 64, 1), generator=g).repeat_interleave(4, 2).expand(1, 1, 256, 12)
    full[..., 100:112] = stripes
    part = full.clone()
    for j in (3, 7, 11, 15, 16):
        part[part == j] = 1
    return [full.long(), part.long()]


def main():
    torch.set_grad_enabled(False)
    os.chdir(REF)                          # load_average_feature reads a path relative to the checkout
    sys.path.insert(0, REF)
    from oracle import sean_oracle as SO
    import models.sean_codes.models.pix2pix_model as P

    params = SO.synth_sean_params(SEED)
    tmp = tempfile.mkdtemp()
    opt = copy.copy(P.SEAN_OPT)
    opt.gpu_ids, opt.checkpoints_dir = [], tmp
    os.makedirs(os.path.join(tmp, opt.name))
    torch.save(params, os.path.join(tmp, opt.name, "latest_net_G.pth"))
    torch.Tensor.cuda = lambda self, *a, **k: self
    draws = []
    orig_randn = torch.randn
    gen = torch.Generator()

    def randn(*size, device=None, **kw):
        if device == "cuda":
            t = orig_randn(*size, generator=gen)
            draws.append(t.clone())
            return t
        return orig_randn(*size, device=device, **kw)

    model = P.Pix2PixModel(opt)           # util.load_network: strict load of the synthetic state_dict
    model.eval()
    mean = P.load_average_feature()
    mean_codes = torch.stack([mean[str(j)]["ACE"].float() for j in range(19)])
    out = {"mean_codes": mean_codes.numpy(), "n_keys": np.int64(len(params)), "seed": np.int64(SEED)}
    torch.randn = randn
    try:
        for case, labels in enumerate(label_maps()):
            g = torch.Generator().manual_seed(40 + case)
            code = torch.randn(1, 19, 512, generator=g) * 0.5
            code[0, [2, 9, 13]] = 0                      # all-zero rows -> the mean codes
            draws.clear()
            noise_seed = 31 + case
            gen.manual_seed(noise_seed)
            taps = {}
            hooks = [getattr(model.netG, name).register_forward_hook(
                lambda m, i, o, name=name: taps.__setitem__(name, o.clone())) for name, *_ in SO.BLOCKS]
            img = P.decode_sean(model, code, labels.float())
            for h in hooks:
                h.remove()
            assert len(draws) == 18, len(draws)
            assert all(torch.equal(a, b) for a, b in zip(draws, SO.golden_noise(noise_seed)))
            # independent check of the oracle while the reference is at hand
            ours, _ = SO.decode_ref(params, code, labels, mean_codes, draws)
            rms = float(img.pow(2).mean().sqrt())
            print(f"case {case}: image rms {rms:.4g}, oracle max abs {float((img - ours).abs().max()):.3g}; "
                  "block max |x|: " + ", ".join(f"{k} {float(v.abs().max()):.3g}" for k, v in taps.items()))
            out[f"c{case}_labels"] = labels.numpy().astype(np.int8)
            out[f"c{case}_code"] = code.numpy()
            # the draws are regenerated from the seed (SO.golden_noise); their first values pin that regeneration
            out[f"c{case}_noise_seed"] = np.int64(noise_seed)
            out[f"c{case}_noise_head"] = np.stack([d.reshape(-1)[:16].numpy() for d in draws])
            out[f"c{case}_image"] = SO.golden_sample_image(img).numpy()
            for name, t in taps.items():        # one intermediate per resolution
                out[f"c{case}_{name}"] = SO.golden_sample_block(t).numpy()
    finally:
        torch.randn = orig_randn
    np.savez_compressed(os.path.join(GOLD, "sean.npz"), **out)
    print("wrote", os.path.join(GOLD, "sean.npz"))


if __name__ == "__main__":
    main()

"""Golden vectors for HairFast's latent modulation nets: run the UNMODIFIED reference classes of models/Encoders.py
(the checkout oracle/build_ref.py builds, baseline.refenv) on the CPU with the seeded parameters of
``modulation_oracle.synth_params`` and store tests/golden/modulation.npz.  No weights are stored; the tests regenerate
them from the seeds.

Cases: RotateModel at B = 1 and 2 (its inputs the strided ``latent_W[:, :6]`` views, as Alignment.py:61 passes them),
ClipBlendingModel at B = 1 with the two CLIP embeddings stored, and PostProcessModel's latent path (its own
``forward`` with ``encoder_face`` / ``to_feature`` replaced by stand-ins returning the stored codes).  Latent rows get
different scales so that a PixelNorm over the wrong dimension is visible."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
SEEDS = {"rotate": 31, "blending": 32, "post_1": 33, "post_2": 34, "inputs": 35}


def latents(g, batch, rows=18):
    """N(0, 1) rows scaled 0.25 .. 2 by row, so PixelNorm over the rows differs from one over the channels."""
    scale = torch.linspace(0.25, 2.0, rows)[None, :, None]
    return torch.randn(batch, rows, 512, generator=g) * scale


def main():
    torch.set_grad_enabled(False)
    from baseline import refenv
    refenv.activate(overlay=False, chdir=False)
    import clip
    from torch import nn
    import models.Encoders as E
    from oracle import modulation_oracle as O

    g = torch.Generator().manual_seed(SEEDS["inputs"])
    out = {f"seed_{k}": np.int64(v) for k, v in SEEDS.items()}

    rot = E.RotateModel()
    rot.modulation_module_list.load_state_dict(O.stack_state_dict(O.synth_params(SEEDS["rotate"], 6)), strict=True)
    for b in (1, 2):
        w_from, w_to = latents(g, b), latents(g, b)
        out[f"rotate_b{b}_from"], out[f"rotate_b{b}_to"] = w_from.numpy(), w_to.numpy()
        out[f"rotate_b{b}_out"] = rot(w_from[:, :6], w_to[:, :6]).numpy()

    load = clip.load
    clip.load = lambda name, device="cpu", **kw: load(name, device="cpu", **kw)      # the stand-in stays on the CPU
    try:
        bl = E.ClipBlendingModel()
    finally:
        clip.load = load
    bl.modulation_module_list.load_state_dict(O.stack_state_dict(O.synth_params(SEEDS["blending"], 12)), strict=True)
    face_img, color_img = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1, torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    lat_face, lat_color = latents(g, 1, 12), latents(g, 1, 12)
    out["blending_latent_face"], out["blending_latent_color"] = lat_face.numpy(), lat_color.numpy()
    out["blending_embed_face"] = bl.get_image_embed(face_img).numpy()
    out["blending_embed_color"] = bl.get_image_embed(color_img).numpy()
    out["blending_out"] = bl(lat_face, lat_color, face_img, color_img).numpy()

    pp = E.PostProcessModel.__new__(E.PostProcessModel)
    nn.Module.__init__(pp)
    pp.to_latent_1 = nn.ModuleList([E.ModulationModule(18, i == 4) for i in range(5)])
    pp.to_latent_2 = nn.ModuleList([E.ModulationModule(18, i == 4) for i in range(5)])
    pp.to_latent_1.load_state_dict(O.stack_state_dict(O.synth_params(SEEDS["post_1"], 18)), strict=True)
    pp.to_latent_2.load_state_dict(O.stack_state_dict(O.synth_params(SEEDS["post_2"], 18)), strict=True)
    pp.pixelnorm = E.PixelNorm()
    pp.latent_avg = 0.5 * torch.randn(18, 512, generator=g)
    s_face, s_hair = latents(g, 1), latents(g, 1)
    codes = {"source": s_face, "target": s_hair}
    pp.encoder_face = lambda img: (codes[img], [torch.zeros(1, 1, 2, 2)])
    pp.to_feature = nn.Identity()
    finall_s, _ = E.PostProcessModel.forward(pp, "source", "target")
    out["post_s_face"], out["post_s_hair"] = s_face.numpy(), s_hair.numpy()
    out["post_latent_avg"], out["post_out"] = pp.latent_avg.numpy(), finall_s.numpy()

    np.savez_compressed(os.path.join(GOLD, "modulation.npz"), **out)
    print("wrote", os.path.join(GOLD, "modulation.npz"), os.path.getsize(os.path.join(GOLD, "modulation.npz")))


if __name__ == "__main__":
    main()

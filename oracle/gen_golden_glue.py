"""Golden vectors for the stage glue (SURVEY 8f-4): the UNMODIFIED reference ``utils/bicubic.py::BicubicDownSample``
(factor 2 and 4, as Embedding / Blending build it) on CPU -> tests/golden/glue.npz.  Build-container only; test
infrastructure (see oracle/README.md)."""
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
    sys.path.insert(0, REF)
    from utils.bicubic import BicubicDownSample
    from oracle import glue_oracle as GO
    out = {}
    x = torch.rand(2, 3, 96, 160, generator=torch.Generator().manual_seed(61)) * 2 - 1
    out["x"] = x.numpy()
    for f in (2, 4):
        ref = BicubicDownSample(factor=f, cuda=False)
        y = ref(x)
        yo = GO.bicubic_downsample_ref(x, f)
        k_ref = ref.k1[0, 0, :, 0]
        print(f"bicubic f={f}: ref vs oracle max abs", float((y - yo).abs().max()), "taps diff",
              float((k_ref - GO.bicubic_taps(f)).abs().max()), tuple(y.shape))
        out[f"y_f{f}"] = y.numpy()
        out[f"k_f{f}"] = k_ref.numpy()
    x255 = (x + 1) * 127.5
    y = BicubicDownSample(factor=4, cuda=False)(x255, clip_round=True)
    yo = GO.bicubic_downsample_ref(x255, 4, clip_round=True)
    print("bicubic f=4 clip_round: ref vs oracle max abs", float((y - yo).abs().max()))
    out["y_f4_clip_round"] = y.numpy()
    # ---- DilateErosion (utils/image_utils.py:27-55).  The module imports models.Net (-> gdown, clip, the JIT ops):
    # stub what this image lacks, nothing of it is executed by the class.
    import types
    import torch.utils.cpp_extension as ce
    ce.load = lambda *a, **k: None
    for name in ("gdown", "clip"):
        sys.modules.setdefault(name, types.ModuleType(name))
    from utils.image_utils import DilateErosion
    g = torch.Generator().manual_seed(63)
    blobs = (torch.nn.functional.avg_pool2d(torch.rand(3, 1, 64, 96, generator=g), 9, 1, 4) > 0.52).float()
    blobs[0, 0, :3, :] = 1.0                                   # touch the border: zero padding erodes it
    out["mask_in"] = blobs.numpy().astype(np.uint8)
    for it in (1, 5):
        d, e = DilateErosion(dilate_erosion=it, device="cpu").mask(blobs)
        do, eo = GO.dilate_erode_ref(blobs, it)
        print(f"dilate/erode it={it}: ref vs oracle mismatches", int((d != do).sum()), int((e != eo).sum()),
              "ones", int(blobs.sum()), int(d.sum()), int(e.sum()))
        out[f"dilate_it{it}"] = d.numpy().astype(np.uint8)
        out[f"erode_it{it}"] = e.numpy().astype(np.uint8)
    labels = torch.randint(0, 19, (2, 1, 128, 128), generator=g).float()
    d, e = DilateErosion(dilate_erosion=2, device="cpu").hair_from_mask(labels)
    out["labels"] = labels.numpy().astype(np.uint8)
    out["hair_dilate"] = d.numpy().astype(np.uint8)
    out["hair_erode"] = e.numpy().astype(np.uint8)
    # ---- F-space alignment: run the reference's OWN source lines (models/Alignment.py:139-159, the body of
    # align_images between the SEAN re-encoding and the save_all block) on synthetic inputs.  Nothing is copied into the
    # repo: the text is read from the checkout here, dedented and exec'd with the names it uses.
    import textwrap
    import torch.nn.functional as F
    src = open(os.path.join(REF, "models", "Alignment.py")).read().split("\n")
    block = textwrap.dedent("\n".join(src[138:159]))                 # lines 139..159 (1-based)
    assert block.lstrip().startswith("masks = [") and "latent_F_align = latent_F_2" in block, block[:200]
    gm = torch.Generator().manual_seed(64)

    def blob(seed_shift):
        return (torch.nn.functional.avg_pool2d(torch.rand(1, 1, 256, 256, generator=gm), 15, 1, 7) > 0.5).float()
    ns = {"torch": torch, "F": F, "hair_mask1": blob(0), "hair_mask2": blob(1), "hair_mask_target": blob(2),
          "self": types.SimpleNamespace(dilate_erosion=DilateErosion(dilate_erosion=5, device="cpu"))}
    for name in ("intermediate_align", "latent_F_1", "latent_F_out_new", "latent_F_2"):
        ns[name] = torch.randn(1, 64, 32, 32, generator=gm)
    inputs = {k: ns[k].clone() for k in ("hair_mask1", "hair_mask2", "hair_mask_target", "intermediate_align",
                                         "latent_F_1", "latent_F_out_new", "latent_F_2")}
    exec(block, ns)
    mo = GO.align_masks_ref(inputs["hair_mask1"], inputs["hair_mask2"], inputs["hair_mask_target"])
    fo = GO.align_f_space_ref(inputs["intermediate_align"], inputs["latent_F_1"], inputs["latent_F_out_new"],
                              inputs["latent_F_2"], ns["free_mask"])
    print("align masks: ref vs oracle mismatches", int((ns["masks"] != mo).sum()),
          "| latent_F_align ref vs oracle max abs", float((ns["latent_F_align"] - fo).abs().max()))
    for k, v in inputs.items():
        out["fs_" + k] = v.numpy()
    out["fs_masks"] = ns["masks"].numpy().astype(np.uint8)
    out["fs_free_mask"] = ns["free_mask"].numpy().astype(np.uint8)
    out["fs_latent_F_align"] = ns["latent_F_align"].numpy()
    # Embedding mixing (models/Embedding.py:86-92): the three statements inside `if len(images_to_name) > 1:`
    esrc = open(os.path.join(REF, "models", "Embedding.py")).read().split("\n")
    eblock = textwrap.dedent("\n".join(esrc[85:88]) + "\n" + esrc[91])       # lines 86-88 and 92 (1-based)
    assert "hair_mask = torch.where(masks == 13" in eblock and "latent_F = latent_F + self.opts.mixing" in eblock, eblock
    labels = torch.randint(10, 16, (2, 1, 256, 256), generator=gm)
    labels = torch.nn.functional.interpolate(labels[:, :, ::16, ::16].float(), size=(256, 256), mode="nearest").long()
    ens = {"torch": torch, "F": F, "masks": labels, "device": "cpu",
           "latent_F": torch.randn(2, 64, 32, 32, generator=gm), "latent_F_from_W": torch.randn(2, 64, 32, 32, generator=gm),
           "self": types.SimpleNamespace(opts=types.SimpleNamespace(mixing=0.95))}
    out["mix_labels"] = labels.numpy().astype(np.uint8)
    out["mix_latent_F"] = ens["latent_F"].numpy().copy()
    out["mix_latent_F_from_W"] = ens["latent_F_from_W"].numpy()
    lf0 = ens["latent_F"].clone()
    exec(eblock, ens)
    mo = GO.mix_f_space_ref(lf0, ens["latent_F_from_W"], labels, 0.95)
    print("embedding mixing: ref vs oracle max abs", float((ens["latent_F"] - mo).abs().max()))
    out["mix_out"] = ens["latent_F"].numpy()
    np.savez_compressed(os.path.join(GOLD, "glue.npz"), **out)
    print("glue.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()

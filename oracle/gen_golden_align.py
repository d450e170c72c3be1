"""Golden vectors of the FFHQ face alignment: run the UNMODIFIED reference ``align_face`` (utils/shape_predictor.py:80-194,
the checkout oracle/build_ref.py builds, baseline.refenv) on the seeded synthetic cases of ``align_oracle.CASES`` and
store tests/golden/align.npz.

dlib is replaced inside ``utils.shape_predictor`` by a stand-in whose detector returns one rectangle and whose predictor
returns the case's landmarks.  Pillow >= 10 no longer has ``Image.ANTIALIAS``, which the shrink branch (:149) names; it
was always an alias of ``LANCZOS`` and is restored as such here.  Each case stores its landmarks, its image parameters
(the image is rebuilt from them by ``align_oracle.synth_image``), the uint8 output of ``return_tensors=False`` (stored
per channel as its differences along each row, modulo 256, which compress several times better; a PIL or float case
whose pixels equal those of the uint8 case with the same parameters names that twin instead) and the boxes the reference used (recorded from its ``Image.resize``, ``Image.crop`` and ``np.pad`` calls).  The float output
of ``return_tensors=True`` is checked here to be ``ToTensor()`` of the same image."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def main():
    from baseline import refenv
    refenv.activate(overlay=False, chdir=False)
    import PIL.Image
    import utils.shape_predictor as sp
    from oracle import align_oracle as O
    from oracle.align_oracle import FakeDlib

    if not hasattr(PIL.Image, "ANTIALIAS"):
        PIL.Image.ANTIALIAS = PIL.Image.LANCZOS
    out = {"case_names": np.array(list(O.CASES))}
    calls = []
    crop0, resize0, pad0 = PIL.Image.Image.crop, PIL.Image.Image.resize, np.pad

    def crop(self, box=None):
        calls.append(("crop", tuple(int(v) for v in box)))
        return crop0(self, box)

    def resize(self, size, *a, **k):
        calls.append(("resize", tuple(int(v) for v in size)))
        return resize0(self, size, *a, **k)

    def pad(array, pad_width, *a, **k):
        calls.append(("pad", tuple(int(v) for v in np.asarray(pad_width).ravel())))
        return pad0(array, pad_width, *a, **k)

    dlib = sp.dlib
    PIL.Image.Image.crop, PIL.Image.Image.resize, np.pad = crop, resize, pad
    try:
        for name, (h, w, seed, mid, io, angle, form) in O.CASES.items():
            data, lm, _ = O.case_input(name)
            fake = FakeDlib([lm])
            sp.dlib = fake
            calls.clear()
            imgs = sp.align_face([data], fake.predictor, return_tensors=False)
            boxes = list(calls)
            tens = sp.align_face([data], fake.predictor, return_tensors=True)
            assert len(imgs) == 1 and len(tens) == 1 and imgs[0].mode == "RGB" and imgs[0].size == (1024, 1024)
            img = np.asarray(imgs[0])
            assert torch.equal(tens[0], torch.from_numpy(img).permute(2, 0, 1).float().div(255).clamp(0, 1))
            out[f"{name}_lm"] = lm
            out[f"{name}_params"] = np.array([h, w, seed, mid[0], mid[1], io], dtype=np.int64)
            out[f"{name}_angle"] = np.float64(angle)
            twins = [n for n, c in O.CASES.items() if c[:6] == O.CASES[name][:6] and c[6] == "u8" and n != name]
            if twins and np.array_equal(img, O.decode_output(out[f"{twins[0]}_out_dx"])):
                out[f"{name}_twin"] = np.array(twins[0])      # same pixels as the uint8 case of the same parameters
            else:
                out[f"{name}_out_dx"] = O.encode_output(img)
            rs = [v for k, v in boxes if k == "resize" and v != (1024, 1024)]
            cr = [v for k, v in boxes if k == "crop"]
            pd = [v for k, v in boxes if k == "pad"]
            # np.pad widths ((top, bottom), (left, right), (0, 0)) -> (left, top, right, bottom)
            out[f"{name}_rsize"] = np.array(rs[0] if rs else (-1, -1), dtype=np.int64)
            out[f"{name}_crop"] = np.array(cr[0] if cr else (-1,) * 4, dtype=np.int64)
            out[f"{name}_pad"] = np.array((pd[0][2], pd[0][0], pd[0][3], pd[0][1]) if pd else (-1,) * 4, dtype=np.int64)
            print(name, "rsize", rs, "crop", cr, "pad", pd)
    finally:
        PIL.Image.Image.crop, PIL.Image.Image.resize, np.pad = crop0, resize0, pad0
        sp.dlib = dlib
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "align.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

"""Golden vectors for CtrlHair's shape adaptor: run the UNMODIFIED reference ``Generator(cfg)`` (config 054) with
``get_hair_face_code`` / ``get_new_shape`` (models/CtrlHair/shape_branch/solver.py:248-262) on the CPU with the seeded
parameters of ``shape_adaptor_oracle.synth_params`` and store tests/golden/shape_adaptor.npz.  The reference is the
one oracle/build_ref.py builds (baseline.refenv); no weights are stored, the tests regenerate them from the seed.

Per label case: the mask, both codes, the output labels and the fp16 top-2 logit margin per pixel.  The new shape is
decoded from the case's own face code and the hair code of the next case, as ``shape_module`` mixes two masks."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
SEED = 7


def main():
    torch.set_grad_enabled(False)
    from baseline import refenv
    refenv.activate(overlay=False, chdir=False)
    from models.CtrlHair.shape_branch import solver
    from oracle import shape_adaptor_oracle as O

    gen = O.reference_generator()
    assert [(k, tuple(v.shape)) for k, v in gen.state_dict().items()] == list(O.config054_shapes().items())
    params = O.synth_params(SEED)
    gen.load_state_dict(params, strict=True)
    cases = O.label_cases()
    names = list(cases)
    out = {"seed": np.int64(SEED), "names": np.array(names)}
    codes = {n: solver.get_hair_face_code(gen, cases[n].clone()) for n in names}
    for i, n in enumerate(names):
        hair_from = names[(i + 1) % len(names)]
        face_code, hair_code = codes[n][0], codes[hair_from][1]
        labels = solver.get_new_shape(gen, face_code, hair_code)
        # the logits, for the per-pixel margin: forward_decode_by_code without the softmax
        hl = gen.forward_hair_decoder(hair_code, face_code)
        fl = gen.forward_face_decoder(face_code)
        lg = torch.cat([fl[:, :O.HAIR_IDX], hl, fl[:, O.HAIR_IDX:]], 1)[0]
        assert torch.equal(lg.argmax(0), labels)
        out[f"{n}_mask"] = cases[n].numpy().astype(np.uint8)
        out[f"{n}_face_code"] = codes[n][0].numpy()
        out[f"{n}_hair_code"] = codes[n][1].numpy()
        out[f"{n}_hair_from"] = np.array(hair_from)
        out[f"{n}_labels"] = labels.numpy().astype(np.uint8)
        out[f"{n}_margin"] = O.top2_margin(lg.double()).numpy().astype(np.float16)
        print(f"{n}: hair from {hair_from}, classes out {sorted(set(labels.unique().tolist()))}, "
              f"min margin {float(out[f'{n}_margin'].min()):.3g}")
    np.savez_compressed(os.path.join(GOLD, "shape_adaptor.npz"), **out)
    print("wrote", os.path.join(GOLD, "shape_adaptor.npz"), os.path.getsize(os.path.join(GOLD, "shape_adaptor.npz")))


if __name__ == "__main__":
    main()

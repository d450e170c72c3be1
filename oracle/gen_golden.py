"""Generate the committed golden vectors under tests/golden/ by running the
UNMODIFIED reference (imported from the checkout named by HAIRFAST_REFERENCE, CPU fp32 branches) on
seeded synthetic parameters.  Test infrastructure only (see oracle/README.md).

Run once in the build container (the reference does not exist on the GPU box):

    python oracle/gen_golden.py

The reference's op package JIT-builds two CUDA extensions at import time
(models/stylegan2/op/fused_act.py:10-16, upfirdn2d.py:10-16).  CPU tensors never
touch them (fused_act.py:86, upfirdn2d.py:146), so ``cpp_extension.load`` is
stubbed for this process; nothing in the checkout is modified or copied.
"""
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


def import_reference():
    import torch.utils.cpp_extension as ce
    ce.load = lambda *a, **k: None          # CPU branches never call into it
    sys.path.insert(0, REF)
    import models.stylegan2.model as ref_model
    import models.stylegan2.op as ref_op
    return ref_model, ref_op


def main():
    torch.set_grad_enabled(False)
    from oracle import stylegan2_oracle as O
    ref_model, ref_op = import_reference()
    os.makedirs(GOLD, exist_ok=True)

    # ---- 1. op level: upfirdn2d (every mode the reference dispatches) + fused_leaky_relu
    g = torch.Generator().manual_seed(10)
    x = torch.randn(2, 3, 9, 9, generator=g)
    k4 = O.make_kernel([1, 3, 3, 1])
    k3 = O.make_kernel([1, 2, 1])
    kasym = torch.randn(4, 4, generator=g)        # non-symmetric: pins the flip
    cases = {
        "blur_up1_k4_pad11": (k4 * 4, 1, 1, (1, 1)),      # Blur after up-conv, model.py:204-210
        "rgbup_up2_k4_pad21": (k4 * 4, 2, 1, (2, 1)),     # Upsample of the skip, model.py:40-48
        "down2_k4_pad11": (k4, 1, 2, (1, 1)),             # Downsample, model.py:56-74
        "asym_up2_down1": (kasym, 2, 1, (2, 1)),
        "asym_up1_down2_pad20": (kasym, 1, 2, (2, 0)),
        "k3_up1_negpad": (k3, 1, 1, (-1, 2)),
        "asym_up2_down2": (kasym, 2, 2, (1, 2)),
    }
    out = {"x": x.numpy()}
    for name, (k, up, down, pad) in cases.items():
        y = ref_op.upfirdn2d(x, k, up=up, down=down, pad=pad)
        out[name + "__k"] = k.numpy()
        out[name + "__cfg"] = np.array([up, down, pad[0], pad[1]], dtype=np.int64)
        out[name + "__y"] = y.numpy()
    xb = torch.randn(2, 5, 4, 6, generator=g)
    bb = torch.randn(5, generator=g)
    out["lrelu_x"] = xb.numpy(); out["lrelu_b"] = bb.numpy()
    out["lrelu_y"] = ref_op.fused_leaky_relu(xb, bb).numpy()
    x2 = torch.randn(3, 5, generator=g)
    out["lrelu2d_x"] = x2.numpy()
    out["lrelu2d_y"] = ref_op.fused_leaky_relu(x2, bb).numpy()
    np.savez_compressed(os.path.join(GOLD, "ops.npz"), **out)
    print("ops.npz", len(out))

    # ---- 2. module level: ModulatedConv2d / StyledConv / ToRGB on small shapes
    out = {}
    torch.manual_seed(0)
    for name, (cin, cout, r, up) in {"plain_64_48_r8": (64, 48, 8, False),
                                     "up_64_32_r8": (64, 32, 8, True),
                                     "plain_32_32_r16": (32, 32, 16, False)}.items():
        m = ref_model.StyledConv(cin, cout, 3, 512, upsample=up)
        m.noise.weight.data.normal_(0, 0.3)
        m.activate.bias.data.normal_(0, 0.3)
        m.conv.modulation.bias.data.add_(0.1 * torch.randn(cin))
        xx = torch.randn(2, cin, r, r); st = torch.randn(2, 512)
        ro = r * 2 if up else r
        nz = torch.randn(2, 1, ro, ro)
        out[name + "__x"] = xx.numpy(); out[name + "__style"] = st.numpy(); out[name + "__noise"] = nz.numpy()
        for kk, vv in m.state_dict().items():
            out[name + "__p__" + kk] = vv.numpy()
        out[name + "__modconv"] = m.conv(xx, st).numpy()
        out[name + "__styled"] = m(xx, st, noise=nz).numpy()
    m = ref_model.ToRGB(64, 512)
    m.bias.data.normal_(0, 0.3)
    xx = torch.randn(2, 64, 8, 8); st = torch.randn(2, 512); sk = torch.randn(2, 3, 4, 4)
    out["torgb__x"] = xx.numpy(); out["torgb__style"] = st.numpy(); out["torgb__skip"] = sk.numpy()
    for kk, vv in m.state_dict().items():
        out["torgb__p__" + kk] = vv.numpy()
    out["torgb__y_skip"] = m(xx, st, sk).numpy()
    out["torgb__y_noskip"] = m(xx, st, None).numpy()
    np.savez_compressed(os.path.join(GOLD, "modules.npz"), **out)
    print("modules.npz", len(out))

    # ---- 3. config 1 of BASELINE.json: ModulatedConv2d 512->512 @64^2, B=1 (SURVEY 8d)
    torch.manual_seed(0)
    m = ref_model.ModulatedConv2d(512, 512, 3, 512)
    m.modulation.weight.data.normal_()            # EqualLinear ctor already N(0,1); explicit per 8d
    xx = torch.randn(1, 512, 64, 64); st = torch.randn(1, 512)
    y = m(xx, st)
    # inputs are re-derivable from the seed; store the output subsampled + full stats
    np.savez_compressed(os.path.join(GOLD, "config1_modconv512.npz"),
                        y_sub=y[:, ::8, ::4, ::4].numpy(), y_absmax=float(y.abs().max()),
                        y_mean=float(y.mean()), y_std=float(y.std()),
                        weight_sub=m.weight[0, ::64, ::64].numpy(), x_sub=xx[0, ::64, ::8, ::8].numpy(),
                        style=st.numpy())
    print("config1_modconv512.npz")

    # ---- 4. generator level: size=256 generator (channels 512..128), every partial range swap() uses
    size = 256
    params = O.synth_generator_params(size=size, seed=0)
    gen = ref_model.Generator(size, 512, 8)
    missing = gen.load_state_dict(params, strict=True)      # pins the 135-key layout
    gen.eval()
    lat = torch.randn(2, gen.n_latent, 512, generator=torch.Generator().manual_seed(2))
    noise = O.synth_noise(size, batch=2, seed=3)
    out = {"latent": lat.numpy()}
    img, _ = gen([lat], input_is_latent=True, noise=noise)
    out["full__image"] = img[:, :, ::4, ::4].numpy()
    out["full__image_absmax"] = np.float32(img.abs().max())
    out["full__image_sum"] = np.float64(img.double().sum())
    f03, s03 = gen([lat], input_is_latent=True, noise=noise, start_layer=0, end_layer=3)
    out["r0_3__out"] = f03[:, ::8].numpy(); out["r0_3__skip"] = s03.numpy()
    g2 = torch.Generator().manual_seed(4)
    lin16 = torch.randn(2, 512, 16, 16, generator=g2)
    f33, s33 = gen([lat], input_is_latent=True, noise=noise, start_layer=3, end_layer=3, layer_in=lin16)
    out["layer_in16"] = lin16[:, ::8].numpy()
    out["r3_3__out"] = f33[:, ::8].numpy(); out["r3_3__skip"] = s33.numpy()
    lin32 = torch.randn(2, 512, 32, 32, generator=g2)
    i46, _ = gen([lat], input_is_latent=True, noise=noise, start_layer=4, end_layer=8, layer_in=lin32)
    out["r4_end__image"] = i46[:, :, ::4, ::4].numpy()
    lin64 = torch.randn(2, 512, 64, 64, generator=g2)
    i56, _ = gen([lat], input_is_latent=True, noise=noise, start_layer=5, end_layer=8, layer_in=lin64)
    out["r5_end__image"] = i56[:, :, ::4, ::4].numpy()
    # stored-noise path (randomize_noise=False uses the registered buffers, model.py:500-503)
    ib, _ = gen([lat[:1]], input_is_latent=True, randomize_noise=False)
    out["bufnoise__image"] = ib[:, :, ::4, ::4].numpy()
    # mapping network (not used by swap(), part of the Generator surface)
    z = torch.randn(3, 512, generator=g2)
    out["z"] = z.numpy(); out["mapping__w"] = gen.get_latent(z).numpy()
    np.savez_compressed(os.path.join(GOLD, "generator256.npz"), **out)
    print("generator256.npz", len(out))

    # ---- 4b. FeatureStyleEncoder's generator copy: insert_feature at idx 5 (alpha = 1) + return_features
    sys.path.insert(0, os.path.join(REF, "models", "FeatureStyleEncoder"))
    from pixel2style2pixel.models.stylegan2.model import Generator as FSEGenerator
    fgen = FSEGenerator(size, 512, 8)
    fgen.load_state_dict(params, strict=True)
    fgen.eval()
    fea = torch.randn(2, 512, 16, 16, generator=torch.Generator().manual_seed(6))
    feats = [None] * 5 + [fea] + [None] * 12
    fimg, fouts = fgen([lat], input_is_latent=True, noise=noise, return_features=True, features_in=feats,
                       feature_scale=1.0)
    np.savez_compressed(os.path.join(GOLD, "generator256_fse.npz"),
                        image=fimg[:, :, ::4, ::4].numpy(), n_outs=np.int64(len(fouts)),
                        out0=fouts[0][:, ::64].numpy(), out4=fouts[4][:, ::16].numpy(),
                        out5=fouts[5][:, ::16].numpy(), out6=fouts[6][:, ::16, ::2, ::2].numpy(),
                        out_last=fouts[-1][:, ::16, ::8, ::8].numpy())
    print("generator256_fse.npz", len(fouts))

    # ---- 5. full-size 1024^2 generator, B=1 (config 2 shape), subsampled output
    size = 1024
    params = O.synth_generator_params(size=size, seed=0)
    gen = ref_model.Generator(size, 512, 8)
    gen.load_state_dict(params, strict=True)                # pins the 171-key layout
    lat = torch.randn(1, 18, 512, generator=torch.Generator().manual_seed(0))
    noise = O.synth_noise(size, batch=1, seed=1)
    img, _ = gen([lat], input_is_latent=True, noise=noise)
    np.savez_compressed(os.path.join(GOLD, "generator1024.npz"),
                        image_sub=img[:, :, ::16, ::16].numpy(),
                        image_rows=img[:, :, 511:513, :].numpy(),
                        image_absmax=np.float32(img.abs().max()),
                        image_sum=np.float64(img.double().sum()),
                        image_sqsum=np.float64((img.double() ** 2).sum()))
    print("generator1024.npz")


if __name__ == "__main__":
    main()

"""CPU oracle for SEAN's ``decode_sean`` (SPADE generator in UI_mode).  TEST INFRASTRUCTURE ONLY -- same rules as
stylegan2_oracle.py (imported only by tests/, tools/ and the golden script).

Functional fp32 restatement (torch CPU, no nn.Module, no reference imports), in the reference's plain convolution form:
* ``decode_sean`` -- models/sean_codes/models/pix2pix_model.py:309-325 (per-class code or mean code, :312-315);
  ``preprocess_input`` one-hot map (:124-149);
* ``SPADEGenerator.forward`` -- models/sean_codes/models/networks/generator.py:72-109 (num_upsampling_layers='normal');
* ``SPADEResnetBlock.forward`` -- models/sean_codes/models/networks/architecture.py:69-96, spectral-norm convolutions
  in eval mode (weight = weight_orig / (u . W v), no power iteration);
* ``ACE.forward`` (status 'UI_mode') and ``SPADE.forward`` -- models/sean_codes/models/networks/normalization.py:108-189,
  249-257; eval-mode ``SynchronizedBatchNorm2d(affine=False)`` = running statistics, eps 1e-5.

It also states the lookup-table forms the CUDA path uses (``onehot_table`` / ``onehot_conv_lut`` / ``style_tables`` /
``style_conv_lut``); tests/test_sean_oracle.py checks them against the plain convolutions.

Pinned by tests/golden/sean.npz, produced by oracle/gen_golden_sean.py from the unmodified reference
``Pix2PixModel(SEAN_OPT)`` with the seeded parameters of ``synth_sean_params`` (no pretrained weights exist).
"""
from __future__ import annotations

import types
import zlib
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor

N_CLASSES = 19
STYLE = 512
NHIDDEN = 128
SIZE = 256
# (name, fin, fout, resolution, use_rgb); generator.py:35-43 with ngf = 64; a nearest 2x upsample precedes every block
# but head_0 and G_middle_1 (generator.py:83-101)
BLOCKS = [("head_0", 1024, 1024, 8, True), ("G_middle_0", 1024, 1024, 16, True), ("G_middle_1", 1024, 1024, 16, True),
          ("up_0", 1024, 512, 32, True), ("up_1", 512, 256, 64, True), ("up_2", 256, 128, 128, True),
          ("up_3", 128, 64, 256, False)]
UPSAMPLE_BEFORE = {"G_middle_0", "up_0", "up_1", "up_2", "up_3"}


def block_aces(fin: int, fout: int) -> List[Tuple[str, int]]:
    """ACE layers of one block in the order their noise is drawn: ace_s (learned shortcut, computed first by
    ``shortcut``), ace_0, ace_1 (architecture.py:69-93)."""
    fmid = min(fin, fout)
    return ([("ace_s", fin)] if fin != fout else []) + [("ace_0", fin), ("ace_1", fmid)]


def noise_shapes() -> List[Tuple[int, int, int, int]]:
    """Shapes of the 18 ``torch.randn(1, W, H, 1)`` draws (normalization.py:111) in draw order."""
    return [(1, res, res, 1) for _, fin, fout, res, _ in BLOCKS for _ in block_aces(fin, fout)]


def golden_noise(seed: int) -> List[Tensor]:
    """The 18 ACE noise draws of one golden case: ``torch.randn`` of ``noise_shapes()`` in order from a CPU generator
    seeded with `seed` (tests/golden/sean.npz stores the seed and the first values of each draw, not the draws)."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g) for s in noise_shapes()]


def golden_sample_image(img: Tensor) -> Tensor:
    """The part of the [3,256,256] image the golden stores: every fourth pixel."""
    return img[:, ::4, ::4]


def golden_sample_block(x: Tensor) -> Tensor:
    """The part of a [1,C,R,R] block output the golden stores: 16 channels, at most 16 x 16 pixels."""
    c, r = x.shape[1], x.shape[-1]
    return x[0, ::c // 16, ::max(1, r // 16), ::max(1, r // 16)]


# ------------------------------------------------------------------------------------------------ parameters
def sean_param_layout() -> List[Tuple[str, Tuple[int, ...]]]:
    """Key / shape layout of ``SPADEGenerator(SEAN_OPT).state_dict()`` (pinned against the reference class by the
    strict load in gen_golden_sean.py)."""
    L: List[Tuple[str, Tuple[int, ...]]] = []
    zc = [(1, 32, 3), (4, 64, 32), (7, 128, 64), (10, 128, 256), (14, 512, 256)]     # architecture.py:154-175
    for idx, cout, cin in zc:
        L += [(f"Zencoder.model.{idx}.weight", (cout, cin, 3, 3)), (f"Zencoder.model.{idx}.bias",
                                                                   (cin if idx == 10 else cout,))]
    L += [("fc.weight", (1024, N_CLASSES, 3, 3)), ("fc.bias", (1024,))]
    for name, fin, fout, _, use_rgb in BLOCKS:
        fmid = min(fin, fout)
        for conv, ci, co, k, bias in [("conv_0", fin, fmid, 3, True), ("conv_1", fmid, fout, 3, True)] + (
                [("conv_s", fin, fout, 1, False)] if fin != fout else []):
            if bias:
                L.append((f"{name}.{conv}.bias", (co,)))
            L += [(f"{name}.{conv}.weight_orig", (co, ci, k, k)), (f"{name}.{conv}.weight_u", (co,)),
                  (f"{name}.{conv}.weight_v", (ci * k * k,))]
        for ace, c in block_aces(fin, fout):
            p = f"{name}.{ace}."
            L += [(p + "blending_gamma", (1,)), (p + "blending_beta", (1,)), (p + "noise_var", (c,))]
            L += [(p + "Spade.param_free_norm.running_mean", (c,)), (p + "Spade.param_free_norm.running_var", (c,)),
                  (p + "Spade.param_free_norm.num_batches_tracked", ()),
                  (p + "Spade.mlp_shared.0.weight", (NHIDDEN, N_CLASSES, 3, 3)), (p + "Spade.mlp_shared.0.bias", (NHIDDEN,)),
                  (p + "Spade.mlp_gamma.weight", (c, NHIDDEN, 3, 3)), (p + "Spade.mlp_gamma.bias", (c,)),
                  (p + "Spade.mlp_beta.weight", (c, NHIDDEN, 3, 3)), (p + "Spade.mlp_beta.bias", (c,)),
                  (p + "param_free_norm.running_mean", (c,)), (p + "param_free_norm.running_var", (c,)),
                  (p + "param_free_norm.num_batches_tracked", ())]
            if use_rgb:
                for j in range(N_CLASSES):
                    L += [(p + f"fc_mu{j}.weight", (STYLE, STYLE)), (p + f"fc_mu{j}.bias", (STYLE,))]
                L += [(p + "conv_gamma.weight", (c, STYLE, 3, 3)), (p + "conv_gamma.bias", (c,)),
                      (p + "conv_beta.weight", (c, STYLE, 3, 3)), (p + "conv_beta.bias", (c,))]
    L += [("conv_img.weight", (3, 64, 3, 3)), ("conv_img.bias", (3,))]
    return L


def _fan_in(shape) -> int:
    return int(np.prod(shape[1:])) if len(shape) > 1 else 1


def synth_sean_params(seed: int) -> Dict[str, Tensor]:
    """Seeded parameters that make every term of the decode matter: non-zero noise_var and blending logits, BatchNorm
    running statistics away from (0, 1), spectral-norm u / v consistent with weight_orig (u = W v / |W v|).  Each key
    draws from its own generator (seed, crc32(key)), so the values do not depend on the key order."""
    out: Dict[str, Tensor] = {}
    for key, shape in sean_param_layout():
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(key.encode()))
        leaf = key.rsplit(".", 1)[-1]
        if leaf == "num_batches_tracked":
            out[key] = torch.zeros((), dtype=torch.int64)
            continue
        r = torch.randn(shape, generator=g)
        if leaf == "running_mean":
            v = 0.2 * r
        elif leaf == "running_var":
            v = 0.5 + 1.5 * torch.rand(shape, generator=g)
        elif leaf in ("blending_gamma", "blending_beta"):
            v = r
        elif leaf == "noise_var":
            v = 0.2 * r
        elif leaf in ("weight_u", "weight_v"):
            continue                                         # filled from weight_orig below
        elif key.startswith("fc.") or "mlp_shared" in key:
            v = 0.3 * r if leaf == "weight" else 0.1 * r
        elif "fc_mu" in key:
            v = r / STYLE ** 0.5 if leaf == "weight" else 0.1 * r
        elif leaf == "weight_orig" or leaf == "weight":
            gain = 0.5 if ("mlp_" in key or "conv_gamma" in key or "conv_beta" in key) else 1.0
            v = r / _fan_in(shape) ** 0.5 * (0.3 if key.startswith("conv_img") else gain)
        else:                                                # biases
            v = 0.05 * r
        out[key] = v.contiguous()
    for key in [k for k in out if k.endswith(".weight_orig")]:
        pre = key[: -len("weight_orig")]
        w = out[key].reshape(out[key].shape[0], -1)
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32((pre + "weight_v").encode()))
        v = torch.randn(w.shape[1], generator=g)
        v = v / v.norm()
        u = w @ v
        out[pre + "weight_u"], out[pre + "weight_v"] = (u / u.norm()).contiguous(), v.contiguous()
    # BatchNorm running statistics: those of one seeded decode (blocky labels, random codes, noise drawn as in
    # normalization.py:111), perturbed -- with independent random statistics the residual stream grows ~5x per block
    g = torch.Generator().manual_seed(seed * 1000003 + 7)
    labels = torch.randint(0, N_CLASSES, (1, 1, 16, 16), generator=g).repeat_interleave(16, 2).repeat_interleave(16, 3)
    code = torch.randn(1, N_CLASSES, STYLE, generator=g) * 0.5
    noise = [torch.randn(s, generator=g) for s in noise_shapes()]
    decode_ref(out, code, labels, code[0], noise, calib=g)
    return out


# ------------------------------------------------------------------------------------------------ plain form
def spectral_weight(p: Dict[str, Tensor], pre: str) -> Tensor:
    """torch.nn.utils.spectral_norm in eval mode: weight_orig / (u . (W v))."""
    w = p[pre + "weight_orig"]
    sigma = torch.dot(p[pre + "weight_u"], w.reshape(w.shape[0], -1) @ p[pre + "weight_v"])
    return w / sigma


def one_hot(labels: Tensor) -> Tensor:
    """preprocess_input (pix2pix_model.py:136-141): [1,1,H,W] int64 -> [1,19,H,W] fp32."""
    b, _, h, w = labels.shape
    return torch.zeros(b, N_CLASSES, h, w).scatter_(1, labels.long(), 1.0)


def style_codes(image_code: Tensor, mean_codes: Tensor) -> Tensor:
    """pix2pix_model.py:310-315: [19,512] -- image_code[0, j] unless that row is all zero, else the mean code."""
    rows = [image_code[0, j] if not torch.all(image_code[0, j] == 0) else mean_codes[j] for j in range(N_CLASSES)]
    return torch.stack(rows).float()


def ace_ref(p: Dict[str, Tensor], pre: str, x: Tensor, seg: Tensor, codes: Tensor, rnd: Tensor, use_rgb: bool,
            calib: Optional[torch.Generator] = None) -> Tensor:
    """normalization.py:108-189 (UI_mode, batch 1) with SPADE (:249-257).  ``calib``: first set the BatchNorm running
    statistics to this input's channel statistics, perturbed (what a trained network's statistics look like)."""
    noise = (rnd * p[pre + "noise_var"]).transpose(1, 3)
    if calib is not None:
        v = x + noise
        mean, var = v.mean((0, 2, 3)), v.var((0, 2, 3)) + 1e-3
        p[pre + "param_free_norm.running_mean"] = mean + 0.2 * var.sqrt() * torch.randn(mean.shape, generator=calib)
        p[pre + "param_free_norm.running_var"] = var * (0.5 + 1.5 * torch.rand(var.shape, generator=calib))
    normalized = F.batch_norm(x + noise, p[pre + "param_free_norm.running_mean"], p[pre + "param_free_norm.running_var"],
                              None, None, False, 0.0, 1e-5)
    segmap = F.interpolate(seg, size=x.shape[2:], mode="nearest")
    actv = F.relu(F.conv2d(segmap, p[pre + "Spade.mlp_shared.0.weight"], p[pre + "Spade.mlp_shared.0.bias"], padding=1))
    gamma_spade = F.conv2d(actv, p[pre + "Spade.mlp_gamma.weight"], p[pre + "Spade.mlp_gamma.bias"], padding=1)
    beta_spade = F.conv2d(actv, p[pre + "Spade.mlp_beta.weight"], p[pre + "Spade.mlp_beta.bias"], padding=1)
    if not use_rgb:
        return normalized * (1 + gamma_spade) + beta_spade
    h, w = x.shape[2:]
    middle_avg = torch.zeros(1, STYLE, h, w)
    for j in range(segmap.shape[1]):
        mask = segmap[0, j].bool()
        if mask.any():
            mu = F.relu(F.linear(codes[j], p[pre + f"fc_mu{j}.weight"], p[pre + f"fc_mu{j}.bias"]))
            middle_avg[0][:, mask] = mu[:, None]
    gamma_avg = F.conv2d(middle_avg, p[pre + "conv_gamma.weight"], p[pre + "conv_gamma.bias"], padding=1)
    beta_avg = F.conv2d(middle_avg, p[pre + "conv_beta.weight"], p[pre + "conv_beta.bias"], padding=1)
    ga, ba = torch.sigmoid(p[pre + "blending_gamma"]), torch.sigmoid(p[pre + "blending_beta"])
    gamma = ga * gamma_avg + (1 - ga) * gamma_spade
    beta = ba * beta_avg + (1 - ba) * beta_spade
    return normalized * (1 + gamma) + beta


def block_ref(p, name, fin, fout, use_rgb, x, seg, codes, noise_iter, calib=None) -> Tensor:
    """architecture.py:69-96."""
    pre = name + "."
    if fin != fout:
        xs = ace_ref(p, pre + "ace_s.", x, seg, codes, next(noise_iter), use_rgb, calib)
        xs = F.conv2d(xs, spectral_weight(p, pre + "conv_s."))
    else:
        xs = x
    dx = ace_ref(p, pre + "ace_0.", x, seg, codes, next(noise_iter), use_rgb, calib)
    dx = F.conv2d(F.leaky_relu(dx, 0.2), spectral_weight(p, pre + "conv_0."), p[pre + "conv_0.bias"], padding=1)
    dx = ace_ref(p, pre + "ace_1.", dx, seg, codes, next(noise_iter), use_rgb, calib)
    dx = F.conv2d(F.leaky_relu(dx, 0.2), spectral_weight(p, pre + "conv_1."), p[pre + "conv_1.bias"], padding=1)
    return xs + dx


@torch.no_grad()
def decode_ref(p: Dict[str, Tensor], image_code: Tensor, labels: Tensor, mean_codes: Tensor,
               noise: List[Tensor], calib: Optional[torch.Generator] = None) -> Tuple[Tensor, Dict[str, Tensor]]:
    """decode_sean (pix2pix_model.py:309-325) -> ([3,256,256] image, {block name: block output [1,C,R,R]})."""
    codes = style_codes(image_code.float(), mean_codes.float())
    seg = one_hot(labels)
    x = F.conv2d(F.interpolate(seg, size=(8, 8)), p["fc.weight"], p["fc.bias"], padding=1)
    it = iter(noise)
    taps = {}
    for name, fin, fout, _, use_rgb in BLOCKS:
        if name in UPSAMPLE_BEFORE:
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        x = block_ref(p, name, fin, fout, use_rgb, x, seg, codes, it, calib)
        taps[name] = x
    img = torch.tanh(F.conv2d(F.leaky_relu(x, 0.2), p["conv_img.weight"], p["conv_img.bias"], padding=1))
    return img[0], taps


# ------------------------------------------------------------------------------------------------ lookup-table form
def label_map(labels: Tensor, res: int) -> Tensor:
    """Nearest downsampling of the [1,1,S,S] labels to [res,res]: L[y,x] = label[y*S/res, x*S/res]."""
    s = labels.shape[-1]
    f = s // res
    return labels[0, 0, ::f, ::f].long()


def onehot_table(weight: Tensor) -> Tensor:
    """Conv2d(19 -> Cout, 3x3) weight [Cout,19,3,3] -> table [9][19][Cout] (tap = ky*3 + kx)."""
    return weight.permute(2, 3, 1, 0).reshape(9, weight.shape[1], weight.shape[0]).contiguous()


def _tap_gather(L: Tensor, table_fn, cout: int) -> Tensor:
    """sum over the 3x3 taps inside the map of table_fn(tap)[L(p + tap)]: [Cout, R, R]."""
    r = L.shape[0]
    out = torch.zeros(cout, r, r)
    for tap in range(9):
        dy, dx = tap // 3 - 1, tap % 3 - 1
        ys, xs = slice(max(0, -dy), r - max(0, dy)), slice(max(0, -dx), r - max(0, dx))
        src = L[max(0, dy): r - max(0, -dy), max(0, dx): r - max(0, -dx)]
        out[:, ys, xs] += table_fn(tap)[src].permute(2, 0, 1)
    return out


def onehot_conv_lut(L: Tensor, weight: Tensor, bias: Tensor) -> Tensor:
    """conv2d(one_hot(L), weight, bias, padding=1) as y[p] = b + sum_{valid taps} W[:, L(p+tap), tap]: [Cout,R,R]."""
    t = onehot_table(weight)
    return _tap_gather(L, lambda tap: t[tap], weight.shape[0]) + bias.view(-1, 1, 1)


def style_tables(weight: Tensor, mu: Tensor) -> Tensor:
    """T[j][tap][c] = W[c, :, tap] . mu_j for a [C,512,3,3] weight and the [19,512] class vectors mu."""
    return torch.einsum("ckt,jk->jtc", weight.reshape(weight.shape[0], weight.shape[1], 9), mu).contiguous()


def style_conv_lut(L: Tensor, weight: Tensor, bias: Tensor, mu: Tensor) -> Tensor:
    """conv2d(middle_avg, weight, bias, padding=1) where middle_avg[:, p] = mu[L(p)]: [C,R,R]."""
    t = style_tables(weight, mu)
    return _tap_gather(L, lambda tap: t[:, tap], weight.shape[0]) + bias.view(-1, 1, 1)


# ------------------------------------------------------------------------------------------------ stand-in model
class _Node(torch.nn.Module):
    def __getitem__(self, i):
        return getattr(self, str(i))


def stand_in_model(params, dev):
    """A ``Pix2PixModel`` stand-in for decode_sean: ``.netG`` is a module tree with the reference's attribute names (the
    SPADEGenerator.state_dict keys) holding `params` on `dev`, ``.opt`` HairFast's SEAN options.  Lets the GPU tests and
    tools/bench_sean.py run without the reference tree."""
    root = _Node()
    for key, t in params.items():
        *path, leaf = key.split(".")
        m = root
        for name in path:
            if not hasattr(m, name):
                m.add_module(name, _Node())
            m = getattr(m, name)
            if name == "param_free_norm":
                m.eps = 1e-5
        if leaf in ("weight_u", "weight_v", "running_mean", "running_var", "num_batches_tracked"):
            m.register_buffer(leaf, t.clone())
        else:
            m.register_parameter(leaf, torch.nn.Parameter(t.clone(), requires_grad=False))
    opt = types.SimpleNamespace(ngf=64, label_nc=19, semantic_nc=19, crop_size=256, aspect_ratio=1.0,
                                num_upsampling_layers="normal", norm_G="spectralspadesyncbatch3x3", no_instance=True,
                                contain_dontcare_label=False)
    root.opt = opt
    return types.SimpleNamespace(netG=root.to(dev).eval(), opt=opt)

"""CPU oracle for SEAN's ``encode_sean`` (the Zencoder).  TEST INFRASTRUCTURE ONLY -- same rules as sean_oracle.py
(imported only by tests/, tools/ and the golden script).

``encode_ref`` is a functional fp32 restatement (torch CPU, no nn.Module, no reference imports) of
* ``encode_sean`` -- models/sean_codes/models/pix2pix_model.py:299-306, ``Pix2PixModel.forward(mode='style_code')``
  (:74-77) and the one-hot map of ``preprocess_input`` (:124-149);
* ``Zencoder(3, 512, ngf 32, n_downsampling 2)`` -- models/sean_codes/models/networks/architecture.py:154-207.

``instance_norm_lrelu`` / ``transposed_parity_weight`` / ``conv_transpose_four_parity`` / ``class_means`` state the
forms the CUDA path uses; tests/test_sean_encode_oracle.py checks them in float64 against the plain operations.

Pinned by tests/golden/sean_encode.npz, produced by oracle/gen_golden_sean_encode.py from the unmodified reference
``Pix2PixModel(SEAN_OPT)`` with the seeded parameters of ``sean_oracle.synth_sean_params``.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from oracle.sean_oracle import N_CLASSES, SIZE, label_map, one_hot

Tensor = torch.Tensor
def golden_images(seed: int, batch: int) -> Tensor:
    """The [B,3,256,256] images of one encode golden case, in [-1, 1] (regenerated from the stored seed)."""
    return torch.rand(batch, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def golden_sample_enc(x: Tensor) -> Tensor:
    """The part of a [B,C,R,R] Zencoder activation the golden stores: 16 channels, 16 x 16 pixels per sample."""
    c, r = x.shape[1], x.shape[-1]
    return x[:, ::max(1, c // 16), ::max(1, r // 16), ::max(1, r // 16)]


@torch.no_grad()
def encode_ref(p: Dict[str, Tensor], images: Tensor, labels: Tensor) -> Tuple[Tensor, Dict[str, Tensor]]:
    """encode_sean (pix2pix_model.py:299-306) -> Pix2PixModel.forward(mode='style_code') (:74-77) on the one-hot map of
    preprocess_input (:124-149) -> Zencoder(3, 512, ngf 32, n_downsampling 2).forward (architecture.py:154-207).
    images [B,3,256,256], labels [B,1,256,256] -> ([B,19,512] codes, taps: "in1".."in4" = the four InstanceNorm +
    LeakyReLU outputs, "pre_tanh" = the last convolution's output)."""
    w = lambda i: p[f"Zencoder.model.{i}.weight"]
    b = lambda i: p[f"Zencoder.model.{i}.bias"]
    taps = {}
    act = lambda t: F.leaky_relu(F.instance_norm(t, eps=1e-5), 0.2)       # InstanceNorm2d(affine=False), LeakyReLU(0.2)
    x = F.conv2d(F.pad(images.float(), (1, 1, 1, 1), mode="reflect"), w(1), b(1))          # :159-160
    x = taps["in1"] = act(x)
    x = taps["in2"] = act(F.conv2d(x, w(4), b(4), stride=2, padding=1))                  # :162-166
    x = taps["in3"] = act(F.conv2d(x, w(7), b(7), stride=2, padding=1))
    # :168-173; InstanceNorm2d(64) after a 256-channel output: affine=False, so torch normalises all 256 channels
    x = taps["in4"] = act(F.conv_transpose2d(x, w(10), b(10), stride=2, padding=1, output_padding=1))
    x = taps["pre_tanh"] = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), w(14), b(14))      # :175
    codes = torch.tanh(x)
    seg = F.interpolate(one_hot(labels), size=codes.shape[2:], mode="nearest")          # :181
    out = torch.zeros(codes.shape[0], seg.shape[1], codes.shape[1])
    for i in range(codes.shape[0]):                                                      # :195-205
        for j in range(seg.shape[1]):
            mask = seg.bool()[i, j]
            area = int(mask.sum())
            if area > 0:
                out[i, j] = codes[i].masked_select(mask).reshape(codes.shape[1], area).mean(1)
    return out, taps


def instance_norm_lrelu(x: Tensor, slope: float = 0.2) -> Tensor:
    """The kernels' InstanceNorm: no conv bias in front (a per-channel constant cancels in x - mean), per-(b, c) mean,
    then the biased variance of the centred values, eps 1e-5; then LeakyReLU."""
    m = x.mean((2, 3), keepdim=True)
    v = (x - m).pow(2).mean((2, 3), keepdim=True)
    return F.leaky_relu((x - m) / torch.sqrt(v + 1e-5), slope)


def transposed_parity_weight(w: Tensor) -> Tensor:
    """ConvTranspose2d(3, stride 2, padding 1, output_padding 1) weight [cin, cout, 3, 3] -> the [4*cout, cin, 3, 3]
    correlation weights of the four output parities (a, b) = (y % 2, x % 2), rows n = (o/32)*128 + (2a + b)*32 + o%32
    (cout % 32 == 0).  Output 2m takes kernel row 1 at input m (tap dy = 1); output 2m + 1 takes kernel row 2 at input
    m (dy = 1) and kernel row 0 at input m + 1 (dy = 2); the same for columns."""
    cin, cout = w.shape[:2]
    kmap = {0: {1: 1}, 1: {1: 2, 2: 0}}                  # parity -> {tap d: kernel index}
    out = torch.zeros(4 * cout, cin, 3, 3, dtype=w.dtype)
    o = torch.arange(cout)
    for a in (0, 1):
        for bb in (0, 1):
            rows = (o // 32) * 128 + (2 * a + bb) * 32 + o % 32
            for dy, ky in kmap[a].items():
                for dx, kx in kmap[bb].items():
                    out[rows, :, dy, dx] = w[:, :, ky, kx].t()
    return out


def conv_transpose_four_parity(x: Tensor, w: Tensor) -> Tensor:
    """conv_transpose2d(x, w, stride=2, padding=1, output_padding=1) as one zero-padded 3x3 correlation with the
    four-parity weights, whose output rows are stored at (2y + a, 2x + b) (the pixel shuffle of the epilogue)."""
    cout = w.shape[1]
    y4 = F.conv2d(x, transposed_parity_weight(w), padding=1)
    bsz, _, h, wd = y4.shape
    y4 = y4.view(bsz, cout // 32, 2, 2, 32, h, wd)                       # [b][o/32][a][b'][o%32][y][x]
    return y4.permute(0, 1, 4, 5, 2, 6, 3).reshape(bsz, cout, 2 * h, 2 * wd)


def class_means(codes: Tensor, labels: Tensor) -> Tensor:
    """The kernels' class means: codes [B,C,128,128] (after tanh), labels [B,1,256,256] -> [B,19,C]; class j's mean
    over the pixels of label_map(labels[b], 128) equal to j, exactly 0 where there is none."""
    out = []
    for i in range(codes.shape[0]):
        L = label_map(labels[i: i + 1], codes.shape[-1]).reshape(-1)
        flat = codes[i].reshape(codes.shape[1], -1)
        sums = torch.zeros(N_CLASSES, codes.shape[1], dtype=codes.dtype).index_add_(0, L, flat.t())
        cnt = torch.bincount(L, minlength=N_CLASSES).to(codes.dtype)
        out.append(torch.where(cnt[:, None] > 0, sums / cnt.clamp_min(1)[:, None], torch.zeros_like(sums)))
    return torch.stack(out)

"""PostProcess conv stack of HairFast's Blending stage (SURVEY 8f-1) on the wgmma convolution kernels.

Drop-in counterparts of the reference classes ``PostProcessModel`` builds (models/Encoders.py:106-118):

* ``FeatureEncoder`` / ``FeatureEncoderMult`` -- models/Net.py:334-477: the ArcFace iresnet50 trunk with the content
  branch and the 18 ``nn.Linear(960*9, 512)`` heads; ``fs_layers=[9]`` (the only configuration HairFast uses) taps the
  content branch after ``block_2`` (128 channels, 64x64) with a 3x3 / stride-1 second convolution;
* ``FeatureiResnet`` -- models/Encoders.py:35-57: six stride-1 ``IBasicBlock`` at 64x64 with widths
  1024 -> 1024 -> 768 -> 512 and a conv1x1 + BatchNorm shortcut where the width changes;
* ``IBasicBlock`` / ``conv1x1`` / ``conv3x3`` -- models/Net.py:139-190.

Same constructor arguments, ``forward`` signatures and ``state_dict`` keys as the reference (``load_state_dict(...,
strict=True)`` of a PostProcess checkpoint works).  CUDA tensors only, eval mode only (running BatchNorm statistics):
``Blending`` calls ``PostProcessModel().eval()`` under ``torch.inference_mode`` (models/Blending.py:29,35).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import graphs, nn16
from .encoders import IBasicBlock, _PackCacheMixin, _params_key, fs_encoder_v2

__all__ = ["FeatureEncoder", "FeatureEncoderMult", "FeatureiResnet", "IBasicBlock", "conv1x1", "conv3x3",
           "transform_to_256"]

# content-branch second convolution per F-space layer index (models/Net.py:118-138)
fs_kernals = {0: (12, 12), 1: (12, 12), 2: (6, 6), 3: (6, 6), 4: (3, 3), 5: (3, 3), 6: (3, 3), 7: (3, 3)}
fs_strides = {0: (7, 7), 1: (7, 7), 2: (4, 4), 3: (4, 4), 4: (2, 2), 5: (2, 2), 6: (1, 1), 7: (1, 1)}


def conv3x3(in_planes, out_planes, stride=1, groups=1, dilation=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=dilation, groups=groups, bias=False,
                     dilation=dilation)


def conv1x1(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=1, stride=stride, bias=False)


def transform_to_256(x: torch.Tensor) -> torch.Tensor:
    """``transforms.Resize((256, 256))`` (models/Net.py:12-14).  Uses torchvision when it is installed so the result
    is whatever the reference computes in the same environment (torchvision >= 0.17 antialiases tensors by default,
    the reference's pinned 0.14 does not); otherwise plain bilinear interpolation."""
    if tuple(x.shape[-2:]) == (256, 256):
        return x
    try:
        from torchvision.transforms import functional as TF
    except ImportError:
        return F.interpolate(x, size=(256, 256), mode="bilinear", align_corners=False)
    return TF.resize(x, [256, 256])


class FeatureEncoder(fs_encoder_v2):
    """models/Net.py:334-394 -- structurally the FeatureStyleEncoder trunk (content branch after ``block_3``)."""

    def __init__(self, n_styles=18, opts=None, residual=False, use_coeff=False, resnet_layer=None, video_input=False,
                 f_maps=512, stride=(1, 1)):
        super().__init__(n_styles=n_styles, opts=opts, residual=residual, use_coeff=use_coeff,
                         resnet_layer=resnet_layer, video_input=video_input, f_maps=f_maps, stride=stride)


class FeatureEncoderMult(FeatureEncoder):
    """models/Net.py:396-477.  ``forward(x) -> (latents [B,18,512], [content per fs_layer])``."""

    def __init__(self, fs_layers=(5,), ranks=None, **kwargs):
        super().__init__(**kwargs)
        if ranks is not None:
            raise NotImplementedError("FeatureEncoderMult(ranks=...) (low-rank content heads) is not on the HairFast path")
        self.fs_layers = fs_layers
        self.ranks = ranks
        shift = 0 if max(fs_layers) <= 7 else 2
        scale = 1 if max(fs_layers) <= 7 else 2
        self.content_layer = nn.ModuleList()
        self._content_strides = []
        for layer in fs_layers:
            kern, stride = fs_kernals[layer - shift], fs_strides[layer - shift]
            if kern != (3, 3):
                raise NotImplementedError(f"FeatureEncoderMult: fs_layer {layer} needs a {kern} / stride {stride} "
                                          "content convolution; only the 3x3 cases are implemented")
            self.content_layer.append(nn.Sequential(
                nn.BatchNorm2d(256 // scale, eps=1e-05), nn.Conv2d(256 // scale, 512, 3, 1, 1, bias=False),
                nn.BatchNorm2d(512, eps=1e-05), nn.PReLU(num_parameters=512),
                nn.Conv2d(512, 512, kernel_size=kern, stride=stride, padding=(1, 1), bias=False),
                nn.BatchNorm2d(512, eps=1e-05)))
            self._content_strides.append(stride[0])
        self._content_stage = 2 if max(fs_layers) <= 7 else 1      # after block_3 / after block_2 (Net.py:453-470)
        self._pk = None

    def _content_branches(self):
        return list(self.content_layer)

    @torch.no_grad()
    def forward(self, x):
        return self._graphed_trunk(transform_to_256(x))


class FeatureiResnet(_PackCacheMixin, nn.Module):
    """models/Encoders.py:35-57."""

    def __init__(self, blocks, inplanes=1024):
        super().__init__()
        res_blocks = {}
        for n, (planes, num_blocks) in enumerate(blocks, start=1):
            for k in range(1, num_blocks + 1):
                downsample = None
                if inplanes != planes:
                    downsample = nn.Sequential(conv1x1(inplanes, planes, 1), nn.BatchNorm2d(planes, eps=1e-05))
                res_blocks[f"res_block_{n}_{k}"] = IBasicBlock(inplanes, planes, 1, downsample, 1, 64, 1)
                inplanes = planes
        self.res_blocks = nn.ModuleDict(res_blocks)
        self._pk = None

    def _pack(self):
        key = _params_key(self)
        if self._pk is None or self._pk[0] != key:
            self._pk = (key, [m.packed() for m in self.res_blocks.values()])
        return self._pk[1]

    @torch.no_grad()
    def forward(self, x):
        if self.training:
            raise RuntimeError("FeatureiResnet: only eval-mode (running BatchNorm statistics) forward is implemented")
        if not x.is_cuda:
            raise RuntimeError("FeatureiResnet: input must be a CUDA tensor (no CPU fallback)")
        return graphs.run(self, "res", _params_key(self), self._forward_impl, x)

    def _forward_impl(self, x):
        blocks = self._pack()
        # x is fp32 NCHW (torch.cat of the two content maps); the first block's BatchNorm rides on the layout change
        raw = nn16.to_nhwc16(x)
        bn = nn16.to_nhwc16(x, scale=blocks[0].pre[0], shift=blocks[0].pre[1])
        for i, blk in enumerate(blocks):
            nxt = blocks[i + 1].pre if i + 1 < len(blocks) else None
            raw, bn = blk(raw, bn, nxt, want_raw=True)
        return nn16.to_nchw32(raw)

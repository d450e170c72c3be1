"""e4e and FeatureStyleEncoder inversion encoders on the H100 convolution kernels (SURVEY 8 rows a13 / a14).

Drop-in module surface (same class names, constructor arguments and ``state_dict`` keys, so the reference
checkpoints load unchanged):

* ``Encoder4Editing`` + ``GradualStyleBlock`` / ``bottleneck_IR`` / ``bottleneck_IR_SE`` / ``SEModule``
  -- models/encoder4editing/models/encoders/psp_encoders.py:34-55,124-200 and helpers.py:57-140;
* ``fs_encoder_v2`` + ``IBasicBlock`` / ``iresnet50`` trunk
  -- models/FeatureStyleEncoder/nets/feature_style_encoder.py:12-65 and arcface/iresnet.py:28-163.

The nn.Modules below only own parameters; ``forward`` runs NHWC 16-bit activations through
``hf_conv2d_forward`` (wgmma implicit GEMM; eval-mode BatchNorm folded into weights / epilogue, PReLU /
LeakyReLU / residual add fused) plus a few HBM-bound glue kernels (``nn16``: SE pooling + gate, SE combine,
FPN upsample-add, adaptive pooling).  The small dense style heads (EqualLinear / nn.Linear) are plain cuBLAS GEMMs
through torch.
Eval mode only (running statistics); CUDA only, no fallback.
"""
from __future__ import annotations

import math
from collections import namedtuple

import torch
from torch import nn

from . import graphs, nn16
from .model import EqualLinear


def _params_key(module: nn.Module):
    """Version key of every parameter / buffer (repack when a weight changes).  Walking the module tree costs
    milliseconds for a 600-tensor encoder -- as much as its kernels at swap()'s batch sizes -- so the tensor LIST is
    cached on the module; `nn.Module._apply` (.to / .cuda / .float: the calls that replace buffer objects) drops it
    (`_PackCacheMixin`), `load_state_dict` copies in place and shows up in `_version`."""
    ts = module.__dict__.get("_hf_tensors")
    if ts is None:
        ts = list(module.parameters()) + list(module.buffers())
        module.__dict__["_hf_tensors"] = ts
    return tuple([(t.data_ptr(), t._version) for t in ts])


class _PackCacheMixin:
    """Invalidate the cached tensor list (and with it the packed operands / captured graphs) on device / dtype moves."""

    def _apply(self, fn, *args, **kwargs):
        self.__dict__.pop("_hf_tensors", None)
        self.__dict__.pop("_hf_graphs", None)
        return super()._apply(fn, *args, **kwargs)


# ------------------------------------------------------------------------------------------------
# shared pre-activation residual block:  BN -> conv3x3 -> [BN] -> PReLU -> conv3x3(stride) -> BN [-> SE] + shortcut
# ------------------------------------------------------------------------------------------------
class _PackedIRBlock:
    """Packed form of one bottleneck_IR(_SE) / IBasicBlock."""

    def __init__(self, bn_in, conv1, bn_mid, prelu, conv2, bn_out, se, shortcut_conv, shortcut_bn, stride):
        self.stride = stride
        self.pre = nn16.bn_affine(bn_in)                       # applied by the PRODUCER of this block's input
        mid_scale, mid_shift = nn16.bn_affine(bn_mid) if bn_mid is not None else (None, None)
        self.conv1 = nn16.PackedConv2d(conv1.weight, mid_scale)
        self.mid_shift = mid_shift
        self.slope = prelu.weight.detach().float().contiguous()
        out_scale, self.out_shift = nn16.bn_affine(bn_out)
        self.conv2 = nn16.PackedConv2d(conv2.weight, out_scale, stride=stride)
        self.se = se
        self.sc = None
        if shortcut_conv is not None:
            sc_scale, self.sc_shift = nn16.bn_affine(shortcut_bn)
            self.sc = nn16.PackedConv2d(shortcut_conv.weight, sc_scale, stride=stride)

    def __call__(self, x_raw16, x_bn16, next_affine, want_raw=True):
        """x_raw16 = block input, x_bn16 = bn_in(input).  Returns (out16 | None, next_bn(out)16 | None)."""
        h, _, _ = self.conv1(x_bn16, shift=self.mid_shift, act=1, slope=self.slope)
        shortcut = x_raw16
        sc_stride = self.stride
        if self.sc is not None:
            shortcut, _, _ = self.sc(x_raw16, shift=self.sc_shift)
            sc_stride = 1
        if self.se is None and sc_stride == 1:
            # fully fused: residual add + next block's BatchNorm in the conv epilogue
            out, out_bn, _ = self.conv2(h, shift=self.out_shift, residual16=shortcut, want_y16=want_raw,
                                        y16b_affine=next_affine)
            return out, out_bn
        res, _, _ = self.conv2(h, shift=self.out_shift)
        se = None
        if self.se is not None:                                 # SEModule (helpers.py:57-75)
            se = nn16.se_gate(res, self.se.fc1.weight, self.se.fc2.weight)
        return nn16.scale_add(res, se, shortcut, sc_stride, next_affine, want_y16=want_raw)


# ------------------------------------------------------------------------------------------------
# e4e
# ------------------------------------------------------------------------------------------------
class Bottleneck(namedtuple("Block", ["in_channel", "depth", "stride"])):
    """A named tuple describing a ResNet block."""


def get_block(in_channel, depth, num_units, stride=2):
    return [Bottleneck(in_channel, depth, stride)] + [Bottleneck(depth, depth, 1) for _ in range(num_units - 1)]


def get_blocks(num_layers):
    units = {50: [3, 4, 14, 3], 100: [3, 13, 30, 3], 152: [3, 8, 36, 3]}
    if num_layers not in units:
        raise ValueError("Invalid number of layers: {}. Must be one of [50, 100, 152]".format(num_layers))
    u = units[num_layers]
    return [get_block(64, 64, u[0]), get_block(64, 128, u[1]), get_block(128, 256, u[2]), get_block(256, 512, u[3])]


class SEModule(nn.Module):
    def __init__(self, channels, reduction):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc1 = nn.Conv2d(channels, channels // reduction, kernel_size=1, padding=0, bias=False)
        self.relu = nn.ReLU(inplace=True)
        self.fc2 = nn.Conv2d(channels // reduction, channels, kernel_size=1, padding=0, bias=False)
        self.sigmoid = nn.Sigmoid()


class bottleneck_IR(nn.Module):
    _with_se = False

    def __init__(self, in_channel, depth, stride):
        super().__init__()
        self.stride = stride
        if in_channel == depth:
            self.shortcut_layer = nn.MaxPool2d(1, stride)
        else:
            self.shortcut_layer = nn.Sequential(nn.Conv2d(in_channel, depth, (1, 1), stride, bias=False),
                                                nn.BatchNorm2d(depth))
        layers = [nn.BatchNorm2d(in_channel), nn.Conv2d(in_channel, depth, (3, 3), (1, 1), 1, bias=False),
                  nn.PReLU(depth), nn.Conv2d(depth, depth, (3, 3), stride, 1, bias=False), nn.BatchNorm2d(depth)]
        if self._with_se:
            layers.append(SEModule(depth, 16))
        self.res_layer = nn.Sequential(*layers)

    def packed(self):
        r = self.res_layer
        sc = self.shortcut_layer if isinstance(self.shortcut_layer, nn.Sequential) else None
        return _PackedIRBlock(r[0], r[1], None, r[2], r[3], r[4], r[5] if self._with_se else None,
                              sc[0] if sc is not None else None, sc[1] if sc is not None else None, self.stride)


class bottleneck_IR_SE(bottleneck_IR):
    _with_se = True


class GradualStyleBlock(nn.Module):
    def __init__(self, in_c, out_c, spatial):
        super().__init__()
        self.out_c = out_c
        self.spatial = spatial
        num_pools = int(math.log2(spatial))
        modules = [nn.Conv2d(in_c, out_c, kernel_size=3, stride=2, padding=1), nn.LeakyReLU()]
        for _ in range(num_pools - 1):
            modules += [nn.Conv2d(out_c, out_c, kernel_size=3, stride=2, padding=1), nn.LeakyReLU()]
        self.convs = nn.Sequential(*modules)
        self.linear = EqualLinear(out_c, out_c, lr_mul=1)


class _PackedHeads:
    """All GradualStyleBlocks that read the same feature map, run together: the first conv as ONE wide
    conv (shared input, N = heads*512), the following ones as grouped convs (groups = heads)."""

    def __init__(self, heads):
        self.n = len(heads)
        convs = [[m for m in h.convs if isinstance(m, nn.Conv2d)] for h in heads]
        depth = len(convs[0])
        self.first = nn16.PackedConv2d(torch.cat([c[0].weight for c in convs], 0), stride=2)
        self.first_bias = torch.cat([c[0].bias for c in convs], 0).detach().float()
        self.rest, self.rest_bias = [], []
        for d in range(1, depth):
            self.rest.append(nn16.PackedConv2d(torch.cat([c[d].weight for c in convs], 0), stride=2, groups=self.n))
            self.rest_bias.append(torch.cat([c[d].bias for c in convs], 0).detach().float())
        # EqualLinear of every head (psp_encoders.py:47,52-53) = one grouped 1x1 convolution on the [B,1,1,n*512] map
        lin_w = torch.cat([h.linear.weight.detach().float() * h.linear.scale for h in heads], 0)          # [n*512,512]
        self.lin = nn16.PackedConv2d(lin_w.reshape(lin_w.shape[0], lin_w.shape[1], 1, 1), groups=self.n)
        self.lin_b = torch.cat([h.linear.bias.detach().float() * h.linear.lr_mul for h in heads], 0).contiguous()

    def __call__(self, feat16):
        x, _, _ = self.first(feat16, shift=self.first_bias, act=2, slope0=0.01)
        for conv, bias in zip(self.rest, self.rest_bias):
            x, _, _ = conv(x, shift=bias, act=2, slope0=0.01)
        b = x.shape[0]
        if x.shape[1] != 1 or x.shape[2] != 1:
            raise RuntimeError(f"GradualStyleBlock: expected a 1x1 map before the linear layer, got {list(x.shape)}")
        _, _, y = self.lin(x, shift=self.lin_b, want_y16=False, want_y32=True)  # [B, heads*512, 1, 1] fp32
        return y.reshape(b, self.n, -1)                                         # EqualLinear per head


class Encoder4Editing(_PackCacheMixin, nn.Module):
    def __init__(self, num_layers, mode="ir", opts=None):
        super().__init__()
        assert num_layers in [50, 100, 152], "num_layers should be 50,100, or 152"
        assert mode in ["ir", "ir_se"], "mode should be ir or ir_se"
        unit_module = bottleneck_IR if mode == "ir" else bottleneck_IR_SE
        self.input_layer = nn.Sequential(nn.Conv2d(3, 64, (3, 3), 1, 1, bias=False), nn.BatchNorm2d(64), nn.PReLU(64))
        self.body = nn.Sequential(*[unit_module(b.in_channel, b.depth, b.stride)
                                    for block in get_blocks(num_layers) for b in block])
        self.styles = nn.ModuleList()
        log_size = int(math.log(opts.stylegan_size, 2))
        self.style_count = 2 * log_size - 2
        self.coarse_ind = 3
        self.middle_ind = 7
        for i in range(self.style_count):
            spatial = 16 if i < self.coarse_ind else (32 if i < self.middle_ind else 64)
            self.styles.append(GradualStyleBlock(512, 512, spatial))
        self.latlayer1 = nn.Conv2d(256, 512, kernel_size=1, stride=1, padding=0)
        self.latlayer2 = nn.Conv2d(128, 512, kernel_size=1, stride=1, padding=0)
        self._pk = None

    def get_deltas_starting_dimensions(self):
        return list(range(self.style_count))

    def _pack(self):
        key = _params_key(self)
        if self._pk is not None and self._pk["key"] == key:
            return self._pk
        il = self.input_layer
        pk = {"key": key,
              "stem": nn16.PackedStem3x3(il[0].weight, il[1], il[2].weight),      # conv + BN + PReLU, one fused kernel
              "blocks": [m.packed() for m in self.body],
              "lat1": nn16.PackedConv2d(self.latlayer1.weight), "lat2": nn16.PackedConv2d(self.latlayer2.weight),
              "heads": [_PackedHeads(list(self.styles[:self.coarse_ind])),
                        _PackedHeads(list(self.styles[self.coarse_ind:self.middle_ind])),
                        _PackedHeads(list(self.styles[self.middle_ind:]))]}
        self._pk = pk
        return pk

    @torch.no_grad()
    def forward(self, x):
        if self.training:
            raise RuntimeError("Encoder4Editing: only eval-mode (running BatchNorm statistics) forward is implemented")
        if not x.is_cuda:
            raise RuntimeError("Encoder4Editing: input must be a CUDA tensor (no CPU fallback)")
        return graphs.run(self, "e4e", _params_key(self), self._forward_impl, x)

    def _forward_impl(self, x):
        pk = self._pack()
        blocks = pk["blocks"]
        raw, bn = pk["stem"](x, y16b_affine=blocks[0].pre)
        taps = {}
        for i, blk in enumerate(blocks):
            nxt = blocks[i + 1].pre if i + 1 < len(blocks) else None
            raw, bn = blk(raw, bn, nxt, want_raw=True)
            if i in (6, 20, 23):
                taps[i] = raw
        c1, c2, c3 = taps[6], taps[20], taps[23]
        w_coarse = pk["heads"][0](c3)                                  # [B,3,512]; head 0 is the base code
        l1, _, _ = pk["lat1"](c2, shift=self.latlayer1.bias)
        p2 = nn16.upsample_add(c3, l1)
        w_mid = pk["heads"][1](p2)
        l2, _, _ = pk["lat2"](c1, shift=self.latlayer2.bias)
        p1 = nn16.upsample_add(p2, l2)
        w_fine = pk["heads"][2](p1)
        deltas = torch.cat([w_coarse, w_mid, w_fine], 1)               # [B,18,512]
        w = deltas[:, :1].repeat(1, self.style_count, 1)               # w0 duplicated ...
        w[:, 1:] += deltas[:, 1:]                                      # ... plus the per-style deltas (psp_encoders.py:186-200)
        return w


class GradualStyleEncoder(nn.Module):
    def __init__(self, *a, **k):
        raise NotImplementedError("GradualStyleEncoder (pSp) is not on the HairFast path (e4e checkpoints use "
                                  "encoder_type='Encoder4Editing', utils/model_utils.py:17-28)")


class BackboneEncoderUsingLastLayerIntoW(nn.Module):
    def __init__(self, *a, **k):
        raise NotImplementedError("BackboneEncoderUsingLastLayerIntoW is not on the HairFast path")


# ------------------------------------------------------------------------------------------------
# FeatureStyleEncoder
# ------------------------------------------------------------------------------------------------
class IBasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1):
        super().__init__()
        self.bn1 = nn.BatchNorm2d(inplanes, eps=1e-05)
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes, eps=1e-05)
        self.prelu = nn.PReLU(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes, eps=1e-05)
        self.downsample = downsample
        self.stride = stride

    def packed(self):
        ds = self.downsample
        return _PackedIRBlock(self.bn1, self.conv1, self.bn2, self.prelu, self.conv2, self.bn3, None,
                              ds[0] if ds is not None else None, ds[1] if ds is not None else None, self.stride)


def _iresnet_layer(inplanes, planes, blocks, stride=2):
    downsample = nn.Sequential(nn.Conv2d(inplanes, planes, kernel_size=1, stride=stride, bias=False),
                               nn.BatchNorm2d(planes, eps=1e-05))
    layers = [IBasicBlock(inplanes, planes, stride, downsample)]
    layers += [IBasicBlock(planes, planes) for _ in range(1, blocks)]
    return nn.Sequential(*layers)


def _load_arcface_trunk(module, path):
    """The reference does ``iresnet50().load_state_dict(torch.load(path))`` STRICTLY and then takes the trunk children
    (nets/feature_style_encoder.py:16-17,27-33; models/Net.py:340-341).  Here the trunk lives under the encoder's own
    names, so the keys are remapped -- and every trunk tensor of the module must be covered, every trunk key of the file
    must be consumed (a renamed or missing key would otherwise leave random weights silently).  The iresnet head
    (bn2 / fc / features), which the reference also loads and then drops, is the only part allowed to be unused."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    remap = {"conv1": "conv.0", "bn1": "conv.1", "prelu": "conv.2", "layer1": "block_1", "layer2": "block_2",
             "layer3": "block_3", "layer4": "block_4"}
    dropped_heads = ("bn2", "fc", "features", "dropout")
    mine, unexpected = {}, []
    for k, v in sd.items():
        head = k.split(".")[0]
        if head in remap:
            mine[remap[head] + k[len(head):]] = v
        elif head not in dropped_heads:
            unexpected.append(k)
    trunk = tuple(remap.values())
    own = [k for k in module.state_dict() if k.startswith(tuple(t + "." for t in trunk))]
    missing = [k for k in own if k not in mine]
    extra = [k for k in mine if k not in own]
    if missing or extra or unexpected:
        raise RuntimeError(f"ArcFace checkpoint {path} does not match the iresnet50 trunk: missing {missing[:5]}, "
                           f"unexpected {(extra + unexpected)[:5]}")
    module.load_state_dict(mine, strict=False)


class fs_encoder_v2(_PackCacheMixin, nn.Module):
    def __init__(self, n_styles=18, opts=None, residual=False, use_coeff=False, resnet_layer=None, video_input=False,
                 f_maps=512, stride=(1, 1)):
        super().__init__()
        if video_input:
            raise NotImplementedError("fs_encoder_v2(video_input=True) is not on the HairFast path")
        # iresnet50 trunk: children()[:3] = conv1, bn1, prelu; layers [3, 4, 14, 3] (arcface/iresnet.py:140-163)
        self.conv = nn.Sequential(nn.Conv2d(3, 64, kernel_size=3, stride=1, padding=1, bias=False),
                                  nn.BatchNorm2d(64, eps=1e-05), nn.PReLU(64))
        self.block_1 = _iresnet_layer(64, 64, 3)
        self.block_2 = _iresnet_layer(64, 128, 4)
        self.block_3 = _iresnet_layer(128, 256, 14)
        self.block_4 = _iresnet_layer(256, 512, 3)
        if opts is not None and getattr(opts, "arcface_model_path", None):
            _load_arcface_trunk(self, opts.arcface_model_path)
        s = stride[0] if isinstance(stride, (tuple, list)) else stride
        self.content_layer = nn.Sequential(
            nn.BatchNorm2d(256, eps=1e-05), nn.Conv2d(256, 512, kernel_size=3, stride=1, padding=1, bias=False),
            nn.BatchNorm2d(512, eps=1e-05), nn.PReLU(num_parameters=512),
            nn.Conv2d(512, 512, kernel_size=3, stride=s, padding=1, bias=False), nn.BatchNorm2d(512, eps=1e-05))
        self._content_stage = 2                    # the content branch taps the block_3 output
        self._content_strides = [s]
        self.avg_pool = nn.AdaptiveAvgPool2d((3, 3))
        self.styles = nn.ModuleList([nn.Linear(960 * 9, 512) for _ in range(n_styles)])
        self._pk = None

    def _content_branches(self):
        """[(BN, conv3x3, BN, PReLU, conv3x3(stride), BN)] -- one per content output."""
        return [self.content_layer]

    def _pack(self):
        key = _params_key(self)
        if self._pk is not None and self._pk["key"] == key:
            return self._pk
        branches = []
        for cl, stride in zip(self._content_branches(), self._content_strides):
            c_mid_scale, c_mid_shift = nn16.bn_affine(cl[2])
            c_out_scale, c_out_shift = nn16.bn_affine(cl[5])
            branches.append({"pre": nn16.bn_affine(cl[0]),
                             "conv1": nn16.PackedConv2d(cl[1].weight, c_mid_scale), "shift1": c_mid_shift,
                             "slope": cl[3].weight.detach().float().contiguous(),
                             "conv2": nn16.PackedConv2d(cl[4].weight, c_out_scale, stride=stride),
                             "shift2": c_out_shift})
        pk = {"key": key, "stem": nn16.PackedStem3x3(self.conv[0].weight, self.conv[1], self.conv[2].weight),
              "stages": [[b.packed() for b in blk] for blk in (self.block_1, self.block_2, self.block_3, self.block_4)],
              "content": branches,
              # the n_styles nn.Linear(960*9, 512) heads (feature_style_encoder.py:44-45,62-64) stacked: ONE 1x1
              # convolution [B,1,1,8640] -> [B, n_styles*512]
              "style": nn16.PackedConv2d(torch.cat([s.weight.detach().float() for s in self.styles], 0)[:, :, None, None]),
              "style_b": torch.cat([s.bias.detach().float() for s in self.styles], 0).contiguous(),
              "n_styles": len(self.styles)}
        self._pk = pk
        return pk

    def _trunk(self, x):
        """conv stem -> block_1..4 with the pooled features and the content branches: (latents, [content...])."""
        name = type(self).__name__
        if self.training:
            raise RuntimeError(f"{name}: only eval-mode (running BatchNorm statistics) forward is implemented")
        if not x.is_cuda:
            raise RuntimeError(f"{name}: input must be a CUDA tensor (no CPU fallback)")
        pk = self._pack()
        blocks = [b for st in pk["stages"] for b in st]
        ends, n = [], 0
        for st in pk["stages"]:
            n += len(st)
            ends.append(n - 1)
        raw, bn = pk["stem"](x, y16b_affine=blocks[0].pre)
        feats, content = [], []
        for i, blk in enumerate(blocks):
            nxt = blocks[i + 1].pre if i + 1 < len(blocks) else None
            raw, bn = blk(raw, bn, nxt, want_raw=True)
            if i in ends:
                feats.append(nn16.adaptive_avgpool(raw, 3, 3))
                if i == ends[self._content_stage]:
                    for br in pk["content"]:
                        _, cb = nn16.scale_add(raw, y16b_affine=br["pre"], want_y16=False)      # leading BatchNorm
                        h, _, _ = br["conv1"](cb, shift=br["shift1"], act=1, slope=br["slope"])
                        _, _, c = br["conv2"](h, shift=br["shift2"], want_y16=False, want_y32=True)
                        content.append(c)
        b = x.shape[0]
        f = torch.cat(feats, dim=1).reshape(b, 1, 1, -1).to(nn16.torch_dtype())           # [B,1,1,960*9], x.view(B,-1) order
        _, _, out = pk["style"](f, shift=pk["style_b"], want_y16=False, want_y32=True)     # 18 x nn.Linear(8640,512)
        out = out.reshape(b, pk["n_styles"], -1)
        return out, content

    @torch.no_grad()
    def forward(self, x):
        out, content = self._graphed_trunk(x)
        return out, content[0]

    def _graphed_trunk(self, x):
        """`_trunk` through the CUDA-graph cache (graphs.py); the eval / device checks run before any capture."""
        name = type(self).__name__
        if self.training:
            raise RuntimeError(f"{name}: only eval-mode (running BatchNorm statistics) forward is implemented")
        if not x.is_cuda:
            raise RuntimeError(f"{name}: input must be a CUDA tensor (no CPU fallback)")
        return graphs.run(self, "trunk", _params_key(self), self._trunk, x)

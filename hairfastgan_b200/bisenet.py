"""BiSeNet face parsing (SURVEY 8f-3) on the wgmma convolution kernels.

Drop-in counterpart of ``models/CtrlHair/external_code/face_parsing/model.py`` + ``resnet.py`` (the network
``FaceParsing`` builds, my_parsing_util.py:42,77, and ``get_segmentation`` runs five times per swap, models/Net.py:108-115):
same class names, constructor arguments and ``state_dict`` keys, so ``load_state_dict(torch.load(seg.pth))`` works
unchanged.  ``BiSeNet.forward(x) -> (feat_out, feat_out16, feat_out32)``, each ``[B, n_classes, H, W]`` fp32, like the
reference (model.py:227-244).  CUDA tensors only, eval mode only (FaceParsing calls ``.eval()``).

Differences by design: the ResNet-18 backbone is NOT downloaded at construction (resnet.py:71-77 fetches torchvision
weights that the BiSeNet checkpoint overwrites anyway); only ``BiSeNet.forward`` computes -- the sub-modules are
parameter containers.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import graphs, nn16
from .encoders import _PackCacheMixin, _params_key

__all__ = ["BiSeNet", "ConvBNReLU", "BiSeNetOutput", "AttentionRefinementModule", "ContextPath", "FeatureFusionModule",
           "Resnet18", "BasicBlock"]


def _container_forward(self, *a, **k):
    raise RuntimeError(f"{type(self).__name__} is a parameter container here; run BiSeNet.forward")


class ConvBNReLU(nn.Module):
    """model.py:11-30."""
    forward = _container_forward

    def __init__(self, in_chan, out_chan, ks=3, stride=1, padding=1, *args, **kwargs):
        super().__init__()
        self.conv = nn.Conv2d(in_chan, out_chan, kernel_size=ks, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(out_chan)
        nn.init.kaiming_normal_(self.conv.weight, a=1)

    def packed(self):
        scale, shift = nn16.bn_affine(self.bn)
        return nn16.PackedConv2d(self.conv.weight, scale, stride=self.conv.stride[0]), shift


class BiSeNetOutput(nn.Module):
    """model.py:33-48."""
    forward = _container_forward

    def __init__(self, in_chan, mid_chan, n_classes, *args, **kwargs):
        super().__init__()
        self.conv = ConvBNReLU(in_chan, mid_chan, ks=3, stride=1, padding=1)
        self.conv_out = nn.Conv2d(mid_chan, n_classes, kernel_size=1, bias=False)
        nn.init.kaiming_normal_(self.conv_out.weight, a=1)


class AttentionRefinementModule(nn.Module):
    """model.py:70-95."""
    forward = _container_forward

    def __init__(self, in_chan, out_chan, *args, **kwargs):
        super().__init__()
        self.conv = ConvBNReLU(in_chan, out_chan, ks=3, stride=1, padding=1)
        self.conv_atten = nn.Conv2d(out_chan, out_chan, kernel_size=1, bias=False)
        self.bn_atten = nn.BatchNorm2d(out_chan)
        self.sigmoid_atten = nn.Sigmoid()
        nn.init.kaiming_normal_(self.conv_atten.weight, a=1)


class BasicBlock(nn.Module):
    """resnet.py:20-47."""
    forward = _container_forward

    def __init__(self, in_chan, out_chan, stride=1):
        super().__init__()
        self.conv1 = nn.Conv2d(in_chan, out_chan, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(out_chan)
        self.conv2 = nn.Conv2d(out_chan, out_chan, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(out_chan)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = None
        if in_chan != out_chan or stride != 1:
            self.downsample = nn.Sequential(nn.Conv2d(in_chan, out_chan, kernel_size=1, stride=stride, bias=False),
                                            nn.BatchNorm2d(out_chan))
        self.stride = stride


def create_layer_basic(in_chan, out_chan, bnum, stride=1):
    return nn.Sequential(BasicBlock(in_chan, out_chan, stride=stride),
                         *[BasicBlock(out_chan, out_chan, stride=1) for _ in range(bnum - 1)])


class Resnet18(nn.Module):
    """resnet.py:57-84 (without the torchvision weight download of ``init_weight``)."""
    forward = _container_forward

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = create_layer_basic(64, 64, bnum=2, stride=1)
        self.layer2 = create_layer_basic(64, 128, bnum=2, stride=2)
        self.layer3 = create_layer_basic(128, 256, bnum=2, stride=2)
        self.layer4 = create_layer_basic(256, 512, bnum=2, stride=2)


class ContextPath(nn.Module):
    """model.py:98-132."""
    forward = _container_forward

    def __init__(self, *args, **kwargs):
        super().__init__()
        self.resnet = Resnet18()
        self.arm16 = AttentionRefinementModule(256, 128)
        self.arm32 = AttentionRefinementModule(512, 128)
        self.conv_head32 = ConvBNReLU(128, 128, ks=3, stride=1, padding=1)
        self.conv_head16 = ConvBNReLU(128, 128, ks=3, stride=1, padding=1)
        self.conv_avg = ConvBNReLU(512, 128, ks=1, stride=1, padding=0)


class FeatureFusionModule(nn.Module):
    """model.py:178-224."""
    forward = _container_forward

    def __init__(self, in_chan, out_chan, *args, **kwargs):
        super().__init__()
        self.convblk = ConvBNReLU(in_chan, out_chan, ks=1, stride=1, padding=0)
        self.conv1 = nn.Conv2d(out_chan, out_chan // 4, kernel_size=1, stride=1, padding=0, bias=False)
        self.conv2 = nn.Conv2d(out_chan // 4, out_chan, kernel_size=1, stride=1, padding=0, bias=False)
        self.relu = nn.ReLU(inplace=True)
        self.sigmoid = nn.Sigmoid()
        nn.init.kaiming_normal_(self.conv1.weight, a=1)
        nn.init.kaiming_normal_(self.conv2.weight, a=1)


class _PackedBlock:
    def __init__(self, blk: BasicBlock):
        s1, self.shift1 = nn16.bn_affine(blk.bn1)
        s2, self.shift2 = nn16.bn_affine(blk.bn2)
        self.conv1 = nn16.PackedConv2d(blk.conv1.weight, s1, stride=blk.stride)
        self.conv2 = nn16.PackedConv2d(blk.conv2.weight, s2)
        self.ds = None
        if blk.downsample is not None:
            sd, self.shift_ds = nn16.bn_affine(blk.downsample[1])
            self.ds = nn16.PackedConv2d(blk.downsample[0].weight, sd, stride=blk.stride)

    def __call__(self, x16):
        r, _, _ = self.conv1(x16, shift=self.shift1, act=3)
        sc = x16
        if self.ds is not None:
            sc, _, _ = self.ds(x16, shift=self.shift_ds)
        out, _, _ = self.conv2(r, shift=self.shift2, act=3, residual16=sc, act_after_residual=True)   # relu(shortcut + residual)
        return out


class _PackedOutput:
    def __init__(self, head: BiSeNetOutput):
        self.conv, self.shift = head.conv.packed()
        w = head.conv_out.weight.detach().float()
        self.n_classes = w.shape[0]
        if self.n_classes > 32:
            raise NotImplementedError("BiSeNetOutput: more than 32 classes")
        wp = torch.zeros(32, w.shape[1], 1, 1, device=w.device)            # the GEMM N tile is 32 wide
        wp[:self.n_classes] = w
        self.conv_out = nn16.PackedConv2d(wp)

    def lowres(self, x16):
        h, _, _ = self.conv(x16, shift=self.shift, act=3)
        _, _, low = self.conv_out(h, want_y16=False, want_y32=True)         # [B,32,h,w] fp32, classes first
        return low

    def __call__(self, x16, height, width):
        low = self.lowres(x16)
        return nn16.bilinear_upsample_nchw(low, self.n_classes, height, width), low


class BiSeNet(_PackCacheMixin, nn.Module):
    """model.py:217-244."""

    def __init__(self, n_classes, *args, **kwargs):
        super().__init__()
        self.cp = ContextPath()
        self.ffm = FeatureFusionModule(256, 256)
        self.conv_out = BiSeNetOutput(256, 256, n_classes)
        self.conv_out16 = BiSeNetOutput(128, 64, n_classes)
        self.conv_out32 = BiSeNetOutput(128, 64, n_classes)
        self._pk = None

    def _pack(self):
        key = _params_key(self)
        if self._pk is not None and self._pk["key"] == key:
            return self._pk
        cp, rn = self.cp, self.cp.resnet

        def arm(m):
            conv, shift = m.conv.packed()
            a_scale, a_shift = nn16.bn_affine(m.bn_atten)
            return {"conv": conv, "shift": shift, "w": m.conv_atten.weight, "a_scale": a_scale, "a_shift": a_shift}

        avg_scale, avg_shift = nn16.bn_affine(cp.conv_avg.bn)
        pk = {"key": key, "stem": nn16.PackedStem7x7(rn.conv1.weight, rn.bn1),
              "blocks": [[_PackedBlock(b) for b in layer] for layer in (rn.layer1, rn.layer2, rn.layer3, rn.layer4)],
              "arm16": arm(cp.arm16), "arm32": arm(cp.arm32),
              "head32": cp.conv_head32.packed(), "head16": cp.conv_head16.packed(),
              "avg": (cp.conv_avg.conv.weight, avg_scale, avg_shift),
              "ffm": self.ffm.convblk.packed(),
              "out": _PackedOutput(self.conv_out), "out16": _PackedOutput(self.conv_out16),
              "out32": _PackedOutput(self.conv_out32)}
        self._pk = pk
        return pk

    def _trunk(self, x):
        """Everything up to the three head inputs (fuse, feat16_up, feat32_up) -- model.py:226-234."""
        if self.training:
            raise RuntimeError("BiSeNet: only eval-mode (running BatchNorm statistics) forward is implemented")
        if not x.is_cuda:
            raise RuntimeError("BiSeNet: input must be a CUDA tensor (no CPU fallback)")
        if x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError(f"BiSeNet: expected [B,3,H,W], got {list(x.shape)}")
        H, W = x.shape[2:]
        if H % 32 or W % 32:
            raise NotImplementedError(f"BiSeNet: input size {H}x{W} must be a multiple of 32")
        pk = self._pack()
        # ---- Resnet18 (resnet.py:68-79)
        f = nn16.maxpool3x3s2(pk["stem"](x))
        feats = []
        for li, layer in enumerate(pk["blocks"]):
            for blk in layer:
                f = blk(f)
            if li >= 1:
                feats.append(f)
        feat8, feat16, feat32 = feats
        # ---- ContextPath (model.py:108-132)
        w_avg, s_avg, b_avg = pk["avg"]
        avg = nn16.pooled_fc(feat32, w_avg, s_avg, b_avg, act=1)                                   # conv_avg on the pooled map
        a32 = pk["arm32"]
        c32, _, _ = a32["conv"](feat32, shift=a32["shift"], act=3)
        g32 = nn16.pooled_fc(c32, a32["w"], a32["a_scale"], a32["a_shift"], act=2)
        up32 = nn16.gate_add_up(c32, gate=g32, addvec=avg, up=2)                                   # (feat*atten + avg) nearest x2
        feat32_up, _, _ = pk["head32"][0](up32, shift=pk["head32"][1], act=3)
        a16 = pk["arm16"]
        c16, _, _ = a16["conv"](feat16, shift=a16["shift"], act=3)
        g16 = nn16.pooled_fc(c16, a16["w"], a16["a_scale"], a16["a_shift"], act=2)
        up16 = nn16.gate_add_up(c16, gate=g16, addt16=feat32_up, up=2)
        feat16_up, _, _ = pk["head16"][0](up16, shift=pk["head16"][1], act=3)
        # ---- FeatureFusionModule (model.py:200-211); feat_sp = the res3b1 feature (model.py:232)
        fcat = torch.cat([feat8, feat16_up], dim=-1)
        feat, _, _ = pk["ffm"][0](fcat, shift=pk["ffm"][1], act=3)
        atten = nn16.se_gate(feat, self.ffm.conv1.weight, self.ffm.conv2.weight)
        fuse, _ = nn16.scale_add(feat, atten, feat)                                                 # feat*atten + feat
        return pk, fuse, feat16_up, feat32_up, H, W

    def _check(self, x):
        if self.training:
            raise RuntimeError("BiSeNet: only eval-mode (running BatchNorm statistics) forward is implemented")
        if not torch.is_tensor(x) or not x.is_cuda:
            raise RuntimeError("BiSeNet: input must be a CUDA tensor (no CPU fallback)")

    @torch.no_grad()
    def forward(self, x, return_lowres: bool = False):
        self._check(x)
        if return_lowres:
            return self._forward_impl(x, True)
        return graphs.run(self, "fwd", _params_key(self), self._forward_impl, x)

    def _forward_impl(self, x, return_lowres: bool = False):
        pk, fuse, feat16_up, feat32_up, H, W = self._trunk(x)
        # ---- heads + bilinear upsampling (model.py:235-241)
        o, lo = pk["out"](fuse, H, W)
        o16, lo16 = pk["out16"](feat16_up, H, W)
        o32, lo32 = pk["out32"](feat32_up, H, W)
        if return_lowres:
            return [t[:, :pk["out"].n_classes] for t in (lo, lo16, lo32)]
        return o, o16, o32

    @torch.no_grad()
    def parse_labels(self, x):
        """``self(x)[0].argmax(1)`` -- what face parsing keeps of the network (my_parsing_util.py:87-88,
        models/Net.py:108-115) -- as int64 labels [B,H,W], bit-identical to the arg-max of ``forward``'s first output:
        the two auxiliary heads (training-time supervision, model.py:236-237) are not evaluated and the upsampling is
        fused with the arg-max (``hf_bilinear_argmax_nchw_f32``), so the 19 x H x W fp32 logits are never written."""
        self._check(x)
        return graphs.run(self, "labels", _params_key(self), self._parse_impl, x)

    def _parse_impl(self, x):
        pk, fuse, _, _, H, W = self._trunk(x)
        low = pk["out"].lowres(fuse)
        return nn16.bilinear_argmax_nchw(low, pk["out"].n_classes, H, W)

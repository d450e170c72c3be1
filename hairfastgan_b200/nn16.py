"""Thin Python layer over the encoder entry points of libhairfast_sm90.so (include/hairfast_b200.h,
"Encoder backbones"): NHWC 16-bit activations, wgmma convolutions with folded BatchNorm / PReLU /
LeakyReLU / residual epilogues, and the HBM-bound glue kernels around them.  CUDA only, forward only."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

import os

from . import _lib


def default_dtype() -> int:
    """16-bit operand / activation type of the ENCODER family (e4e, FS encoder, PostProcess stack, BiSeNet): fp16 unless
    HAIRFAST_ENC_DTYPE or HAIRFAST_DTYPE says bf16.  These are BatchNorm-normalised backbones (eval-mode BN folded into
    the weights, inputs in [-1, 1]; the ArcFace trunk even ships an fp16 autocast switch, arcface/iresnet.py:146) whose
    activations stay far inside fp16's range, and fp16's 11-bit significand matches the TF32 arithmetic of the
    reference's own GPU path (SURVEY F.5) -- ~8x closer than bf16 over the ~50 chained convolutions.  The generator
    keeps bf16 by default (`model.default_dtype`): StyleGAN2 activations times style scales are not bounded."""
    v = os.environ.get("HAIRFAST_ENC_DTYPE") or os.environ.get("HAIRFAST_DTYPE") or "fp16"
    return _lib.HF_BF16 if v.lower() in ("bf16", "bfloat16") else _lib.HF_F16


def torch_dtype(dt: Optional[int] = None):
    dt = default_dtype() if dt is None else dt
    return torch.float16 if dt == _lib.HF_F16 else torch.bfloat16


def _p(t):
    return None if t is None else t.data_ptr()


def _f32(t):
    return None if t is None else t.detach().float().contiguous()


def bn_affine(bn: torch.nn.BatchNorm2d):
    """Eval-mode BatchNorm2d as y = x * scale + shift."""
    scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    shift = bn.bias.detach().float() - bn.running_mean.detach().float() * scale
    return scale.contiguous(), shift.contiguous()


def to_nhwc16(x: torch.Tensor, scale=None, shift=None, c_pad: Optional[int] = None, dtype: Optional[int] = None):
    """[B,C,H,W] fp32 NCHW -> [B,H,W,c_pad] 16-bit NHWC (optionally x*scale[c]+shift[c]; zero channel padding)."""
    if not x.is_cuda:
        raise RuntimeError("to_nhwc16: input must be a CUDA tensor (no CPU fallback)")
    dt = default_dtype() if dtype is None else dtype
    xf = _f32(x)
    b, c, h, w = xf.shape
    cp = c if c_pad is None else c_pad
    y = torch.empty(b, h, w, cp, device=x.device, dtype=torch_dtype(dt))
    sc, sh = _f32(scale), _f32(shift)
    _lib.use_device(x.device.index)
    _lib.check(_lib.lib().hf_nchw_to_nhwc16(xf.data_ptr(), _p(sc), _p(sh), y.data_ptr(), b, c, cp, h, w, dt,
                                            _lib.stream_ptr()), "hf_nchw_to_nhwc16")
    return y


def to_nchw32(x16: torch.Tensor, dtype: Optional[int] = None):
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    y = torch.empty(b, c, h, w, device=x16.device, dtype=torch.float32)
    _lib.check(_lib.lib().hf_nhwc16_to_nchw(x16.data_ptr(), y.data_ptr(), b, c, h, w, dt, _lib.stream_ptr()),
               "hf_nhwc16_to_nchw")
    return y


class PackedConv2d:
    """One nn.Conv2d repacked as a K-major 16-bit GEMM operand (once per weight version).
    ``prepadded``: the input already carries the 1-pixel border (3x3, stride 1; output (H-2) x (W-2)).
    ``transposed``: ``weight`` [cin, cout, 3, 3] of nn.ConvTranspose2d(3, stride 2, padding 1, output_padding 1)."""

    def __init__(self, weight: torch.Tensor, out_scale=None, stride: int = 1, groups: int = 1,
                 cin_pad: Optional[int] = None, dtype: Optional[int] = None, prepadded: bool = False,
                 transposed: bool = False):
        dt = default_dtype() if dtype is None else dtype
        cout, cin_g, k, _ = weight.shape
        if transposed:
            cin_g, cout = cout, cin_g
        cin = cin_g * groups
        self.desc = _lib.hf_conv2d_desc(cin, cout, cin if cin_pad is None else cin_pad, k, stride, groups, dt,
                                        int(prepadded), int(transposed))
        lib = _lib.lib()
        nbytes = lib.hf_conv2d_packed_bytes(C.byref(self.desc))
        if nbytes == 0:
            _lib.check(-1, "hf_conv2d_packed_bytes")
        self.blob = torch.empty(nbytes, dtype=torch.uint8, device=weight.device)
        w, sc = _f32(weight), _f32(out_scale)
        _lib.use_device(weight.device.index)
        _lib.check(lib.hf_conv2d_pack(C.byref(self.desc), w.data_ptr(), _p(sc), self.blob.data_ptr(), _lib.stream_ptr()),
                   "hf_conv2d_pack")
        self.cout, self.k, self.stride, self.dtype = cout, k, stride, dt
        self.prepadded, self.transposed = prepadded, transposed

    def __call__(self, x16: torch.Tensor, shift=None, act: int = 0, slope=None, slope0: float = 0.0, residual16=None,
                 want_y16: bool = True, y16b_affine=None, want_y32: bool = False, act_after_residual: bool = False):
        """Returns (y16 | None, y16b | None, y32 | None)."""
        b, h, w, _ = x16.shape
        if self.transposed:
            ho, wo = 2 * h, 2 * w
        elif self.prepadded:
            ho, wo = h - 2, w - 2
        else:
            ho, wo = ((h + 1) // 2, (w + 1) // 2) if self.stride == 2 else (h, w)
        dev = x16.device
        io = _lib.hf_conv2d_io()
        io.batch, io.height, io.width, io.x16 = b, h, w, x16.data_ptr()
        keep = [_f32(shift), _f32(slope)]
        io.shift, io.act, io.slope, io.slope0 = _p(keep[0]), act, _p(keep[1]), float(slope0)
        if residual16 is not None:
            io.residual16 = residual16.data_ptr()
        io.act_after_residual = 1 if act_after_residual else 0
        y16 = y16b = y32 = None
        if want_y16:
            y16 = torch.empty(b, ho, wo, self.cout, device=dev, dtype=torch_dtype(self.dtype))
            io.y16 = y16.data_ptr()
        if y16b_affine is not None:
            s2, b2 = _f32(y16b_affine[0]), _f32(y16b_affine[1])
            keep += [s2, b2]
            y16b = torch.empty(b, ho, wo, self.cout, device=dev, dtype=torch_dtype(self.dtype))
            io.y16b_scale, io.y16b_shift, io.y16b = s2.data_ptr(), b2.data_ptr(), y16b.data_ptr()
        if want_y32:
            y32 = torch.empty(b, self.cout, ho, wo, device=dev, dtype=torch.float32)
            io.y32_nchw = y32.data_ptr()
        _lib.use_device(dev.index)
        _lib.check(_lib.lib().hf_conv2d_forward(C.byref(self.desc), self.blob.data_ptr(), C.byref(io), _lib.stream_ptr()),
                   "hf_conv2d_forward")
        return y16, y16b, y32


def channel_mean(x16: torch.Tensor, dtype: Optional[int] = None):
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    m = torch.empty(b, c, device=x16.device, dtype=torch.float32)
    ws = torch.empty(_lib.lib().hf_channel_reduce_workspace_bytes(b, h * w, c), device=x16.device, dtype=torch.uint8)
    _lib.check(_lib.lib().hf_channel_mean_nhwc16(x16.data_ptr(), m.data_ptr(), ws.data_ptr(), b, h * w, c, dt,
                                                 _lib.stream_ptr()), "hf_channel_mean_nhwc16")
    return m


def instance_norm_lrelu(x16: torch.Tensor, slope: float = 0.2, dtype: Optional[int] = None):
    """InstanceNorm2d(affine=False) + LeakyReLU(slope) of [B,H,W,C] 16-bit NHWC -> same shape."""
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    y = torch.empty_like(x16)
    ws = torch.empty(_lib.lib().hf_instance_norm_workspace_bytes(b, h * w, c), device=x16.device, dtype=torch.uint8)
    _lib.check(_lib.lib().hf_instance_norm_lrelu_nhwc16(x16.data_ptr(), y.data_ptr(), ws.data_ptr(), b, h * w, c,
                                                        float(slope), dt, _lib.stream_ptr()),
               "hf_instance_norm_lrelu_nhwc16")
    return y


def reflect_pad1(x16: torch.Tensor, dtype: Optional[int] = None):
    """ReflectionPad2d(1) of [B,H,W,C] 16-bit NHWC -> [B,H+2,W+2,C]."""
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    y = torch.empty(b, h + 2, w + 2, c, device=x16.device, dtype=x16.dtype)
    _lib.check(_lib.lib().hf_reflect_pad1_nhwc16(x16.data_ptr(), y.data_ptr(), b, h, w, c, dt, _lib.stream_ptr()),
               "hf_reflect_pad1_nhwc16")
    return y


def se_gate(x16: torch.Tensor, fc1_weight: torch.Tensor, fc2_weight: torch.Tensor, dtype: Optional[int] = None):
    """SEModule gate (helpers.py:57-75) of an NHWC 16-bit tensor: [B,C] fp32."""
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    w1, w2 = _f32(fc1_weight).reshape(-1, c), _f32(fc2_weight).reshape(c, -1)
    gate = torch.empty(b, c, device=x16.device, dtype=torch.float32)
    ws = torch.empty(_lib.lib().hf_channel_reduce_workspace_bytes(b, h * w, c), device=x16.device, dtype=torch.uint8)
    _lib.check(_lib.lib().hf_se_gate_nhwc16(x16.data_ptr(), w1.data_ptr(), w2.data_ptr(), gate.data_ptr(), ws.data_ptr(),
                                            b, h * w, c, w1.shape[0], dt, _lib.stream_ptr()), "hf_se_gate_nhwc16")
    return gate


def scale_add(res16, se=None, shortcut16=None, shortcut_stride: int = 1, y16b_affine=None, want_y16: bool = True,
              dtype: Optional[int] = None):
    """res16 * se[b,c] + shortcut16[:, ::s, ::s] (s = shortcut_stride): the shortcut must be [B, H*s, W*s, C].  The
    MaxPool2d(1, 2) shortcut of an odd (2H-1) x (2W-1) input also subsamples to H x W, but the kernel indexes the
    shortcut with the pitch of 2H x 2W, so that shape is rejected here rather than read out of bounds."""
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = res16.shape
    if shortcut16 is not None:
        want = (b, h * shortcut_stride, w * shortcut_stride, c)
        if tuple(shortcut16.shape) != want:
            raise ValueError(f"scale_add: shortcut of shape {list(shortcut16.shape)}, expected {list(want)} "
                             f"for stride {shortcut_stride}")
    y = torch.empty_like(res16) if want_y16 else None
    yb, s2, b2 = None, None, None
    if y16b_affine is not None:
        s2, b2 = _f32(y16b_affine[0]), _f32(y16b_affine[1])
        yb = torch.empty_like(res16)
    sef = _f32(se)
    _lib.check(_lib.lib().hf_scale_add_nhwc16(res16.data_ptr(), _p(sef), _p(shortcut16), shortcut_stride, _p(s2), _p(b2),
                                              _p(y), _p(yb), b, h, w, c, dt, _lib.stream_ptr()), "hf_scale_add_nhwc16")
    return y, yb


def upsample_add(x16, y16, dtype: Optional[int] = None):
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    _, hh, ww, _ = y16.shape
    out = torch.empty_like(y16)
    _lib.check(_lib.lib().hf_upsample_add_nhwc16(x16.data_ptr(), y16.data_ptr(), out.data_ptr(), b, h, w, hh, ww, c, dt,
                                                 _lib.stream_ptr()), "hf_upsample_add_nhwc16")
    return out


def adaptive_avgpool(x16, oh: int, ow: int, dtype: Optional[int] = None):
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    y = torch.empty(b, c, oh, ow, device=x16.device, dtype=torch.float32)
    _lib.check(_lib.lib().hf_adaptive_avgpool_nhwc16(x16.data_ptr(), y.data_ptr(), b, h, w, c, oh, ow, dt,
                                                     _lib.stream_ptr()), "hf_adaptive_avgpool_nhwc16")
    return y


# ------------------------------------------------------------------------------------------------ BiSeNet glue
class PackedStem7x7:
    """Resnet18.conv1 + bn1 + ReLU (face_parsing/resnet.py:60-61,69-70) as ONE fused kernel (`hf_stem7x7s2_nhwc16`):
    the 7x7 window is gathered in shared memory, no im2col tensor in HBM.  Packed weights: 16-bit [64][184] with
    k = ky*24 + kx*3 + c and the BatchNorm scale folded in; the BatchNorm shift is the epilogue bias."""

    def __init__(self, weight: torch.Tensor, bn: torch.nn.BatchNorm2d, dtype: Optional[int] = None):
        self.dtype = default_dtype() if dtype is None else dtype
        scale, self.shift = bn_affine(bn)
        w = _f32(weight)
        cout = w.shape[0]
        if tuple(w.shape) != (64, 3, 7, 7):
            raise NotImplementedError(f"stem7x7s2: expected a [64,3,7,7] weight, got {list(w.shape)}")
        wk = (w * scale.view(-1, 1, 1, 1)).permute(0, 2, 3, 1).reshape(cout, 7, 21)      # [n][ky][kx*3 + c]
        packed = torch.zeros(cout, 184, device=w.device, dtype=torch.float32)
        packed[:, :168].view(cout, 7, 24)[:, :, :21] = wk
        self.wp = packed.to(torch_dtype(self.dtype)).contiguous()

    def __call__(self, x: torch.Tensor):
        """[B,3,H,W] fp32 NCHW -> [B,Ho,Wo,64] 16-bit NHWC."""
        if not x.is_cuda:
            raise RuntimeError("stem7x7s2: input must be a CUDA tensor (no CPU fallback)")
        xf = _f32(x)
        b, c, h, w = xf.shape
        if c != 3:
            raise ValueError("stem7x7s2: expected a 3-channel image")
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        y = torch.empty(b, ho, wo, 64, device=x.device, dtype=torch_dtype(self.dtype))
        _lib.use_device(x.device.index)
        _lib.check(_lib.lib().hf_stem7x7s2_nhwc16(xf.data_ptr(), self.wp.data_ptr(), self.shift.data_ptr(), y.data_ptr(),
                                                  b, h, w, self.dtype, _lib.stream_ptr()), "hf_stem7x7s2_nhwc16")
        return y


class PackedStem3x3:
    """Conv2d(3, 64, 3, 1, 1) + eval BatchNorm + PReLU of the IR-SE / iresnet encoders (psp_encoders.py:176-178,
    arcface/iresnet.py:92-95) as ONE fused kernel (`hf_stem3x3_nhwc16`): fp32 NCHW image in, the raw 16-bit NHWC
    activation and (optionally) its BatchNorm-affined copy for the first residual block out.  Packed weights: 16-bit
    [64][56], k = ky*16 + kx*4 + c, BatchNorm scale folded in."""

    def __init__(self, weight: torch.Tensor, bn: torch.nn.BatchNorm2d, prelu_weight: torch.Tensor,
                 dtype: Optional[int] = None):
        self.dtype = default_dtype() if dtype is None else dtype
        w = _f32(weight)
        if tuple(w.shape) != (64, 3, 3, 3):
            raise NotImplementedError(f"stem3x3: expected a [64,3,3,3] weight, got {list(w.shape)}")
        scale, self.shift = bn_affine(bn)
        self.slope = _f32(prelu_weight).reshape(-1)
        if self.slope.numel() != 64:
            raise NotImplementedError("stem3x3: per-channel PReLU (64 slopes) expected")
        wk = (w * scale.view(-1, 1, 1, 1)).permute(0, 2, 3, 1)                   # [n][ky][kx][c]
        packed = torch.zeros(64, 56, device=w.device, dtype=torch.float32)
        packed[:, :48].view(64, 3, 4, 4)[:, :, :3, :3] = wk
        self.wp = packed.to(torch_dtype(self.dtype)).contiguous()

    def __call__(self, x: torch.Tensor, y16b_affine=None):
        """[B,3,H,W] fp32 NCHW -> (y16, y16b | None), both [B,H,W,64] 16-bit NHWC."""
        if not x.is_cuda:
            raise RuntimeError("stem3x3: input must be a CUDA tensor (no CPU fallback)")
        xf = _f32(x)
        b, c, h, w = xf.shape
        if c != 3:
            raise ValueError("stem3x3: expected a 3-channel image")
        y = torch.empty(b, h, w, 64, device=x.device, dtype=torch_dtype(self.dtype))
        yb = s2 = b2 = None
        if y16b_affine is not None:
            s2, b2 = _f32(y16b_affine[0]), _f32(y16b_affine[1])
            yb = torch.empty_like(y)
        _lib.use_device(x.device.index)
        _lib.check(_lib.lib().hf_stem3x3_nhwc16(xf.data_ptr(), self.wp.data_ptr(), self.shift.data_ptr(),
                                                self.slope.data_ptr(), _p(s2), _p(b2), y.data_ptr(), _p(yb), b, h, w,
                                                self.dtype, _lib.stream_ptr()), "hf_stem3x3_nhwc16")
        return y, yb


def stem7x7s2(x: torch.Tensor, weight: torch.Tensor, bn: torch.nn.BatchNorm2d, dtype: Optional[int] = None):
    return PackedStem7x7(weight, bn, dtype)(x)


def maxpool3x3s2(x16: torch.Tensor, dtype: Optional[int] = None):
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    y = torch.empty(b, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c, device=x16.device, dtype=x16.dtype)
    _lib.check(_lib.lib().hf_maxpool3x3s2_nhwc16(x16.data_ptr(), y.data_ptr(), b, h, w, c, dt, _lib.stream_ptr()),
               "hf_maxpool3x3s2_nhwc16")
    return y


def pooled_fc(x16: torch.Tensor, weight: torch.Tensor, scale=None, shift=None, act: int = 0,
              dtype: Optional[int] = None):
    """act((W . mean_hw(x)) * scale + shift): [B,H,W,C] 16-bit NHWC -> [B,Cout] fp32 (act: 0 none, 1 ReLU, 2 sigmoid)."""
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    wf = _f32(weight).reshape(weight.shape[0], c)
    sc, sh = _f32(scale), _f32(shift)
    out = torch.empty(b, wf.shape[0], device=x16.device, dtype=torch.float32)
    ws = torch.empty(_lib.lib().hf_channel_reduce_workspace_bytes(b, h * w, c), device=x16.device, dtype=torch.uint8)
    _lib.check(_lib.lib().hf_pooled_fc_nhwc16(x16.data_ptr(), wf.data_ptr(), _p(sc), _p(sh), act, out.data_ptr(),
                                              ws.data_ptr(), b, h * w, c, wf.shape[0], dt, _lib.stream_ptr()),
               "hf_pooled_fc_nhwc16")
    return out


def gate_add_up(x16: torch.Tensor, gate=None, addvec=None, addt16=None, up: int = 1, dtype: Optional[int] = None):
    """nearest_up(x * gate[b,c] + addvec[b,c] + addt): [B,h,w,C] -> [B,h*up,w*up,C] 16-bit NHWC."""
    dt = default_dtype() if dtype is None else dtype
    b, h, w, c = x16.shape
    y = torch.empty(b, h * up, w * up, c, device=x16.device, dtype=x16.dtype)
    g, a = _f32(gate), _f32(addvec)
    _lib.check(_lib.lib().hf_gate_add_up_nhwc16(x16.data_ptr(), _p(g), _p(a), _p(addt16), y.data_ptr(), b, h, w, c, up, dt,
                                                _lib.stream_ptr()), "hf_gate_add_up_nhwc16")
    return y


def bilinear_upsample_nchw(x: torch.Tensor, channels: int, height: int, width: int):
    """F.interpolate(x[:, :channels], (height, width), mode='bilinear', align_corners=True) on fp32 NCHW."""
    b, cin, h, w = x.shape
    y = torch.empty(b, channels, height, width, device=x.device, dtype=torch.float32)
    _lib.check(_lib.lib().hf_bilinear_upsample_nchw_f32(x.data_ptr(), y.data_ptr(), b, channels, cin, h, w, height, width,
                                                        _lib.stream_ptr()), "hf_bilinear_upsample_nchw_f32")
    return y


def bilinear_argmax_nchw(x: torch.Tensor, channels: int, height: int, width: int):
    """argmax over the first `channels` planes of F.interpolate(x, (height, width), 'bilinear', align_corners=True):
    int64 labels [B, height, width]; the full-resolution logits are never written."""
    b, cin, h, w = x.shape
    y = torch.empty(b, height, width, device=x.device, dtype=torch.int64)
    _lib.check(_lib.lib().hf_bilinear_argmax_nchw_f32(x.data_ptr(), y.data_ptr(), b, channels, cin, h, w, height, width,
                                                      _lib.stream_ptr()), "hf_bilinear_argmax_nchw_f32")
    return y

"""H100-native StyleGAN2 generator modules -- a drop-in for the reference module surface
``models/stylegan2/model.py`` (PixelNorm :16, Upsample :35, Downsample :56, Blur :77, EqualLinear :134,
ModulatedConv2d :183, NoiseInjection :282, ConstantInput :296, StyledConv :309, ToRGB :346,
Generator :368): identical constructor / forward signatures and identical ``state_dict`` keys, so
``generator.load_state_dict(ckpt['g_ema'])`` (models/Net.py:39) and every ``net.generator(...)`` call
in models/{Embedding,Alignment,Blending}.py work unchanged.

The modules only hold parameters and translate the call into one C-ABI call of
libhairfast_sm90.so (include/hairfast_b200.h):

* ``Generator.forward``      -> ``hf_generator_forward`` (whole chain, fused epilogues)
* ``StyledConv`` / ``ModulatedConv2d`` -> ``hf_conv_forward``
* ``ToRGB``                  -> ``hf_torgb_forward``
* ``Blur`` / ``Upsample`` / ``Downsample`` / ``FusedLeakyReLU`` -> the op package.

Forward only (the reference path runs under ``torch.inference_mode``); CUDA only, no fallback.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import random

import torch
from torch import nn
from torch.nn import functional as F

from . import _lib
from .op import FusedLeakyReLU, fused_leaky_relu, upfirdn2d


def default_dtype() -> int:
    """16-bit operand type of the tensor-core path: bf16 unless HAIRFAST_DTYPE=fp16."""
    return _lib.HF_F16 if os.environ.get("HAIRFAST_DTYPE", "bf16").lower() in ("fp16", "f16", "half") else _lib.HF_BF16


def _ptr(t):
    return None if t is None else t.data_ptr()


def _f32c(t: torch.Tensor) -> torch.Tensor:
    t = t.detach()
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _alloc_bytes(nbytes: int, device) -> torch.Tensor:
    # torch's caching allocator returns >= 512-byte aligned blocks
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


class PixelNorm(nn.Module):
    def forward(self, input):
        return input * torch.rsqrt(input.square().mean(dim=1, keepdim=True) + 1e-8)


def make_kernel(k):
    k = torch.as_tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = torch.outer(k, k)
    return k / k.sum()


class Upsample(nn.Module):
    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        self.register_buffer("kernel", make_kernel(kernel) * (factor ** 2))
        p = self.kernel.shape[0] - factor
        self.pad = ((p + 1) // 2 + factor - 1, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=self.factor, down=1, pad=self.pad)


class Downsample(nn.Module):
    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        self.register_buffer("kernel", make_kernel(kernel))
        p = self.kernel.shape[0] - factor
        self.pad = ((p + 1) // 2, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=1, down=self.factor, pad=self.pad)


class Blur(nn.Module):
    def __init__(self, kernel, pad, upsample_factor=1):
        super().__init__()
        k = make_kernel(kernel)
        if upsample_factor > 1:
            k = k * (upsample_factor ** 2)
        self.register_buffer("kernel", k)
        self.pad = pad

    def forward(self, input):
        return upfirdn2d(input, self.kernel, pad=self.pad)


class EqualLinear(nn.Module):
    """Equalised-lr linear layer (reference model.py:134-163).  The mapping MLP is not on the swap()
    path (input_is_latent=True everywhere); it runs as a cuBLAS GEMM + our fused bias/lrelu op."""

    def __init__(self, in_dim, out_dim, bias=True, bias_init=0, lr_mul=1, activation=None):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_dim, in_dim).div_(lr_mul))
        self.bias = nn.Parameter(torch.full((out_dim,), float(bias_init))) if bias else None
        self.activation = activation
        self.scale = (1 / math.sqrt(in_dim)) * lr_mul
        self.lr_mul = lr_mul

    def forward(self, input):
        w = self.weight * self.scale
        if self.activation:
            return fused_leaky_relu(F.linear(input, w), self.bias * self.lr_mul)
        return F.linear(input, w, bias=None if self.bias is None else self.bias * self.lr_mul)

    def __repr__(self):
        return f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]})"


class ScaledLeakyReLU(nn.Module):
    def __init__(self, negative_slope=0.2):
        super().__init__()
        self.negative_slope = negative_slope

    def forward(self, input):
        return F.leaky_relu(input, negative_slope=self.negative_slope) * math.sqrt(2)


def _expect_shape(t: torch.Tensor, shape, what: str) -> None:
    """The C ABI receives raw pointers: every tensor's full shape is checked here, where the reference would raise
    a shape error from torch (None in `shape` = any size)."""
    ok = t.dim() == len(shape) and all(e is None or int(a) == int(e) for a, e in zip(t.shape, shape))
    if not ok:
        want = "[" + ", ".join("*" if e is None else str(e) for e in shape) + "]"
        raise RuntimeError(f"{what}: expected shape {want}, got {list(t.shape)}")


class _PackedConv:
    """Lazily (re)packed tensor-core operand of one ModulatedConv2d, keyed on the parameter version."""

    def __init__(self):
        self.key = None
        self.blob = None
        self.desc = None

    def get(self, conv: "ModulatedConv2d", dtype: int):
        w = conv.weight
        blur = conv.blur.kernel if conv.upsample else None
        key = (w.data_ptr(), w._version, str(w.device), dtype, None if blur is None else blur._version)
        if key != self.key:
            lib = _lib.lib()
            desc = _lib.hf_conv_desc(conv.in_channel, conv.out_channel, conv.kernel_size, int(conv.upsample), dtype)
            nbytes = lib.hf_conv_packed_bytes(C.byref(desc))
            if nbytes == 0:
                _lib.check(-1, "hf_conv_packed_bytes")
            blob = _alloc_bytes(nbytes, w.device)
            wf = _f32c(w)
            bf = None if blur is None else _f32c(blur)
            _lib.check(lib.hf_conv_pack(C.byref(desc), wf.data_ptr(), _ptr(bf), blob.data_ptr(), _lib.stream_ptr()),
                       "hf_conv_pack")
            self.key, self.blob, self.desc = key, blob, desc
        return self.desc, self.blob


class ModulatedConv2d(nn.Module):
    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True, upsample=False,
                 downsample=False, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        self.eps = 1e-8
        self.kernel_size = kernel_size
        self.in_channel = in_channel
        self.out_channel = out_channel
        self.upsample = upsample
        self.downsample = downsample
        if upsample:
            factor = 2
            p = (len(blur_kernel) - factor) - (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2 + factor - 1, p // 2 + 1), upsample_factor=factor)
        if downsample:
            raise NotImplementedError(
                "ModulatedConv2d(downsample=True) is never built by the Generator (reference model.py:265-271 is "
                "dead code on the inference path) and is not implemented")
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.padding = kernel_size // 2
        self.weight = nn.Parameter(torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))
        self.modulation = EqualLinear(style_dim, in_channel, bias_init=1)
        self.demodulate = demodulate
        self._packed = _PackedConv()

    def __repr__(self):
        return (f"{self.__class__.__name__}({self.in_channel}, {self.out_channel}, {self.kernel_size}, "
                f"upsample={self.upsample}, downsample={self.downsample})")

    def _run(self, input, style, noise=None, noise_weight=None, act_bias=None, act=0, dtype=None):
        if not input.is_cuda:
            raise RuntimeError("ModulatedConv2d: input must be a CUDA tensor (no CPU fallback)")
        dtype = default_dtype() if dtype is None else dtype
        lib = _lib.lib()
        _lib.use_device(input.device.index)
        batch, cin, height, width = input.shape
        if cin != self.in_channel:
            raise RuntimeError(f"ModulatedConv2d: expected {self.in_channel} input channels, got {cin}")
        _expect_shape(style, (batch, self.modulation.weight.shape[1]), "ModulatedConv2d style")
        if noise is not None:
            f = 2 if self.upsample else 1
            if noise.dim() != 4 or noise.shape[0] not in (1, batch):
                raise RuntimeError(f"StyledConv noise: expected [1|{batch}, 1, {height * f}, {width * f}], "
                                   f"got {list(noise.shape)}")
            _expect_shape(noise, (None, 1, height * f, width * f), "StyledConv noise")
        desc, blob = self._packed.get(self, dtype)
        x = _f32c(input)
        st = _f32c(style)
        mw, mb = _f32c(self.modulation.weight), _f32c(self.modulation.bias)
        ho, wo = (2 * height, 2 * width) if self.upsample else (height, width)
        y = torch.empty(batch, self.out_channel, ho, wo, device=x.device, dtype=torch.float32)
        ws = _alloc_bytes(lib.hf_conv_workspace_bytes(C.byref(desc), batch, height, width), x.device)
        io = _lib.hf_conv_io()
        io.batch, io.height, io.width = batch, height, width
        io.x, io.x_batch_broadcast = x.data_ptr(), 0
        io.style, io.style_dim, io.style_stride = st.data_ptr(), st.shape[-1], st.stride(0)
        io.mod_weight, io.mod_bias, io.demodulate = mw.data_ptr(), mb.data_ptr(), int(self.demodulate)
        keep = []
        if noise is not None:
            nz = _f32c(noise)
            nwt = _f32c(noise_weight)
            keep += [nz, nwt]
            io.noise, io.noise_batch, io.noise_weight = nz.data_ptr(), nz.shape[0], nwt.data_ptr()
        if act_bias is not None:
            ab = _f32c(act_bias)
            keep.append(ab)
            io.act_bias = ab.data_ptr()
        io.act = act
        io.y, io.workspace = y.data_ptr(), ws.data_ptr()
        _lib.check(lib.hf_conv_forward(C.byref(desc), blob.data_ptr(), C.byref(io), _lib.stream_ptr()),
                   "hf_conv_forward")
        return y

    def forward(self, input, style):
        return self._run(input, style)


class NoiseInjection(nn.Module):
    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(1))

    def forward(self, image, noise=None):
        if noise is None:
            batch, _, height, width = image.shape
            noise = image.new_empty(batch, 1, height, width).normal_()
        return image + self.weight * noise


class ConstantInput(nn.Module):
    def __init__(self, channel, size=4):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))

    def forward(self, input):
        return self.input.repeat(input.shape[0], 1, 1, 1)


class StyledConv(nn.Module):
    def __init__(self, in_channel, out_channel, kernel_size, style_dim, upsample=False, blur_kernel=[1, 3, 3, 1],
                 demodulate=True):
        super().__init__()
        self.conv = ModulatedConv2d(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                                    blur_kernel=blur_kernel, demodulate=demodulate)
        self.noise = NoiseInjection()
        self.activate = FusedLeakyReLU(out_channel)

    def forward(self, input, style, noise=None):
        """conv -> + noise_weight * noise -> lrelu(. + bias) * sqrt(2), one fused kernel epilogue.
        ``noise=None`` draws N(0,1) of shape [B,1,Ho,Wo] from torch's generator, exactly where the
        reference does (model.py:288-291), so seeded runs consume the RNG identically."""
        if noise is None:
            batch, _, height, width = input.shape
            f = 2 if self.conv.upsample else 1
            noise = input.new_empty(batch, 1, height * f, width * f).normal_()
        return self.conv._run(input, style, noise=noise, noise_weight=self.noise.weight,
                              act_bias=self.activate.bias, act=1)


class ToRGB(nn.Module):
    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        if upsample:
            self.upsample = Upsample(blur_kernel)
        self.conv = ModulatedConv2d(in_channel, 3, 1, style_dim, demodulate=False)
        self.bias = nn.Parameter(torch.zeros(1, 3, 1, 1))

    def forward(self, input, style, skip=None):
        if not input.is_cuda:
            raise RuntimeError("ToRGB: input must be a CUDA tensor (no CPU fallback)")
        lib = _lib.lib()
        _lib.use_device(input.device.index)
        batch, cin, height, width = input.shape
        _expect_shape(input, (batch, self.conv.in_channel, height, width), "ToRGB input")
        _expect_shape(style, (batch, self.conv.modulation.weight.shape[1]), "ToRGB style")
        if skip is not None:
            _expect_shape(skip, (batch, 3, height // 2, width // 2), "ToRGB skip")
            if height % 2 or width % 2:
                raise RuntimeError("ToRGB: a skip needs an even-sized input")
        x, st = _f32c(input), _f32c(style)
        w, mw, mb = _f32c(self.conv.weight), _f32c(self.conv.modulation.weight), _f32c(self.conv.modulation.bias)
        bias = _f32c(self.bias)
        sk = upk = None
        if skip is not None:
            if not hasattr(self, "upsample"):
                raise RuntimeError("ToRGB(upsample=False) cannot take a skip")
            sk, upk = _f32c(skip), _f32c(self.upsample.kernel)
        y = torch.empty(batch, 3, height, width, device=x.device, dtype=torch.float32)
        ws = _alloc_bytes(batch * cin * 4, x.device)
        _lib.check(lib.hf_torgb_forward(x.data_ptr(), st.data_ptr(), st.stride(0), st.shape[-1], w.data_ptr(),
                                        mw.data_ptr(), mb.data_ptr(), bias.data_ptr(), _ptr(upk), _ptr(sk),
                                        y.data_ptr(), batch, cin, height, width, ws.data_ptr(), _lib.stream_ptr()),
                   "hf_torgb_forward")
        return y


class Generator(nn.Module):
    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], lr_mlp=0.01):
        super().__init__()
        self.size = size
        self.style_dim = style_dim
        self.channel_multiplier = channel_multiplier
        mapping = [PixelNorm()]
        mapping += [EqualLinear(style_dim, style_dim, lr_mul=lr_mlp, activation="fused_lrelu") for _ in range(n_mlp)]
        self.style = nn.Sequential(*mapping)
        self.channels = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * channel_multiplier,
                         128: 128 * channel_multiplier, 256: 64 * channel_multiplier,
                         512: 32 * channel_multiplier, 1024: 16 * channel_multiplier}
        self.input = ConstantInput(self.channels[4])
        self.conv1 = StyledConv(self.channels[4], self.channels[4], 3, style_dim, blur_kernel=blur_kernel)
        self.to_rgb1 = ToRGB(self.channels[4], style_dim, upsample=False)
        self.log_size = int(math.log(size, 2))
        self.num_layers = (self.log_size - 2) * 2 + 1
        self.convs = nn.ModuleList()
        self.upsamples = nn.ModuleList()
        self.to_rgbs = nn.ModuleList()
        self.noises = nn.Module()
        for layer_idx in range(self.num_layers):
            res = (layer_idx + 5) // 2
            self.noises.register_buffer(f"noise_{layer_idx}", torch.randn(1, 1, 2 ** res, 2 ** res))
        in_channel = self.channels[4]
        for i in range(3, self.log_size + 1):
            out_channel = self.channels[2 ** i]
            self.convs.append(StyledConv(in_channel, out_channel, 3, style_dim, upsample=True, blur_kernel=blur_kernel))
            self.convs.append(StyledConv(out_channel, out_channel, 3, style_dim, blur_kernel=blur_kernel))
            self.to_rgbs.append(ToRGB(out_channel, style_dim))
            in_channel = out_channel
        self.n_latent = self.log_size * 2 - 2
        self._pack_key = None
        self._packed = None
        self._workspace = {}
        self.compute_dtype = None      # None -> default_dtype()

    # ------------------------------------------------------------------ reference helper surface
    def make_noise(self):
        device = self.input.input.device
        noises = [torch.randn(1, 1, 4, 4, device=device)]
        for i in range(3, self.log_size + 1):
            noises += [torch.randn(1, 1, 2 ** i, 2 ** i, device=device) for _ in range(2)]
        return noises

    def mean_latent(self, n_latent):
        latent_in = torch.randn(n_latent, self.style_dim, device=self.input.input.device)
        return self.style(latent_in).mean(0, keepdim=True)

    def get_latent(self, input):
        return self.style(input)

    # ------------------------------------------------------------------ packing
    def _styled(self):
        return [self.conv1] + list(self.convs)

    def _rgbs(self):
        return [self.to_rgb1] + list(self.to_rgbs)

    def _config(self):
        dtype = default_dtype() if self.compute_dtype is None else self.compute_dtype
        return _lib.hf_gen_config(self.size, self.style_dim, self.channel_multiplier, dtype)

    def _ensure_packed(self, device):
        cfg = self._config()
        params = [self.input.input]
        for s in self._styled():
            params += [s.conv.weight, s.conv.modulation.weight, s.conv.modulation.bias, s.noise.weight, s.activate.bias]
            if s.conv.upsample:
                params.append(s.conv.blur.kernel)
        for r in self._rgbs():
            params += [r.conv.weight, r.conv.modulation.weight, r.conv.modulation.bias, r.bias]
            if hasattr(r, "upsample"):
                params.append(r.upsample.kernel)
        key = (cfg.dtype, str(device), tuple((p.data_ptr(), p._version) for p in params))
        if key == self._pack_key:
            return cfg
        lib = _lib.lib()
        w = _lib.hf_gen_weights()
        keep = []

        def P(t):
            t = _f32c(t)
            if t.device != device:
                raise RuntimeError("Generator parameters and inputs are on different devices")
            keep.append(t)
            return t.data_ptr()

        w.const_input = P(self.input.input)
        for i, s in enumerate(self._styled()):
            w.conv_weight[i] = P(s.conv.weight)
            w.conv_mod_weight[i] = P(s.conv.modulation.weight)
            w.conv_mod_bias[i] = P(s.conv.modulation.bias)
            w.conv_blur_kernel[i] = P(s.conv.blur.kernel) if s.conv.upsample else None
            w.conv_noise_weight[i] = P(s.noise.weight)
            w.conv_act_bias[i] = P(s.activate.bias)
        for i, r in enumerate(self._rgbs()):
            w.rgb_weight[i] = P(r.conv.weight)
            w.rgb_mod_weight[i] = P(r.conv.modulation.weight)
            w.rgb_mod_bias[i] = P(r.conv.modulation.bias)
            w.rgb_bias[i] = P(r.bias)
            w.rgb_up_kernel[i] = P(r.upsample.kernel) if hasattr(r, "upsample") else None
        nbytes = lib.hf_generator_packed_bytes(C.byref(cfg))
        if nbytes == 0:
            _lib.check(-1, "hf_generator_packed_bytes")
        blob = _alloc_bytes(nbytes, device)
        _lib.check(lib.hf_generator_pack(C.byref(cfg), C.byref(w), blob.data_ptr(), _lib.stream_ptr()),
                   "hf_generator_pack")
        self._packed, self._pack_key = blob, key
        del keep
        return cfg

    def _get_workspace(self, cfg, batch, device):
        # one grow-only buffer per device: the layout is recomputed from (cfg, batch) on every call, so a
        # workspace sized for a larger batch serves every smaller one.  Captured CUDA graphs bake the pointer in, so a
        # growth allocates at least the graph batch cap up front and drops the graphs captured on the old buffer.
        nbytes = _lib.lib().hf_generator_workspace_bytes(C.byref(cfg), batch)
        ws = self._workspace.get(str(device))
        if ws is None or ws.numel() < nbytes:
            from . import graphs
            if ws is not None:
                self.__dict__.pop("_hf_graphs", None)             # graphs on the old buffer are dropped with it
            if graphs.enabled() and batch <= graphs._max_batch():
                nbytes = max(nbytes, _lib.lib().hf_generator_workspace_bytes(C.byref(cfg), graphs._max_batch()))
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("Generator workspace must be allocated before a CUDA-graph capture")
            ws = self._workspace[str(device)] = _alloc_bytes(nbytes, device)
        return ws

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def consume_noise(self, batch: int, device=None) -> None:
        """Advance the RNG exactly as a full ``forward(..., noise=None, randomize_noise=True)`` of ``batch`` samples
        would (one ``normal_()`` of shape [batch,1,R,R] per StyledConv, in execution order -- NoiseInjection.forward,
        model.py:288-291) without running the network.  Used by the opt-in FSE fast path (`fse_fast.py`) that skips
        the reconstruction image nobody reads while keeping every later random draw of ``swap()`` unchanged."""
        dev = self.input.input.device if device is None else device
        for i in range(self.num_layers):
            r = 4 if i == 0 else 2 ** ((i + 1) // 2 + 2)
            torch.empty(batch, 1, r, r, device=dev, dtype=torch.float32).normal_()

    def forward(self, styles, return_latents=False, inject_index=None, truncation=1, truncation_latent=None,
                input_is_latent=False, noise=None, randomize_noise=True, layer_in=None, skip=None,
                start_layer=0, end_layer=8, return_rgb=False):
        latent = self._build_latent(styles, inject_index, truncation, truncation_latent, input_is_latent)
        if noise is None and latent.is_cuda and latent.dim() == 3:
            # the fixed launch sequence of this (batch, range) signature replays as one CUDA graph (graphs.py); explicit
            # noise lists / the FSE feature insertion / large batches stay eager
            from . import graphs
            cfg = self._ensure_packed(latent.device)

            def fn(lat, lin, sk):
                early, feat, rgb, _ = self._run(lat, None, randomize_noise, lin, sk, start_layer, end_layer)
                return early, feat, rgb
            early, out_feat, out_rgb = graphs.run_multi(
                self, ("gen", start_layer, end_layer, bool(randomize_noise), cfg.dtype), self._pack_key, fn,
                (latent if latent.dtype == torch.float32 else latent.float(), layer_in, skip), int(latent.shape[0]),
                uses_rng=bool(randomize_noise))
        else:
            early, out_feat, out_rgb, _ = self._run(latent, noise, randomize_noise, layer_in, skip, start_layer,
                                                    end_layer)
        if early:
            return out_feat, out_rgb
        return (out_rgb, latent) if return_latents else (out_rgb, None)

    def _build_latent(self, styles, inject_index, truncation, truncation_latent, input_is_latent):
        """styles -> [B, n_latent, style_dim] exactly as the reference does (model.py:494-531)."""
        if not input_is_latent:
            styles = [self.style(s) for s in styles]
        if truncation < 1:
            styles = [truncation_latent + truncation * (s - truncation_latent) for s in styles]
        if len(styles) < 2:
            inject_index = self.n_latent
            latent = styles[0].unsqueeze(1).repeat(1, inject_index, 1) if styles[0].ndim < 3 else styles[0]
        else:
            if inject_index is None:
                inject_index = random.randint(1, self.n_latent - 1)
            latent = torch.cat([styles[0].unsqueeze(1).repeat(1, inject_index, 1),
                                styles[1].unsqueeze(1).repeat(1, self.n_latent - inject_index, 1)], 1)
        return latent

    def _run(self, latent, noise, randomize_noise, layer_in=None, skip=None, start_layer=0, end_layer=8,
             features_in=None, feature_scale=1.0, return_features=False):
        """One hf_generator_forward call.  Returns (early_exit, out_feature, out_rgb, outs)."""
        if not latent.is_cuda:
            raise RuntimeError("Generator: latent must be a CUDA tensor (hairfastgan_b200 has no CPU fallback)")
        device = latent.device
        _lib.use_device(device.index)
        cfg = self._ensure_packed(device)
        lib = _lib.lib()
        batch = latent.shape[0]
        n_layers = self.log_size - 2
        _expect_shape(latent, (batch, self.n_latent, self.style_dim), "Generator latent")

        # which layers execute -- mirror of the reference loop (model.py:534-557)
        run = [start_layer == 0] + [False] * n_layers
        if end_layer != 0:
            for k in range(1, n_layers + 1):
                if k < start_layer:
                    continue
                if k == start_layer:
                    run[k] = True
                    continue
                if k > end_layer:
                    break
                run[k] = True
        if not any(run):
            raise RuntimeError(f"Generator: start_layer={start_layer}, end_layer={end_layer} executes nothing")
        last = max(k for k in range(n_layers + 1) if run[k])
        early = last < n_layers

        # noise: explicit list, registered buffers, or fresh draws in reference order (model.py:497-503, :288-291)
        if noise is None:
            noise = [None] * self.num_layers if randomize_noise else \
                [getattr(self.noises, f"noise_{i}") for i in range(self.num_layers)]
        lat = _f32c(latent)
        io = _lib.hf_gen_io()
        io.batch, io.latent = batch, lat.data_ptr()
        keep = [lat]
        for k in range(n_layers + 1):
            if not run[k]:
                continue
            for i in ([0] if k == 0 else [2 * k - 1, 2 * k]):
                nz = noise[i]
                if nz is None:
                    r = 4 if i == 0 else 2 ** ((i + 1) // 2 + 2)
                    nz = lat.new_empty(batch, 1, r, r).normal_()
                r = 4 if i == 0 else 2 ** ((i + 1) // 2 + 2)
                if nz.dim() != 4 or nz.shape[0] not in (1, batch):
                    raise RuntimeError(f"noise[{i}]: expected [1|{batch}, 1, {r}, {r}], got {list(nz.shape)}")
                _expect_shape(nz, (None, 1, r, r), f"Generator noise[{i}]")
                nz = _f32c(nz)
                keep.append(nz)
                io.noise[i], io.noise_batch[i] = nz.data_ptr(), nz.shape[0]
        io.start_layer, io.end_layer = start_layer, end_layer
        if start_layer > 0:
            if layer_in is None:
                raise RuntimeError("Generator: start_layer > 0 needs layer_in (reference model.py:546)")
            r_in = 4 * 2 ** (start_layer - 1)           # the input of layer k is the output of layer k-1
            _expect_shape(layer_in, (batch, self.channels[r_in], r_in, r_in), "Generator layer_in")
            li = _f32c(layer_in)
            keep.append(li)
            io.layer_in = li.data_ptr()
            if skip is not None:
                _expect_shape(skip, (batch, 3, r_in, r_in), "Generator skip")
                sk = _f32c(skip)
                keep.append(sk)
                io.skip_in = sk.data_ptr()
        res_last = 4 * 2 ** last
        out_rgb = torch.empty(batch, 3, res_last, res_last, device=device, dtype=torch.float32)
        io.out_rgb = out_rgb.data_ptr()
        out_feat = None
        if early:
            out_feat = torch.empty(batch, self.channels[res_last], res_last, res_last, device=device,
                                   dtype=torch.float32)
            io.out_feature = out_feat.data_ptr()
        # FeatureStyleEncoder generator variant: insert_feature / return_features
        io.feature_alpha = float(feature_scale)
        if features_in is not None:
            for i, f in enumerate(features_in):
                if f is None or i == 0 or i >= self.num_layers:
                    continue
                if float(feature_scale) != 1.0:
                    raise RuntimeError("Generator: insert_feature is implemented for feature_scale == 1.0 only "
                                       "(HairFast always runs min(1, 1e-4 * 1e5) = 1.0)")
                # features_in[i] replaces the INPUT of the conv at latent index i (FSE model.py:527-560): the output
                # of styled conv i-1, resolution 4 * 2^(i // 2)
                r_f = 4 * 2 ** (i // 2)
                _expect_shape(f, (batch, self.channels[r_f], r_f, r_f), f"Generator features_in[{i}]")
                ff = _f32c(f)
                keep.append(ff)
                io.feature_in[i] = ff.data_ptr()
        outs = None
        if return_features:
            outs = [torch.empty(batch, self.channels[4], 4, 4, device=device, dtype=torch.float32)]
            io.features_out[0] = outs[0].data_ptr()
            for k in range(n_layers + 1):
                for i in ([0] if k == 0 else [2 * k - 1, 2 * k]):
                    r = 4 * 2 ** k
                    t = torch.empty(batch, self.channels[r], r, r, device=device, dtype=torch.float32) if run[k] else None
                    outs.append(t)
                    if t is not None:
                        io.features_out[i + 1] = t.data_ptr()
        ws = self._get_workspace(cfg, batch, device)
        flag = C.c_int(0)
        _lib.check(lib.hf_generator_forward(C.byref(cfg), self._packed.data_ptr(), C.byref(io), ws.data_ptr(),
                                            C.byref(flag), _lib.stream_ptr()), "hf_generator_forward")
        return early, out_feat, out_rgb, outs

"""SEAN's ``decode_sean`` (models/sean_codes/models/pix2pix_model.py:309-325) and ``encode_sean`` (:299-306) on the
sm_90a kernels.

``decode_sean(sean_model, image_code, target_mask)`` has the reference's signature and result ([3,256,256] fp32 on the
device of ``target_mask``).  It runs the UI_mode forward of ``sean_model.netG`` (``SPADEGenerator``,
models/sean_codes/models/networks/generator.py:72-109) batch 1:

* the one-hot convolutions (``fc``, every ``SPADE.mlp_shared``) are table lookups (``hf_sean_onehot_conv``);
* each ACE's style convolutions ``conv_gamma`` / ``conv_beta`` over the piecewise-constant ``middle_avg`` become
  per-call tables ``T[j][tap] = W[:, :, tap] . mu_j`` of the 19 class vectors (``hf_sean_style_tables``), gathered over
  the 3x3 taps of the label map by ``hf_sean_ace_apply``, which also applies the BatchNorm, the noise, the blend and
  the block's leaky ReLU;
* ``mlp_gamma || mlp_beta`` (one 128 -> 2C convolution), ``conv_0``, ``conv_1`` (+ the shortcut as residual) and
  ``conv_s`` run on the wgmma convolution (``hf_conv2d_forward``); spectral norm and the ACE blend weights are folded
  into the packed weights.

No host synchronisation except one read of the out-of-range label count.  The 18 noise tensors are drawn with
``torch.randn(1, R, R, 1)`` in the reference's order (per block ace_s, ace_0, ace_1), so the RNG stream after the
call is the reference's; ``noise=`` injects explicit draws instead.  The Zencoder pass UI_mode runs on an empty
placeholder batch has no effect and is skipped.  Activations are 16-bit NHWC in the encoder family's type
(``nn16.default_dtype``, fp16 unless HAIRFAST_ENC_DTYPE / HAIRFAST_DTYPE say bf16).

``encode_sean(sean_model, images, labels)`` runs ``sean_model.netG.Zencoder`` (architecture.py:154-207) for a batch:
reflection pads (``hf_reflect_pad1_nhwc16``) in front of the prepadded 3x3 convolutions, the two stride-2
convolutions, the ConvTranspose2d in its four-parity form, all on the wgmma convolution; InstanceNorm + LeakyReLU
(``hf_instance_norm_lrelu_nhwc16``); tanh and the per-class means over the nearest 128^2 label map
(``hf_sean_class_means``).  The biases of the four convolutions in front of an InstanceNorm cancel in it and are not
applied.  One host synchronisation: the read of the out-of-range label count.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import _lib, nn16, packcache

N_CLASSES = 19
STYLE = 512
SIZE = 256
# (name, fin, fout, resolution, use_rgb) of SPADEGenerator with ngf 64, num_upsampling_layers 'normal'
# (generator.py:35-43, 83-101); a nearest 2x upsample precedes every block but head_0 and G_middle_1
BLOCKS = [("head_0", 1024, 1024, 8, True), ("G_middle_0", 1024, 1024, 16, True), ("G_middle_1", 1024, 1024, 16, True),
          ("up_0", 1024, 512, 32, True), ("up_1", 512, 256, 64, True), ("up_2", 256, 128, 128, True),
          ("up_3", 128, 64, 256, False)]
UPSAMPLE_BEFORE = {"G_middle_0", "up_0", "up_1", "up_2", "up_3"}
LEVELS = [8, 16, 32, 64, 128, 256]           # label maps hf_sean_labels writes, in order
# the SEAN_OPT HairFast builds (pix2pix_model.py:328-339); anything else raises NotImplementedError
SUPPORTED_OPT = {"ngf": 64, "label_nc": 19, "semantic_nc": 19, "crop_size": 256, "aspect_ratio": 1.0,
                 "num_upsampling_layers": "normal", "norm_G": "spectralspadesyncbatch3x3", "no_instance": True,
                 "contain_dontcare_label": False}

_mean_codes_cache = {}
MAP_SIZE = sum(r * r for r in LEVELS)                        # int8 entries hf_sean_labels writes per sample
CODE_RES = 128                                               # the Zencoder's code map (architecture.py:178-181)
MAP_OFFSET_128 = sum(r * r for r in LEVELS[:LEVELS.index(CODE_RES)])
# Zencoder(3, 512, ngf 32, n_downsampling 2) (architecture.py:154-175, pix2pix SEAN_OPT): state_dict key -> shape.
# model.10 is the ConvTranspose2d(128, 256) (weight [cin, cout, 3, 3]); the InstanceNorms have no parameters.
ZENCODER_SHAPES = {"model.1.weight": (32, 3, 3, 3), "model.1.bias": (32,), "model.4.weight": (64, 32, 3, 3),
                   "model.4.bias": (64,), "model.7.weight": (128, 64, 3, 3), "model.7.bias": (128,),
                   "model.10.weight": (128, 256, 3, 3), "model.10.bias": (256,), "model.14.weight": (512, 256, 3, 3),
                   "model.14.bias": (512,)}


def check_opt(opt) -> None:
    for k, v in SUPPORTED_OPT.items():
        if getattr(opt, k, None) != v:
            raise NotImplementedError(f"decode_sean: SEAN option {k}={getattr(opt, k, None)!r} is not supported "
                                      f"(only HairFast's SEAN_OPT: {k}={v!r})")


def _spectral(conv) -> torch.Tensor:
    """Weight of a spectral-norm conv in eval mode: weight_orig / (u . W v) (no power iteration)."""
    if not hasattr(conv, "weight_orig"):
        return conv.weight.detach().float()
    w = conv.weight_orig.detach().float()
    sigma = torch.dot(conv.weight_u.detach().float(), w.reshape(w.shape[0], -1) @ conv.weight_v.detach().float())
    return w / sigma


def _onehot_table(weight: torch.Tensor) -> torch.Tensor:
    """[Cout,19,3,3] -> [9][19][Cout] (tap = ky*3 + kx)."""
    w = weight.detach().float()
    return w.permute(2, 3, 1, 0).reshape(9, w.shape[1], w.shape[0]).contiguous()


class _PackedACE:
    def __init__(self, ace, use_rgb: bool, dtype: int):
        bn = ace.param_free_norm
        self.bn_scale = (1.0 / torch.sqrt(bn.running_var.detach().float() + bn.eps)).contiguous()
        self.bn_shift = (-bn.running_mean.detach().float() * self.bn_scale).contiguous()
        self.noise_var = ace.noise_var.detach().float().contiguous()
        self.C = self.noise_var.numel()
        sp = ace.Spade
        self.hidden_table = _onehot_table(sp.mlp_shared[0].weight)
        self.hidden_bias = sp.mlp_shared[0].bias.detach().float().contiguous()
        wg, wb = sp.mlp_gamma.weight.detach().float(), sp.mlp_beta.weight.detach().float()
        bg, bb = sp.mlp_gamma.bias.detach().float(), sp.mlp_beta.bias.detach().float()
        self.use_rgb = use_rgb
        if use_rgb:
            # gamma = a_g * gamma_avg + (1 - a_g) * gamma_spade (normalization.py:177-181): the blend weights go into the
            # SPADE conv weights and the style tables' weights; both biases into the SPADE conv's epilogue shift
            ag = torch.sigmoid(ace.blending_gamma.detach().float())
            ab = torch.sigmoid(ace.blending_beta.detach().float())
            wg, wb = wg * (1 - ag), wb * (1 - ab)
            bg = bg * (1 - ag) + ace.conv_gamma.bias.detach().float() * ag
            bb = bb * (1 - ab) + ace.conv_beta.bias.detach().float() * ab
            tw = torch.cat([ace.conv_gamma.weight.detach().float() * ag, ace.conv_beta.weight.detach().float() * ab])
            self.tw = tw.permute(2, 3, 0, 1).reshape(9 * 2 * self.C, STYLE).contiguous()     # row tap*2C + n
            self.fc_w = torch.stack([getattr(ace, f"fc_mu{j}").weight.detach().float()
                                     for j in range(N_CLASSES)]).contiguous()
            self.fc_b = torch.stack([getattr(ace, f"fc_mu{j}").bias.detach().float()
                                     for j in range(N_CLASSES)]).contiguous()
        self.spade_conv = nn16.PackedConv2d(torch.cat([wg, wb]), dtype=dtype)
        self.spade_shift = torch.cat([bg, bb]).contiguous()


class _PackedBlock:
    def __init__(self, blk, name, fin, fout, res, use_rgb, dtype):
        self.name, self.fin, self.fout, self.res = name, fin, fout, res
        self.learned = fin != fout
        self.ace_s = _PackedACE(blk.ace_s, use_rgb, dtype) if self.learned else None
        self.ace_0 = _PackedACE(blk.ace_0, use_rgb, dtype)
        self.ace_1 = _PackedACE(blk.ace_1, use_rgb, dtype)
        self.conv_0 = nn16.PackedConv2d(_spectral(blk.conv_0), dtype=dtype)
        self.b0 = blk.conv_0.bias.detach().float().contiguous()
        self.conv_1 = nn16.PackedConv2d(_spectral(blk.conv_1), dtype=dtype)
        self.b1 = blk.conv_1.bias.detach().float().contiguous()
        self.conv_s = nn16.PackedConv2d(_spectral(blk.conv_s), dtype=dtype) if self.learned else None

    def aces(self):
        return ([self.ace_s] if self.learned else []) + [self.ace_0, self.ace_1]


class PackedSEAN:
    """SPADEGenerator parameters in the kernels' layouts (once per parameter version)."""

    def __init__(self, netG, dtype: Optional[int] = None):
        self.dtype = nn16.default_dtype() if dtype is None else dtype
        self.device = netG.fc.weight.device
        if self.device.type != "cuda":
            raise RuntimeError("decode_sean: the SEAN model must be on a CUDA device (no CPU fallback)")
        check_opt(netG.opt)
        _lib.use_device(self.device.index)
        self.fc_table = _onehot_table(netG.fc.weight)
        self.fc_bias = netG.fc.bias.detach().float().contiguous()
        self.blocks = [_PackedBlock(getattr(netG, n), n, fi, fo, r, rgb, self.dtype) for n, fi, fo, r, rgb in BLOCKS]
        self.img_w = netG.conv_img.weight.detach().float().contiguous()
        self.img_b = netG.conv_img.bias.detach().float().contiguous()
        self.rgb_aces = [a for b in self.blocks for a in b.aces() if a.use_rgb]
        self.n_noise = sum(len(b.aces()) for b in self.blocks)


def _pack(netG) -> PackedSEAN:
    dt = nn16.default_dtype()
    return packcache.get(netG, "_hf_sean_pack", (netG,), dt, lambda: PackedSEAN(netG, dt))[0]


def mean_style_codes(device) -> torch.Tensor:
    """The reference's mean style codes (load_average_feature, pix2pix_model.py:274-290) as [19,512] fp32 on
    `device`, loaded once per process."""
    key = str(device)
    if key not in _mean_codes_cache:
        import importlib
        ref = importlib.import_module("models.sean_codes.models.pix2pix_model")
        d = ref.load_average_feature()
        _mean_codes_cache[key] = torch.stack([d[str(j)]["ACE"].float().reshape(STYLE).to(device)
                                              for j in range(N_CLASSES)]).contiguous()
    return _mean_codes_cache[key]


def draw_noise(device, order: Sequence[int]) -> List[torch.Tensor]:
    """The 18 ``torch.randn(1, W, H, 1)`` draws of the ACE layers (normalization.py:111), in order."""
    return [torch.randn(1, r, r, 1, device=device) for r in order]


def noise_resolutions() -> List[int]:
    return [res for _, fin, fout, res, _ in BLOCKS for _ in range(3 if fin != fout else 2)]


class PackedZencoder:
    """Zencoder parameters in the kernels' layouts (once per parameter version)."""

    def __init__(self, zenc, dtype: Optional[int] = None):
        sd = zenc.state_dict()
        got = {k: tuple(v.shape) for k, v in sd.items()}
        if got != ZENCODER_SHAPES:
            raise NotImplementedError(f"encode_sean: only HairFast's Zencoder(3, 512, ngf 32, n_downsampling 2) is "
                                      f"supported; its parameters are {ZENCODER_SHAPES}, got {got}")
        self.dtype = nn16.default_dtype() if dtype is None else dtype
        self.device = sd["model.1.weight"].device
        if self.device.type != "cuda":
            raise RuntimeError("encode_sean: the SEAN model must be on a CUDA device (no CPU fallback)")
        _lib.use_device(self.device.index)
        w = lambda i: sd[f"model.{i}.weight"].float()
        dt = self.dtype
        # the biases of model.1 / 4 / 7 / 10 are constant per channel and cancel in the InstanceNorm that follows
        self.conv1 = nn16.PackedConv2d(w(1), cin_pad=32, prepadded=True, dtype=dt)
        self.conv4 = nn16.PackedConv2d(w(4), stride=2, dtype=dt)
        self.conv7 = nn16.PackedConv2d(w(7), stride=2, dtype=dt)
        self.conv10 = nn16.PackedConv2d(w(10), stride=2, transposed=True, dtype=dt)
        self.conv14 = nn16.PackedConv2d(w(14), prepadded=True, dtype=dt)
        self.bias14 = sd["model.14.bias"].float().contiguous()


def _pack_zencoder(zenc) -> PackedZencoder:
    dt = nn16.default_dtype()
    return packcache.get(zenc, "_hf_zencoder_pack", (zenc,), dt, lambda: PackedZencoder(zenc, dt))[0]


# ------------------------------------------------------------------------------------------------ kernel wrappers
def label_maps(target_mask: torch.Tensor) -> List[torch.Tensor]:
    """[1,1,256,256] labels -> int8 maps at 8..256.  Raises ValueError for labels outside 0..18."""
    if target_mask.dim() != 4 or tuple(target_mask.shape[:2]) != (1, 1) or tuple(target_mask.shape[2:]) != (SIZE, SIZE):
        raise NotImplementedError(f"decode_sean: target_mask must be [1,1,{SIZE},{SIZE}], got {list(target_mask.shape)}")
    lab = target_mask.reshape(SIZE, SIZE).long().contiguous()       # preprocess_input's .long() (pix2pix_model.py:126)
    maps = torch.empty(sum(r * r for r in LEVELS), dtype=torch.int8, device=lab.device)
    bad = torch.empty(1, dtype=torch.int32, device=lab.device)
    _lib.check(_lib.lib().hf_sean_labels(lab.data_ptr(), maps.data_ptr(), bad.data_ptr(), SIZE, _lib.stream_ptr()),
               "hf_sean_labels")
    n_bad = int(bad.item())
    if n_bad:
        raise ValueError(f"decode_sean: {n_bad} labels of target_mask are outside 0..{N_CLASSES - 1}")
    out, off = [], 0
    for r in LEVELS:
        out.append(maps[off: off + r * r].view(r, r))
        off += r * r
    return out


def onehot_conv(L: torch.Tensor, table: torch.Tensor, bias: Optional[torch.Tensor], relu: bool, dtype: int):
    r, cout = L.shape[0], table.shape[-1]
    y = torch.empty(1, r, r, cout, device=L.device, dtype=nn16.torch_dtype(dtype))
    _lib.check(_lib.lib().hf_sean_onehot_conv(L.data_ptr(), table.data_ptr(), nn16._p(bias), 3 if relu else 0,
                                              y.data_ptr(), r, cout, dtype, _lib.stream_ptr()), "hf_sean_onehot_conv")
    return y


def style_tables(aces: Sequence[_PackedACE], image_code: torch.Tensor, mean_codes: torch.Tensor) -> List[torch.Tensor]:
    """Per-call [19][9][2C] tables of every ACE that uses the style codes (two launches)."""
    dev = image_code.device
    ic = image_code.detach().reshape(N_CLASSES, STYLE).float().contiguous()
    tables = [torch.empty(N_CLASSES, 9, 2 * a.C, device=dev, dtype=torch.float32) for a in aces]
    arr = (_lib.hf_sean_ace_tables * len(aces))()
    for i, (a, t) in enumerate(zip(aces, tables)):
        arr[i] = _lib.hf_sean_ace_tables(a.fc_w.data_ptr(), a.fc_b.data_ptr(), a.tw.data_ptr(), t.data_ptr(), 2 * a.C)
    mu = torch.empty(len(aces), N_CLASSES, STYLE, device=dev, dtype=torch.float32)
    _lib.check(_lib.lib().hf_sean_style_tables(ic.data_ptr(), mean_codes.data_ptr(), arr, len(aces), mu.data_ptr(),
                                               _lib.stream_ptr()), "hf_sean_style_tables")
    return tables


def ace_apply(x16, noise, a: _PackedACE, gamma_beta, table, L, lrelu: bool, dtype: int):
    _, r, _, c = x16.shape
    y = torch.empty_like(x16)
    _lib.check(_lib.lib().hf_sean_ace_apply(x16.data_ptr(), noise.data_ptr(), a.noise_var.data_ptr(),
                                            a.bn_scale.data_ptr(), a.bn_shift.data_ptr(), gamma_beta.data_ptr(),
                                            nn16._p(table), L.data_ptr(), 1 if lrelu else 0, y.data_ptr(), r, c, dtype,
                                            _lib.stream_ptr()), "hf_sean_ace_apply")
    return y


def conv_img(x16, w, b, dtype: int):
    _, r, _, c = x16.shape
    y = torch.empty(3, r, r, device=x16.device, dtype=torch.float32)
    _lib.check(_lib.lib().hf_sean_conv_img(x16.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), r, c, dtype,
                                           _lib.stream_ptr()), "hf_sean_conv_img")
    return y


# ------------------------------------------------------------------------------------------------ forward
def _ace(pk: PackedSEAN, a: _PackedACE, x16, L, noise, table, lrelu: bool):
    hidden = onehot_conv(L, a.hidden_table, a.hidden_bias, True, pk.dtype)               # SPADE.mlp_shared + ReLU
    _, _, gb = a.spade_conv(hidden, shift=a.spade_shift, want_y16=False, want_y32=True)  # gamma_spade || beta_spade
    return ace_apply(x16, noise.reshape(-1).float().contiguous(), a, gb, table, L, lrelu, pk.dtype)


@torch.no_grad()
def run_packed(pk: PackedSEAN, image_code: torch.Tensor, target_mask: torch.Tensor, mean_codes: torch.Tensor,
               noise: Sequence[torch.Tensor], taps: Optional[dict] = None) -> torch.Tensor:
    maps = dict(zip(LEVELS, label_maps(target_mask)))
    tables = iter(style_tables(pk.rgb_aces, image_code, mean_codes))
    it = iter(noise)
    x = onehot_conv(maps[8], pk.fc_table, pk.fc_bias, False, pk.dtype)               # fc (generator.py:75-76)
    for blk in pk.blocks:
        if blk.name in UPSAMPLE_BEFORE:
            x = nn16.gate_add_up(x, up=2, dtype=pk.dtype)                             # nn.Upsample(scale_factor=2)
        x = run_block(pk, blk, x, maps[blk.res], it, tables)
        if taps is not None:
            taps[blk.name] = x
    return conv_img(x, pk.img_w, pk.img_b, pk.dtype)


def run_block(pk: PackedSEAN, blk: _PackedBlock, x, L, noise_iter, table_iter):
    """SPADEResnetBlock.forward (architecture.py:69-96) on [1,R,R,fin] 16-bit NHWC; consumes the block's noise tensors
    and style tables from the two iterators."""
    if blk.learned:
        a = _ace(pk, blk.ace_s, x, L, next(noise_iter), next(table_iter) if blk.ace_s.use_rgb else None, False)
        xs, _, _ = blk.conv_s(a)
    else:
        xs = x
    d = _ace(pk, blk.ace_0, x, L, next(noise_iter), next(table_iter) if blk.ace_0.use_rgb else None, True)
    d, _, _ = blk.conv_0(d, shift=blk.b0)
    d = _ace(pk, blk.ace_1, d, L, next(noise_iter), next(table_iter) if blk.ace_1.use_rgb else None, True)
    x, _, _ = blk.conv_1(d, shift=blk.b1, residual16=xs)
    return x


# ------------------------------------------------------------------------------------------------ encode
def batch_label_maps(labels: torch.Tensor):
    """[B,1,256,256] labels -> (int8 maps [B, MAP_SIZE] (hf_sean_labels per sample), out-of-range counts [B] int32)."""
    b = labels.shape[0]
    lab = labels.reshape(b, SIZE, SIZE).long().contiguous()         # preprocess_input's .long() (pix2pix_model.py:126)
    maps = torch.empty(b, MAP_SIZE, dtype=torch.int8, device=lab.device)
    bad = torch.empty(b, dtype=torch.int32, device=lab.device)
    for i in range(b):
        _lib.check(_lib.lib().hf_sean_labels(lab[i].data_ptr(), maps[i].data_ptr(), bad[i:].data_ptr(), SIZE,
                                             _lib.stream_ptr()), "hf_sean_labels")
    return maps, bad


def class_means(y32: torch.Tensor, maps: torch.Tensor) -> torch.Tensor:
    """tanh + per-class means of the last conv's [B,512,128,128] fp32 output over the 128^2 label maps: [B,19,512]."""
    b, c, h, w = y32.shape
    codes = torch.empty(b, N_CLASSES, c, device=y32.device, dtype=torch.float32)
    _lib.check(_lib.lib().hf_sean_class_means(y32.data_ptr(), maps[:, MAP_OFFSET_128:].data_ptr(), MAP_SIZE,
                                              codes.data_ptr(), b, c, h * w, _lib.stream_ptr()), "hf_sean_class_means")
    return codes


@torch.no_grad()
def run_zencoder(pk: PackedZencoder, images: torch.Tensor, maps: torch.Tensor, taps: Optional[dict] = None):
    """Zencoder.forward (architecture.py:177-207) on [B,3,256,256] images and hf_sean_labels maps -> [B,19,512].
    ``taps`` receives the four InstanceNorm + LeakyReLU outputs (16-bit NHWC) and the pre-tanh conv (fp32 NCHW)."""
    dt = pk.dtype
    x = nn16.reflect_pad1(nn16.to_nhwc16(images, c_pad=32, dtype=dt), dt)             # ReflectionPad2d(1) (:159)
    for i, conv in enumerate((pk.conv1, pk.conv4, pk.conv7, pk.conv10)):
        x, _, _ = conv(x)
        x = nn16.instance_norm_lrelu(x, 0.2, dt)
        if taps is not None:
            taps[f"in{i + 1}"] = x
    _, _, y32 = pk.conv14(nn16.reflect_pad1(x, dt), shift=pk.bias14, want_y16=False, want_y32=True)
    if taps is not None:
        taps["pre_tanh"] = y32
    return class_means(y32, maps)


def encode_sean(sean_model, images, labels):
    """Drop-in for models.sean_codes.models.pix2pix_model.encode_sean: [B,19,512] fp32 style codes on images'
    device.  Raises ValueError for labels outside 0..18."""
    zenc = sean_model.netG.Zencoder
    if not images.is_cuda or not labels.is_cuda:
        raise RuntimeError("encode_sean: images and labels must be CUDA tensors (no CPU fallback)")
    if (images.dim() != 4 or labels.dim() != 4 or images.shape[0] < 1 or tuple(images.shape[1:]) != (3, SIZE, SIZE)
            or tuple(labels.shape) != (images.shape[0], 1, SIZE, SIZE)):
        raise NotImplementedError(f"encode_sean: images must be [B,3,{SIZE},{SIZE}] and labels [B,1,{SIZE},{SIZE}], "
                                  f"got {list(images.shape)} and {list(labels.shape)}")
    pk = _pack_zencoder(zenc)
    _lib.use_device(images.device.index)
    maps, bad = batch_label_maps(labels)
    codes = run_zencoder(pk, images, maps)
    n_bad = int(bad.sum().item())
    if n_bad:
        raise ValueError(f"encode_sean: {n_bad} labels are outside 0..{N_CLASSES - 1}")
    return codes


# ------------------------------------------------------------------------------------------------ decode
def decode_sean(sean_model, image_code, target_mask, noise: Optional[Sequence[torch.Tensor]] = None,
                mean_codes: Optional[torch.Tensor] = None):
    """Drop-in for models.sean_codes.models.pix2pix_model.decode_sean: [3,256,256] fp32 on target_mask's device.
    ``noise``: explicit ACE noise ([1,R,R,1] each, draw order) instead of 18 fresh ``torch.randn`` draws;
    ``mean_codes``: [19,512] instead of the reference's mean style codes."""
    netG = sean_model.netG
    check_opt(sean_model.opt)
    if not target_mask.is_cuda or not image_code.is_cuda:
        raise RuntimeError("decode_sean: image_code and target_mask must be CUDA tensors (no CPU fallback)")
    if image_code.dim() != 3 or image_code.shape[1:] != (N_CLASSES, STYLE):
        raise NotImplementedError(f"decode_sean: image_code must be [1,19,512], got {list(image_code.shape)}")
    dev = target_mask.device
    pk = _pack(netG)
    if mean_codes is None:
        mean_codes = mean_style_codes(dev)
    mean_codes = mean_codes.to(dev).float().contiguous()
    if noise is None:
        noise = draw_noise(dev, noise_resolutions())
    elif len(noise) != pk.n_noise:
        raise ValueError(f"decode_sean: {pk.n_noise} noise tensors expected, got {len(noise)}")
    return run_packed(pk, image_code, target_mask, mean_codes, noise)

"""CtrlHair's shape adaptor (``Alignment.mask_generator``, the ``Generator`` of models/CtrlHair/shape_branch/model.py:
146-199, config 054) on the sm_90a kernels: drop-in ``get_hair_face_code`` and ``get_new_shape``
(shape_branch/solver.py:248-262) with the reference's signatures and results.

Per MaskEncoder (7 x [ZeroPad 1, Conv 4x4 stride 2, LayerNorm, LeakyReLU 0.2], flatten, Linear):

* layer 0 is a lookup (``hf_shape_onehot_s2``): the mask channels are one-hot, so their conv is a gather of one weight
  column per tap, and the conv of the 40 positional channels plus the bias is an input-independent map computed when
  packing (in float64, stored fp32);
* layers 1-6 and the Linear head run on the split-K GEMM (``hf_shape_gemm``) with compact 16-bit weights and the
  im2col gathered from the small NHWC input.

Per MaskDecoder (Linear -> [2048,2,2], 7 x [nearest 2x, Conv 3x3, LayerNorm, LeakyReLU 0.2], Conv 3x3):

* the Linear and layers 0-2 (4^2 .. 16^2 outputs, up to 75 MB of weights) run on the split-K GEMM, the upsample folded
  into its gather;
* layers 3-6 (32^2 .. 256^2) run on the wgmma convolution (``hf_conv2d_forward``) after a nearest upsample
  (``hf_gate_add_up_nhwc16``);
* both out_layers and the argmax over the 19 logits are one kernel (``hf_shape_logits_argmax``); the softmax in front
  of the argmax is monotone and is not computed.

The CtrlHair LayerNorm (whole-sample mean and unbiased std, then per-channel gamma / beta) is
``hf_shape_layer_norm_lrelu``.  Activations are 16-bit NHWC in the encoder family's type (``nn16.default_dtype``).
Networks are packed by state-dict key, each on its own (``get_new_shape`` never packs the encoders), and re-packed by
the rule of ``packcache``.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from . import _lib, nn16, packcache

N_CLASSES = 19
HAIR_IDX = 13                  # HAIR_IDX (models/CtrlHair/global_value_utils.py:52)
SIZE = 256
HAIR_DIM, FACE_DIM = 16, 1024
POS_CHANNELS = 40              # pos_encoding_order 10: sin and cos of 10 frequencies of 2 coordinates
ENC_CH = [32, 64, 128, 256, 512, 1024, 2048]       # MaskEncoder layer outputs, 128^2 .. 2^2
DEC_CH = [2048, 1024, 512, 256, 128, 64, 32]       # MaskDecoder layer outputs, 4^2 .. 256^2
DEC_GEMM_LAYERS = 3            # decoder layers 0..2 on the split-K GEMM, the rest on the wgmma convolution
SLOPE = 0.2
GEMM_1X1, GEMM_S2, GEMM_UP = 0, 1, 2               # hf_shape_gemm modes


def encoder_shapes(n_mask: int, out_dim: int, vae: bool) -> dict:
    """state_dict key -> shape of MaskEncoder(n_mask, out_dim, 'ln', 7, vae_mode=vae) (model.py:68-97)."""
    d, cin = {}, n_mask + POS_CHANNELS
    for i, c in enumerate(ENC_CH):
        d.update({f"layers.{i}.conv.weight": (c, cin, 4, 4), f"layers.{i}.conv.bias": (c,),
                  f"layers.{i}.norm.gamma": (c,), f"layers.{i}.norm.beta": (c,)})
        cin = c
    heads = ["out_layer", "std_out_layer"] if vae else ["out_layer"]
    for h in heads:
        d.update({f"{h}.fc.weight": (out_dim, 4 * ENC_CH[-1]), f"{h}.fc.bias": (out_dim,)})
    return d


def decoder_shapes(in_dim: int, n_out: int) -> dict:
    """state_dict key -> shape of MaskDecoder(in_dim, n_out, 'ln', 7) (model.py:119-143)."""
    d = {"in_layer.fc.weight": (4 * DEC_CH[0], in_dim), "in_layer.fc.bias": (4 * DEC_CH[0],)}
    cin = DEC_CH[0]
    for i, c in enumerate(DEC_CH):
        j = 2 * i + 1                                  # nn.Upsample at the even indices of the Sequential
        d.update({f"layers.{j}.conv.weight": (c, cin, 3, 3), f"layers.{j}.conv.bias": (c,),
                  f"layers.{j}.norm.gamma": (c,), f"layers.{j}.norm.beta": (c,)})
        cin = c
    d.update({"out_layer.conv.weight": (n_out, cin, 3, 3), "out_layer.conv.bias": (n_out,)})
    return d


NETWORK_SHAPES = {"hair_encoder": encoder_shapes(1, HAIR_DIM, True),
                  "face_encoder": encoder_shapes(N_CLASSES - 1, FACE_DIM, False),
                  "hair_decoder": decoder_shapes(FACE_DIM + HAIR_DIM, 1),
                  "face_decoder": decoder_shapes(FACE_DIM, N_CLASSES - 1)}


def _state(net, name: str) -> dict:
    sd = net.state_dict()
    got = {k: tuple(v.shape) for k, v in sd.items()}
    if got != NETWORK_SHAPES[name]:
        raise NotImplementedError(f"shape adaptor: only CtrlHair's config 054 mask generator is supported; its {name} "
                                  f"parameters are {NETWORK_SHAPES[name]}, got {got}")
    dev = next(iter(sd.values())).device
    if dev.type != "cuda":
        raise RuntimeError("shape adaptor: the mask generator must be on a CUDA device (no CPU fallback)")
    _lib.use_device(dev.index)
    return {k: v.detach().float() for k, v in sd.items()}


def _w16(w: torch.Tensor, dtype: int) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> compact [Cout, kh*kw*Cin] 16-bit (k = tap * Cin + c)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(nn16.torch_dtype(dtype)).contiguous()


def onehot_table(w0: torch.Tensor, hair: bool) -> torch.Tensor:
    """Layer-0 weights of the mask channels as [16 taps][20 labels][32] fp32: label j's column of the one-hot input,
    zero for the labels the encoder does not see (hair: all but 13; face: 13) and for 19 (255 in the mask)."""
    n_mask = 1 if hair else N_CLASSES - 1
    cout = w0.shape[0]
    table = torch.zeros(16, N_CLASSES + 1, cout, device=w0.device, dtype=torch.float32)
    labels = [HAIR_IDX] if hair else [j for j in range(N_CLASSES) if j != HAIR_IDX]   # split_hair_face's channels
    table[:, labels] = w0[:, :n_mask].permute(2, 3, 1, 0).reshape(16, n_mask, cout).float()
    return table.contiguous()


def positional_map(w0: torch.Tensor, b0: torch.Tensor, pos: torch.Tensor, n_mask: int) -> torch.Tensor:
    """Conv 4x4 stride 2 (zero pad 1) of the positional channels [40,256,256] plus the bias, in float64:
    [128*128, 32] fp32 (NHWC)."""
    y = F.conv2d(F.pad(pos.double()[None], (1, 1, 1, 1)), w0[:, n_mask:].double(), b0.double(), stride=2)[0]
    return y.permute(1, 2, 0).reshape(-1, w0.shape[0]).float().contiguous()


class PackedEncoder:
    def __init__(self, enc, hair: bool, dtype: int):
        sd = _state(enc, "hair_encoder" if hair else "face_encoder")
        self.dtype, self.hair = dtype, hair
        n_mask = 1 if hair else N_CLASSES - 1
        w0 = sd["layers.0.conv.weight"]
        self.table = onehot_table(w0, hair)
        self.cmap = positional_map(w0, sd["layers.0.conv.bias"], enc.input_embedding[0].to(w0.device), n_mask)
        self.ln = [(sd[f"layers.{i}.norm.gamma"].contiguous(), sd[f"layers.{i}.norm.beta"].contiguous())
                   for i in range(len(ENC_CH))]
        self.convs = [(_w16(sd[f"layers.{i}.conv.weight"], dtype), sd[f"layers.{i}.conv.bias"].contiguous())
                      for i in range(1, len(ENC_CH))]
        # flatten() of NCHW [2048,2,2] reads k = c*4 + pixel; the NHWC input has k = pixel*2048 + c
        fw = sd["out_layer.fc.weight"]
        self.fc_w = fw.view(fw.shape[0], ENC_CH[-1], 4).permute(0, 2, 1).reshape(fw.shape[0], -1)
        self.fc_w = self.fc_w.to(nn16.torch_dtype(dtype)).contiguous()
        self.fc_b = sd["out_layer.fc.bias"].contiguous()


class PackedDecoder:
    def __init__(self, dec, name: str, dtype: int):
        sd = _state(dec, name)
        self.dtype = dtype
        # reshape(-1, 2048, 2, 2) reads output o = c*4 + pixel; rows reordered to pixel*2048 + c (NHWC)
        iw, ib = sd["in_layer.fc.weight"], sd["in_layer.fc.bias"]
        self.in_w = iw.view(DEC_CH[0], 4, -1).permute(1, 0, 2).reshape(4 * DEC_CH[0], -1)
        self.in_w = self.in_w.to(nn16.torch_dtype(dtype)).contiguous()
        self.in_b = ib.view(DEC_CH[0], 4).t().contiguous().reshape(-1)
        self.in_dim = iw.shape[1]
        keys = [f"layers.{2 * i + 1}" for i in range(len(DEC_CH))]
        self.ln = [(sd[k + ".norm.gamma"].contiguous(), sd[k + ".norm.beta"].contiguous()) for k in keys]
        self.bias = [sd[k + ".conv.bias"].contiguous() for k in keys]
        self.gemm_w = [_w16(sd[k + ".conv.weight"], dtype) for k in keys[:DEC_GEMM_LAYERS]]
        self.convs = [nn16.PackedConv2d(sd[k + ".conv.weight"], dtype=dtype) for k in keys[DEC_GEMM_LAYERS:]]
        self.out_w, self.out_b = sd["out_layer.conv.weight"], sd["out_layer.conv.bias"]


class PackedDecoders:
    """Both decoders and the logits table [19][9][32] of their out_layers in cat[face[:13], hair, face[13:]] order."""

    def __init__(self, gen, dtype: int):
        self.hair = PackedDecoder(gen.hair_decoder, "hair_decoder", dtype)
        self.face = PackedDecoder(gen.face_decoder, "face_decoder", dtype)
        w = torch.cat([self.face.out_w[:HAIR_IDX], self.hair.out_w, self.face.out_w[HAIR_IDX:]])
        self.table = w.permute(0, 2, 3, 1).reshape(N_CLASSES, 9, -1).contiguous()
        self.table_bias = torch.cat([self.face.out_b[:HAIR_IDX], self.hair.out_b, self.face.out_b[HAIR_IDX:]]).contiguous()


def pack_encoder(enc, hair: bool) -> PackedEncoder:
    dt = nn16.default_dtype()
    return packcache.get(enc, "_hf_shape_pack", (enc,), dt, lambda: PackedEncoder(enc, hair, dt))[0]


def pack_decoders(gen) -> PackedDecoders:
    dt = nn16.default_dtype()
    return packcache.get(gen, "_hf_shape_decoders_pack", (gen.hair_decoder, gen.face_decoder), dt,
                         lambda: PackedDecoders(gen, dt))[0]


# ------------------------------------------------------------------------------------------------ kernel wrappers
def labels(mask: torch.Tensor):
    """The reference's label handling of a [256,256] mask: ``mask.long()`` (the caller's tensor when it is already
    int64) gets 255 -> 19 in place; returns (int8 labels 0..19, out-of-range count [1] int32 on the device)."""
    lab = mask.long()
    work = lab if lab.is_contiguous() else lab.contiguous()
    L = torch.empty(SIZE, SIZE, dtype=torch.int8, device=mask.device)
    bad = torch.empty(1, dtype=torch.int32, device=mask.device)
    _lib.check(_lib.lib().hf_shape_labels(work.data_ptr(), L.data_ptr(), bad.data_ptr(), SIZE * SIZE,
                                          _lib.stream_ptr()), "hf_shape_labels")
    if work is not lab:
        lab.copy_(work)
    return L, bad


def layer_norm_lrelu(x16: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, dtype: int) -> torch.Tensor:
    """CtrlHair LayerNorm + LeakyReLU(0.2) of one [..., C] 16-bit NHWC sample."""
    c = x16.shape[-1]
    n = x16.numel()
    y = torch.empty_like(x16)
    ws = torch.empty(_lib.lib().hf_shape_layer_norm_workspace_bytes(n), dtype=torch.uint8, device=x16.device)
    _lib.check(_lib.lib().hf_shape_layer_norm_lrelu(x16.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
                                                    ws.data_ptr(), n // c, c, SLOPE, dtype, _lib.stream_ptr()),
               "hf_shape_layer_norm_lrelu")
    return y


def gemm(mode: int, w16: torch.Tensor, x16: torch.Tensor, bias: Optional[torch.Tensor], hin: int, win: int,
         dtype: int, want_y16: bool = True, want_y32: bool = False):
    """hf_shape_gemm of x16 [hin, win, cin] (16-bit NHWC) -> (y16 | None, y32 | None), both [P, cout]."""
    cout = w16.shape[0]
    cin = x16.numel() // (hin * win)
    p = {GEMM_1X1: hin * win, GEMM_S2: hin * win // 4, GEMM_UP: 4 * hin * win}[mode]
    lib = _lib.lib()
    ws = torch.empty(lib.hf_shape_gemm_workspace_bytes(mode, cin, cout, hin, win), dtype=torch.uint8,
                     device=x16.device)
    y16 = torch.empty(p, cout, dtype=nn16.torch_dtype(dtype), device=x16.device) if want_y16 else None
    y32 = torch.empty(p, cout, dtype=torch.float32, device=x16.device) if want_y32 else None
    _lib.check(lib.hf_shape_gemm(mode, w16.data_ptr(), x16.data_ptr(), nn16._p(bias), nn16._p(y32), nn16._p(y16),
                                 ws.data_ptr(), cin, cout, hin, win, dtype, _lib.stream_ptr()), "hf_shape_gemm")
    return y16, y32


# ------------------------------------------------------------------------------------------------ networks
@torch.no_grad()
def run_encoder(pk: PackedEncoder, L: torch.Tensor, taps: Optional[list] = None) -> torch.Tensor:
    """MaskEncoder.forward's mean (model.py:87-97) of the label map: [1, out_dim] fp32.  ``taps`` receives each
    layer's LayerNorm + LeakyReLU output (16-bit NHWC)."""
    dt, r = pk.dtype, SIZE // 2
    x = torch.empty(r, r, ENC_CH[0], dtype=nn16.torch_dtype(dt), device=L.device)
    _lib.check(_lib.lib().hf_shape_onehot_s2(L.data_ptr(), pk.table.data_ptr(), pk.cmap.data_ptr(), x.data_ptr(), r,
                                             ENC_CH[0], dt, _lib.stream_ptr()), "hf_shape_onehot_s2")
    x = layer_norm_lrelu(x, *pk.ln[0], dt)
    if taps is not None:
        taps.append(x)
    for (w, b), ln in zip(pk.convs, pk.ln[1:]):
        x, _ = gemm(GEMM_S2, w, x, b, r, r, dt)
        r //= 2
        x = layer_norm_lrelu(x, *ln, dt)
        if taps is not None:
            taps.append(x.view(r, r, -1))
    _, code = gemm(GEMM_1X1, pk.fc_w, x, pk.fc_b, 1, 1, dt, want_y16=False, want_y32=True)
    return code


@torch.no_grad()
def run_decoder(pk: PackedDecoder, code16: torch.Tensor, taps: Optional[list] = None) -> torch.Tensor:
    """MaskDecoder.forward (model.py:145-150) up to its last LayerNorm + LeakyReLU: [256,256,32] 16-bit NHWC."""
    dt, r = pk.dtype, 2
    x, _ = gemm(GEMM_1X1, pk.in_w, code16, pk.in_b, 1, 1, dt)               # [4, 2048] = [2, 2, 2048] NHWC
    for i, ln in enumerate(pk.ln):
        if i < DEC_GEMM_LAYERS:
            x, _ = gemm(GEMM_UP, pk.gemm_w[i], x, pk.bias[i], r, r, dt)
        else:
            up = nn16.gate_add_up(x.view(1, r, r, -1), up=2, dtype=dt)
            x, _, _ = pk.convs[i - DEC_GEMM_LAYERS](up, shift=pk.bias[i])
        r *= 2
        x = layer_norm_lrelu(x, *ln, dt).view(r, r, -1)
        if taps is not None:
            taps.append(x)
    return x


def logits_argmax(pk: PackedDecoders, hair16: torch.Tensor, face16: torch.Tensor) -> torch.Tensor:
    out = torch.empty(SIZE, SIZE, dtype=torch.int64, device=hair16.device)
    _lib.check(_lib.lib().hf_shape_logits_argmax(hair16.data_ptr(), face16.data_ptr(), pk.table.data_ptr(),
                                                 pk.table_bias.data_ptr(), out.data_ptr(), SIZE, pk.hair.dtype,
                                                 _lib.stream_ptr()), "hf_shape_logits_argmax")
    return out


# ------------------------------------------------------------------------------------------------ drop-ins
def get_hair_face_code(mask_generator, mask):
    """Drop-in for models.CtrlHair.shape_branch.solver.get_hair_face_code: (face_code [1,1024], hair_code [1,16]) fp32
    on the mask's device.  Like the reference, rewrites 255 -> 19 in an int64 ``mask`` and draws the hair encoder's
    discarded ``torch.randn([1, 16])`` from the CPU generator.  Raises ValueError for labels outside {0..19, 255}."""
    if not mask.is_cuda:
        raise RuntimeError("get_hair_face_code: mask must be a CUDA tensor (no CPU fallback)")
    if tuple(mask.shape) != (SIZE, SIZE):
        raise NotImplementedError(f"get_hair_face_code: mask must be [{SIZE},{SIZE}], got {list(mask.shape)}")
    hair_pk = pack_encoder(mask_generator.hair_encoder, True)
    face_pk = pack_encoder(mask_generator.face_encoder, False)
    _lib.use_device(mask.device.index)
    L, bad = labels(mask)
    hair_code = run_encoder(hair_pk, L)
    torch.randn([1, HAIR_DIM])                     # MaskEncoder.vae_resampling (model.py:99-102), result unused
    face_code = run_encoder(face_pk, L)
    n_bad = int(bad.item())
    if n_bad:
        raise ValueError(f"get_hair_face_code: {n_bad} mask labels are outside 0..{N_CLASSES - 1} and 255")
    return face_code, hair_code


def get_new_shape(mask_generator, face_code, new_hair_code):
    """Drop-in for models.CtrlHair.shape_branch.solver.get_new_shape: [256,256] int64 labels on face_code's device."""
    if not face_code.is_cuda or not new_hair_code.is_cuda:
        raise RuntimeError("get_new_shape: face_code and new_hair_code must be CUDA tensors (no CPU fallback)")
    if tuple(face_code.shape) != (1, FACE_DIM) or tuple(new_hair_code.shape) != (1, HAIR_DIM):
        raise NotImplementedError(f"get_new_shape: codes must be [1,{FACE_DIM}] and [1,{HAIR_DIM}], got "
                                  f"{list(face_code.shape)} and {list(new_hair_code.shape)}")
    pk = pack_decoders(mask_generator)
    dt = pk.hair.dtype
    _lib.use_device(face_code.device.index)
    hair_in = nn16.to_nhwc16(torch.cat([face_code, new_hair_code], 1).view(1, -1, 1, 1), dtype=dt)
    face_in = nn16.to_nhwc16(face_code.view(1, -1, 1, 1), dtype=dt)
    hair = run_decoder(pk.hair, hair_in)
    face = run_decoder(pk.face, face_in)
    return logits_argmax(pk, hair, face)

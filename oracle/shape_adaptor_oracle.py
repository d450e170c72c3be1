"""Oracle for CtrlHair's shape adaptor (models/CtrlHair/shape_branch/model.py:146-199, config 054): seeded parameters
for the reference ``Generator``, the label cases of the golden, and float64 restatements of the forms the kernels use
(hairfastgan_b200/shape_adaptor.py): the layer-0 lookup, the stride-2 4x4 and nearest-up 3x3 im2col gathers of the
split-K GEMM, the CtrlHair LayerNorm and the logits argmax.  CPU only; test infrastructure."""
from __future__ import annotations

import torch
import torch.nn.functional as F

N_CLASSES, HAIR_IDX = 19, 13


def reference_generator():
    """The unmodified reference ``Generator(cfg)`` of config 054 on the CPU (needs the reference on sys.path, e.g.
    through baseline.refenv.activate)."""
    from models.CtrlHair.shape_branch.config import cfg
    from models.CtrlHair.shape_branch.model import Generator
    return Generator(cfg).eval()


def config054_shapes() -> dict:
    """state_dict key -> shape of the reference Generator of config 054, in its state_dict order."""
    from hairfastgan_b200.shape_adaptor import NETWORK_SHAPES
    return {f"{net}.{k}": v for net, d in NETWORK_SHAPES.items() for k, v in d.items()}


def synth_params(seed: int) -> dict:
    """Seeded parameters in state_dict order: conv / linear weights N(0, 1/fan_in), biases N(0, 0.05), LayerNorm gamma
    U(0.5, 1.5) and beta N(0, 0.1) (so that the beta path is exercised)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, shape in config054_shapes().items():
        if k.endswith("norm.gamma"):
            t = torch.rand(shape, generator=g) + 0.5
        elif k.endswith("norm.beta"):
            t = torch.randn(shape, generator=g) * 0.1
        elif k.endswith("bias"):
            t = torch.randn(shape, generator=g) * 0.05
        else:
            n = 1
            for d in shape[1:]:
                n *= d
            t = torch.randn(shape, generator=g) / n ** 0.5
        out[k] = t.float()
    return out


def label_cases() -> dict:
    """name -> [256,256] int64 mask."""
    g = torch.Generator().manual_seed(41)
    yy, xx = torch.meshgrid(torch.arange(256), torch.arange(256), indexing="ij")
    face = torch.zeros(256, 256, dtype=torch.int64)
    r2 = (yy - 140) ** 2 + (xx - 128) ** 2
    face[r2 < 90 ** 2] = 1                                           # skin
    face[(r2 < 100 ** 2) & (yy < 110)] = HAIR_IDX                    # hair cap
    face[((yy - 120) ** 2 + (xx - 95) ** 2) < 80] = 4                # eyes
    face[((yy - 120) ** 2 + (xx - 161) ** 2) < 80] = 5
    face[(yy > 180) & (yy < 190) & ((xx - 128).abs() < 25)] = 11     # mouth
    face[yy > 225] = 16                                              # cloth
    allc = torch.randint(0, 19, (16, 16), generator=g)
    allc.view(-1)[:19] = torch.arange(19)
    allc = allc.repeat_interleave(16, 0).repeat_interleave(16, 1)
    nohair = face.clone()
    nohair[nohair == HAIR_IDX] = 0
    hair_only = torch.where(face == HAIR_IDX, face, torch.zeros_like(face))
    some255 = face.clone()
    some255[200:230, 20:90] = 255
    some255[5:9, :] = 255
    odd = nohair.clone()
    odd[41:121:2, 61:181:2] = HAIR_IDX                               # hair at odd rows and columns only
    return {"face": face, "all_classes": allc, "no_hair": nohair, "hair_only": hair_only, "some_255": some255,
            "odd_hair": odd}


# ------------------------------------------------------------------------------------------------ forms, float64
def one_hot_input(mask: torch.Tensor, hair: bool) -> torch.Tensor:
    """mask_label_to_one_hot + split_hair_face (shape_util.py:6-26) of a [256,256] mask: [1, 1 | 18, 256, 256]."""
    m = mask.clone()
    m[m == 255] = 19
    oh = F.one_hot(m, 20).permute(2, 0, 1)[:N_CLASSES].double()[None]
    if hair:
        return oh[:, HAIR_IDX:HAIR_IDX + 1]
    return torch.cat([oh[:, :HAIR_IDX], oh[:, HAIR_IDX + 1:]], 1)


def layer0_lookup(mask, table, cmap) -> torch.Tensor:
    """hf_shape_onehot_s2 restated: [128,128,C] = cmap + sum over the taps inside of table[tap][label]."""
    m = mask.clone()
    m[m == 255] = 19
    lp = F.pad(m, (1, 1, 1, 1), value=-1)
    c = table.shape[-1]
    y = cmap.double().view(128, 128, c).clone()
    for ky in range(4):
        for kx in range(4):
            src = lp[ky:ky + 256:2, kx:kx + 256:2]
            inside = src >= 0
            y += torch.where(inside[..., None], table[ky * 4 + kx].double()[src.clamp(min=0)], torch.zeros(()))
    return y


def gather_gemm(mode: int, x: torch.Tensor, w: torch.Tensor, bias=None) -> torch.Tensor:
    """hf_shape_gemm restated on float64: x [H, W, Cin] NHWC, w [Cout, kh, kw, Cin] -> [P, Cout] with the im2col of
    the given mode (1: zero pad 1 + 4x4 stride 2; 2: nearest 2x up + 3x3 pad 1)."""
    h, wd, cin = x.shape
    if mode == 1:
        xp = F.pad(x.permute(2, 0, 1), (1, 1, 1, 1)).permute(1, 2, 0)
        cols = [xp[ky:ky + h:2, kx:kx + wd:2] for ky in range(4) for kx in range(4)]
    else:
        up = x.repeat_interleave(2, 0).repeat_interleave(2, 1)
        xp = F.pad(up.permute(2, 0, 1), (1, 1, 1, 1)).permute(1, 2, 0)
        cols = [xp[ky:ky + 2 * h, kx:kx + 2 * wd] for ky in range(3) for kx in range(3)]
    a = torch.cat(cols, -1).reshape(-1, len(cols) * cin).double()
    y = a @ w.reshape(w.shape[0], -1).double().t()
    return y if bias is None else y + bias.double()


def layer_norm_lrelu(x: torch.Tensor, gamma, beta, eps: float = 1e-5, slope: float = 0.2) -> torch.Tensor:
    """CtrlHair LayerNorm (my_torchlib/module.py:183-205, batch 1) + LeakyReLU of an NHWC sample [..., C]."""
    x = x.double()
    y = (x - x.mean()) / (x.std() + eps) * gamma.double() + beta.double()
    return torch.where(y > 0, y, y * slope)


def logits(hair_map: torch.Tensor, face_map: torch.Tensor, params: dict) -> torch.Tensor:
    """Both out_layers on [256,256,32] NHWC maps and cat[face[:13], hair, face[13:]]: [19,256,256] float64."""
    def conv(x, w, b):
        return F.conv2d(x.double().permute(2, 0, 1)[None], w.double(), b.double(), padding=1)[0]
    h = conv(hair_map, params["hair_decoder.out_layer.conv.weight"], params["hair_decoder.out_layer.conv.bias"])
    f = conv(face_map, params["face_decoder.out_layer.conv.weight"], params["face_decoder.out_layer.conv.bias"])
    return torch.cat([f[:HAIR_IDX], h, f[HAIR_IDX:]])


def top2_margin(lg: torch.Tensor) -> torch.Tensor:
    """Per pixel, the largest logit minus the second largest."""
    t = lg.topk(2, dim=0).values
    return t[0] - t[1]


# ------------------------------------------------------------------------------------------------ stand-in model
def pos_embedding(size: int = 256, order: int = 10) -> torch.Tensor:
    """The 40 positional channels of MaskEncoder (model.py:18-30): sin then cos of 2^i pi t for i < order, for each
    of the (x, y) coordinates t = j / size, channel = 2 * (function * order + i) + coordinate; [40, size, size]."""
    t = torch.arange(size, dtype=torch.float64) / size
    gx, gy = t[None, :].expand(size, size), t[:, None].expand(size, size)
    chans = []
    for fn in (torch.sin, torch.cos):
        for i in range(order):
            f = (2 ** i) * torch.pi
            chans += [fn(f * gx), fn(f * gy)]
    return torch.stack(chans).float()


def stand_in_generator(params: dict, device) -> torch.nn.Module:
    """A module tree with the reference Generator's attribute names and state-dict keys carrying ``params``, plus the
    encoders' ``input_embedding`` (what hairfastgan_b200.shape_adaptor reads)."""
    root = torch.nn.Module()
    for key, value in params.items():
        *path, leaf = key.split(".")
        m = root
        for p in path:
            if not hasattr(m, p):
                m.add_module(p, torch.nn.Module())
            m = getattr(m, p)
        m.register_parameter(leaf, torch.nn.Parameter(value.clone().to(device), requires_grad=False))
    for name in ("hair_encoder", "face_encoder"):
        if hasattr(root, name):
            getattr(root, name).input_embedding = pos_embedding()[None]
    return root

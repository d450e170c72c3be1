"""Float64 restatement of HairFast's latent modulation stacks (models/Encoders.py:13-137): ModulationModule, the
Rotate / Blending / PostProcess stack calls, seeded parameters under the reference's state-dict keys, and stand-in
modules carrying them (no reference import).

``rnd`` (a 16-bit torch dtype or None) selects the operand-rounded mode: the roundings csrc/hf_modulation.cu applies
(embedding, hidden rows, every weight matrix and each chain operand to 16-bit; everything else exact), so the kernels
can be checked at summation-order tolerance."""
from __future__ import annotations

import torch
from torch import nn

DIM = 512
MODULES = 5
CONFIGS = {6: (512, 512), 12: (1536, 1024), 18: (512, 512)}      # L -> (inp, middle)
FNS = ("gamma_function", "beta_function")


def _r(t: torch.Tensor, rnd) -> torch.Tensor:
    return t.double() if rnd is None else t.to(rnd).double()


def pixel_norm(x: torch.Tensor, dim: int = 1) -> torch.Tensor:
    """models/stylegan2/model.py:21 -- over dim 1, the L rows of a [B, L, 512] latent."""
    x = x.double()
    return x * torch.rsqrt((x * x).mean(dim, keepdim=True) + 1e-8)


def layer_norm(x: torch.Tensor, dims: int, w=None, b=None) -> torch.Tensor:
    """LayerNorm over the last ``dims`` dimensions: biased variance, eps 1e-5."""
    ax = tuple(range(-dims, 0))
    m = x.mean(ax, keepdim=True)
    y = (x - m) / torch.sqrt(((x - m) ** 2).mean(ax, keepdim=True) + 1e-5)
    return y if w is None else y * w.double() + b.double()


def lrelu(x: torch.Tensor) -> torch.Tensor:
    return torch.where(x > 0, x, 0.01 * x)


def hidden(e: torch.Tensor, p: dict, fn: str, rnd=None) -> torch.Tensor:
    """Linear -> LayerNorm([middle]) -> LeakyReLU of the embedding e [..., inp]."""
    h = _r(e, rnd) @ _r(p[f"{fn}.0.weight"], rnd).t() + p[f"{fn}.0.bias"].double()
    return lrelu(layer_norm(h, 1, p[f"{fn}.1.weight"], p[f"{fn}.1.bias"]))


def gamma_beta(e: torch.Tensor, p: dict, rnd=None):
    """(gamma, beta) of one module: the MLPs of Encoders.py:20-21."""
    return tuple(_r(hidden(e, p, fn, rnd), rnd) @ _r(p[f"{fn}.3.weight"], rnd).t() + p[f"{fn}.3.bias"].double()
                 for fn in FNS)


def module(x: torch.Tensor, e: torch.Tensor, p: dict, last: bool, rnd=None, gb=None) -> torch.Tensor:
    """ModulationModule.forward (Encoders.py:24-32); gb = (gamma, beta) given instead of computed from e."""
    y = layer_norm(_r(x, rnd) @ _r(p["fc.weight"], rnd).t() + p["fc.bias"].double(), 2)
    g, b = gamma_beta(e, p, rnd) if gb is None else (gb[0].double(), gb[1].double())
    out = y * (1 + g) + b
    return out if last else lrelu(out)


def stack(x0: torch.Tensor, e: torch.Tensor, params: list, rnd=None, gbs=None, pixel_dim: int = 1) -> torch.Tensor:
    """dt of one stack: PixelNorm then the 5 modules; gbs = per-module (gamma, beta) given instead of computed."""
    x = pixel_norm(x0, pixel_dim)
    for i, p in enumerate(params):
        x = module(x, e, p, i == MODULES - 1, rnd, None if gbs is None else gbs[i])
    return x


def rotate(params, latent_from, latent_to, rnd=None, pixel_dim: int = 1):
    return latent_from.double() + 0.1 * stack(latent_from, latent_to.double(), params, rnd, pixel_dim=pixel_dim)


def blending(params, latent_face, latent_color, embed_face, embed_color, rnd=None):
    n = latent_face.shape[1]
    e = torch.cat((latent_color.double(), embed_face.double()[:, None].expand(-1, n, -1),
                   embed_color.double()[:, None].expand(-1, n, -1)), -1)
    return latent_face.double() + 0.1 * stack(latent_face, e, params, rnd)


def postprocess(params_1, params_2, s_face, s_hair, latent_avg, rnd=None):
    dt_face = stack(s_face, s_hair.double(), params_1, rnd)
    dt_hair = stack(s_hair, s_face.double(), params_2, rnd)
    return latent_avg.double() + 0.1 * (dt_face + dt_hair)


# ------------------------------------------------------------------------------------------------ parameters
def module_shapes(inp: int, middle: int) -> dict:
    d = {"fc.weight": (DIM, DIM), "fc.bias": (DIM,)}
    for f in FNS:
        d.update({f"{f}.0.weight": (middle, inp), f"{f}.0.bias": (middle,), f"{f}.1.weight": (middle,),
                  f"{f}.1.bias": (middle,), f"{f}.3.weight": (DIM, middle), f"{f}.3.bias": (DIM,)})
    return d


def synth_params(seed: int, layers: int) -> list:
    """Per-module parameter dicts of a stack: Linear weights at 1 / sqrt(fan_in), LayerNorm affines away from the
    identity (weight 1 + 0.3 N, bias 0.2 N), small biases."""
    inp, middle = CONFIGS[layers]
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(MODULES):
        p = {}
        for k, shape in module_shapes(inp, middle).items():
            if k.endswith(".1.weight"):
                p[k] = 1 + 0.3 * torch.randn(shape, generator=g)
            elif k.endswith(".1.bias"):
                p[k] = 0.2 * torch.randn(shape, generator=g)
            elif k.endswith("weight"):
                p[k] = torch.randn(shape, generator=g) / shape[1] ** 0.5
            else:
                p[k] = 0.1 * torch.randn(shape, generator=g)
        out.append(p)
    return out


def stack_state_dict(params: list) -> dict:
    """nn.ModuleList state_dict of the per-module dicts."""
    return {f"{i}.{k}": v for i, p in enumerate(params) for k, v in p.items()}


# ------------------------------------------------------------------------------------------------ stand-ins
def param_tree(shapes: dict) -> nn.Module:
    """A module tree holding zero parameters under the given state-dict keys and shapes, and nothing else."""
    root = nn.Module()
    for key, shape in shapes.items():
        *path, leaf = key.split(".")
        m = root
        for name in path:
            if name not in m._modules:
                m.add_module(name, nn.Module())
            m = m._modules[name]
        m.register_parameter(leaf, nn.Parameter(torch.zeros(shape)))
    return root


def stand_in_module(layernum: int, last: bool, inp: int, middle: int) -> nn.Module:
    """ModulationModule's state-dict key layout plus its ``layernum`` / ``last`` flags, which the drop-ins check."""
    m = param_tree(module_shapes(inp, middle))
    m.layernum, m.last = layernum, last
    return m


def stand_in_stack(params: list, layers: int, device=None) -> nn.ModuleList:
    inp, middle = CONFIGS[layers]
    st = nn.ModuleList([stand_in_module(layers, i == MODULES - 1, inp, middle) for i in range(MODULES)])
    st.load_state_dict(stack_state_dict(params), strict=True)
    return st.to(device) if device is not None else st


class StandInRotate(nn.Module):
    def __init__(self, params, device=None):
        super().__init__()
        self.modulation_module_list = stand_in_stack(params, 6, device)


class StandInBlending(nn.Module):
    """get_image_embed is the identity: the 'images' passed are the CLIP embeddings themselves."""

    def __init__(self, params, device=None):
        super().__init__()
        self.modulation_module_list = stand_in_stack(params, 12, device)

    def get_image_embed(self, image_tensor):
        return image_tensor


class StandInPostProcess(nn.Module):
    """encoder_face returns (code, [feature]) of the 'image', which is the code itself; to_feature is the identity."""

    def __init__(self, params_1, params_2, latent_avg, device=None):
        super().__init__()
        self.to_latent_1 = stand_in_stack(params_1, 18, device)
        self.to_latent_2 = stand_in_stack(params_2, 18, device)
        self.latent_avg = latent_avg.to(device) if device is not None else latent_avg
        self.to_feature = nn.Identity()

    def encoder_face(self, x):
        return x, [x[:, :1]]

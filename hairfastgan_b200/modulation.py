"""HairFast's latent modulation nets (models/Encoders.py:13-137) on the sm_90a kernels of csrc/hf_modulation.cu:
drop-in ``forward`` methods for ``RotateModel``, ``ClipBlendingModel`` and ``PostProcessModel`` with the reference's
signatures and results.

A stack is 5 ``ModulationModule(L, last=i == 4, inp, middle)``; one call of the stacks runs as 6 kernels:

* ``hf_mod_embed16``: the embedding rows to 16-bit (Blending's ``cat(latent_color, embed_face, embed_color)`` read
  from its three sources, the CLIP embeddings broadcast over the 12 rows);
* ``hf_mod_hidden`` (2): the ten first Linears of every stack's gamma / beta MLPs as one [10 middle, inp] split-K GEMM,
  reduced with ``LayerNorm([middle])`` + LeakyReLU fused in;
* ``hf_mod_gemm`` (2): the ten second Linears as one grouped split-K GEMM -> gamma / beta in fp32;
* ``hf_mod_chain``: PixelNorm, the five dependent fc + whole-sample LayerNorm + modulation steps and ``base + 0.1 dt``,
  on clusters of 8 CTAs per (stack, sample).

PostProcess's two stacks (``to_latent_1`` / ``to_latent_2``) run in the same 6 launches, plus one ``cudaMemsetAsync``
that zeroes the chain's per-(sample, slice) completion counters.  Weights are packed by
state-dict key and re-packed by the rule of ``packcache``; operands are 16-bit in the encoder family's type
(``nn16.default_dtype``), accumulation and statistics fp32.  The forward draws no random numbers and never waits for
the device.  Only HairFast's three configurations are supported: L = 6 and 18 with (inp, middle) = (512, 512), L = 12
with (1536, 1024).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, nn16, packcache

DIM = 512
MODULES = 5
CONFIGS = {6: (512, 512), 12: (1536, 1024), 18: (512, 512)}      # L -> (inp, middle)
_FNS = ("gamma_function", "beta_function")


def module_shapes(inp: int, middle: int) -> dict:
    """state_dict key -> shape of ModulationModule(L, last, inp, middle) (Encoders.py:14-22)."""
    d = {"fc.weight": (DIM, DIM), "fc.bias": (DIM,)}
    for f in _FNS:
        d.update({f"{f}.0.weight": (middle, inp), f"{f}.0.bias": (middle,), f"{f}.1.weight": (middle,),
                  f"{f}.1.bias": (middle,), f"{f}.3.weight": (DIM, middle), f"{f}.3.bias": (DIM,)})
    return d


def stack_shapes(layers: int) -> dict:
    """state_dict key -> shape of the nn.ModuleList of 5 modules with L = layers."""
    inp, middle = CONFIGS[layers]
    return {f"{i}.{k}": v for i in range(MODULES) for k, v in module_shapes(inp, middle).items()}


def _state(stack, layers: int) -> dict:
    sd = stack.state_dict()
    got = {k: tuple(v.shape) for k, v in sd.items()}
    want = stack_shapes(layers) if layers in CONFIGS else None
    flags = [(getattr(m, "layernum", layers), getattr(m, "last", i == MODULES - 1)) for i, m in enumerate(stack)]
    if got != want or flags != [(layers, i == MODULES - 1) for i in range(MODULES)]:
        raise NotImplementedError(f"modulation: only HairFast's stacks of 5 ModulationModule with L in {sorted(CONFIGS)} "
                                  f"are supported; got L = {layers}, parameters {got}")
    dev = next(iter(sd.values())).device
    if dev.type != "cuda":
        raise RuntimeError("modulation: the modulation modules must be on a CUDA device (no CPU fallback)")
    _lib.use_device(dev.index)
    return {k: v.detach().float() for k, v in sd.items()}


class PackedStacks:
    """One or two stacks in the layouts of hf_modulation.cu: branch j = 2 i + (0 gamma | 1 beta) of module i."""

    def __init__(self, stacks, layers: int, dtype: int):
        sds = [_state(st, layers) for st in stacks]
        inp, middle = CONFIGS[layers]
        t16 = nn16.torch_dtype(dtype)
        self.layers, self.inp, self.middle, self.n, self.dtype = layers, inp, middle, len(stacks), dtype

        def branches(sd, key):
            return [sd[f"{i}.{f}.{key}"] for i in range(MODULES) for f in _FNS]

        self.w1 = torch.stack([torch.cat(branches(sd, "0.weight")) for sd in sds]).to(t16).contiguous()
        self.b1 = torch.stack([torch.cat(branches(sd, "0.bias")) for sd in sds]).contiguous()
        self.ln_w = torch.stack([torch.cat(branches(sd, "1.weight")) for sd in sds]).contiguous()
        self.ln_b = torch.stack([torch.cat(branches(sd, "1.bias")) for sd in sds]).contiguous()
        self.w2 = torch.stack([w for sd in sds for w in branches(sd, "3.weight")]).to(t16).contiguous()
        self.b2 = torch.stack([b for sd in sds for b in branches(sd, "3.bias")]).contiguous()
        self.fc_w = torch.stack([torch.stack([sd[f"{i}.fc.weight"] for i in range(MODULES)]) for sd in sds])
        self.fc_w = self.fc_w.to(t16).contiguous()
        self.fc_b = torch.stack([torch.stack([sd[f"{i}.fc.bias"] for i in range(MODULES)]) for sd in sds]).contiguous()
        self.desc = _lib.hf_mod_desc(layers, inp, middle, len(stacks), dtype)


def pack(owner, stacks, layers: int) -> PackedStacks:
    """The packed stacks, cached on ``owner`` (whose class fixes ``layers``) by ``packcache``."""
    dt = nn16.default_dtype()
    return packcache.get(owner, "_hf_mod_pack", stacks, dt, lambda: PackedStacks(stacks, layers, dt))[0]


# How a [batch, layers, 512] operand is read from its tensor; each caller names the form it means.
ROWS = "rows"                  # [batch, layers, 512]
PER_SAMPLE = "per_sample"      # [batch, 512], the same row for every layer (Blending's CLIP embeddings)
PER_LAYER = "per_layer"        # [layers, 512] or [1, layers, 512], the same rows for every sample (latent_avg)


def rows(t: torch.Tensor, batch: int, layers: int, form: str, what: str):
    """hf_mod_rows of ``t`` read in ``form``; returns (rows, the fp32 tensor to keep alive).  Any other shape raises
    NotImplementedError, a CPU tensor RuntimeError."""
    want = {ROWS: [(batch, layers, DIM)], PER_SAMPLE: [(batch, DIM)],
            PER_LAYER: [(layers, DIM), (1, layers, DIM)]}[form]
    if tuple(t.shape) not in want:
        raise NotImplementedError(f"modulation: {what} has shape {list(t.shape)}; expected "
                                  f"{' or '.join(str(list(w)) for w in want)}")
    if not t.is_cuda:
        raise RuntimeError(f"modulation: {what} must be a CUDA tensor (no CPU fallback)")
    t = t.float()
    if t.stride(-1) != 1:
        t = t.contiguous()
    bs, rs = {ROWS: (t.stride(0), t.stride(1)), PER_SAMPLE: (t.stride(0), 0), PER_LAYER: (0, t.stride(-2))}[form]
    return _lib.hf_mod_rows(t.data_ptr(), bs, rs), t


@torch.no_grad()
def run(pk: PackedStacks, sources, x0s, base, batch: int) -> torch.Tensor:
    """base + 0.1 * (sum over the stacks of stack s run from PixelNorm(x0s[s]) with embedding sources[s]):
    [batch, L, 512] fp32.  sources[s] lists the embedding's 512-wide column blocks as (tensor, form); x0s are ROWS;
    base is (tensor, form)."""
    lib, d, L = _lib.lib(), pk.desc, pk.layers
    keep = []

    def r(t, form, what):
        rr, t = rows(t, batch, L, form, what)
        keep.append(t)
        return rr

    src = [r(t, form, "embedding") for srcs in sources for t, form in srcs]
    x0 = [r(t, ROWS, "latent") for t in x0s]
    base_rows = r(*base, "base latent")
    dev = x0s[0].device
    _lib.use_device(dev.index)
    n_rows, t16, st = batch * L, nn16.torch_dtype(pk.dtype), _lib.stream_ptr()
    nbytes = lib.hf_mod_workspace_bytes(C.byref(d), batch)
    if nbytes == 0:
        _lib.check(-1, "hf_mod_workspace_bytes")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    e16 = torch.empty(pk.n, n_rows, pk.inp, dtype=t16, device=dev)
    h16 = torch.empty(n_rows, pk.n * 2 * MODULES * pk.middle, dtype=t16, device=dev)
    gb = torch.empty(pk.n * 2 * MODULES, n_rows, DIM, dtype=torch.float32, device=dev)
    out = torch.empty(batch, L, DIM, dtype=torch.float32, device=dev)
    _lib.check(lib.hf_mod_embed16(C.byref(d), batch, (_lib.hf_mod_rows * len(src))(*src), e16.data_ptr(), st),
               "hf_mod_embed16")
    _lib.check(lib.hf_mod_hidden(C.byref(d), batch, pk.w1.data_ptr(), e16.data_ptr(), pk.b1.data_ptr(),
                                 pk.ln_w.data_ptr(), pk.ln_b.data_ptr(), h16.data_ptr(), ws.data_ptr(), st),
               "hf_mod_hidden")
    _lib.check(lib.hf_mod_gemm(C.byref(d), batch, 2, pk.w2.data_ptr(), h16.data_ptr(), pk.b2.data_ptr(),
                               gb.data_ptr(), ws.data_ptr(), st), "hf_mod_gemm")
    _lib.check(lib.hf_mod_chain(C.byref(d), batch, pk.fc_w.data_ptr(), pk.fc_b.data_ptr(), gb.data_ptr(),
                                (_lib.hf_mod_rows * 2)(*(x0 + x0)[:2]), C.byref(base_rows), out.data_ptr(),
                                ws.data_ptr(), st), "hf_mod_chain")
    return out


def _batch(t: torch.Tensor, layers: int, what: str) -> int:
    if t.dim() != 3 or t.shape[1:] != (layers, DIM):
        raise NotImplementedError(f"modulation: {what} must be [B, {layers}, {DIM}], got {list(t.shape)}")
    return t.shape[0]


# ------------------------------------------------------------------------------------------------ drop-ins
def rotate_forward(self, latent_from, latent_to):
    """RotateModel.forward (Encoders.py:66-71)."""
    b = _batch(latent_from, 6, "latent_from")
    pk = pack(self, [self.modulation_module_list], 6)
    return run(pk, [[(latent_to, ROWS)]], [latent_from], (latent_from, ROWS), b)


def blending_forward(self, latent_face, latent_color, target_face, hair_color):
    """ClipBlendingModel.forward (Encoders.py:94-103); the CLIP embeddings still come from ``get_image_embed``."""
    b = _batch(latent_face, 12, "latent_face")
    embed_face = self.get_image_embed(target_face)
    embed_color = self.get_image_embed(hair_color)
    pk = pack(self, [self.modulation_module_list], 12)
    return run(pk, [[(latent_color, ROWS), (embed_face, PER_SAMPLE), (embed_color, PER_SAMPLE)]], [latent_face],
               (latent_face, ROWS), b)


def postprocess_forward(self, source, target):
    """PostProcessModel.forward (Encoders.py:119-137): both latent stacks in one call, each on the other image's
    code; the feature path stays ``self.to_feature``."""
    s_face, [f_face] = self.encoder_face(source)
    s_hair, [f_hair] = self.encoder_face(target)
    b = _batch(s_face, 18, "s_face")
    pk = pack(self, [self.to_latent_1, self.to_latent_2], 18)
    finall_s = run(pk, [[(s_hair, ROWS)], [(s_face, ROWS)]], [s_face, s_hair], (self.latent_avg, PER_LAYER), b)
    finall_f = self.to_feature(torch.cat((f_face, f_hair), dim=1))
    return finall_s, finall_f


FORWARDS = {"RotateModel": rotate_forward, "ClipBlendingModel": blending_forward,
            "PostProcessModel": postprocess_forward}


def patch_encoders_module(module) -> bool:
    """Wrap the three classes' ``forward`` in ``models.Encoders`` (the original kept as ``__wrapped__``)."""
    done = False
    for name, fn in FORWARDS.items():
        cls = getattr(module, name, None)
        if cls is None or "forward" not in cls.__dict__ or hasattr(cls.__dict__["forward"], "__wrapped__"):
            continue

        def forward(self, *args, __fn=fn, **kwargs):
            return __fn(self, *args, **kwargs)

        forward.__wrapped__ = cls.__dict__["forward"]
        forward.__name__ = "forward"
        forward.__doc__ = fn.__doc__
        cls.forward = forward
        done = True
    return done


def unpatch_encoders_module(module) -> None:
    for name in FORWARDS:
        cls = getattr(module, name, None)
        orig = getattr(cls.__dict__.get("forward"), "__wrapped__", None) if cls is not None else None
        if orig is not None:
            cls.forward = orig

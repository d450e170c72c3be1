"""Case tables of tests/test_gpu_ops_exact.py and Python restatements of the host-side dispatch of the entry points
they call, so that every case can name the kernel it reaches and tests/test_ops_exact_cases_cpu.py can check,
without a device, that the tables reach every kernel:

* `upfirdn_path`   -- hf_upfirdn2d_f32 (csrc/hf_ops.cu): the 4x4 bulk-copy strip kernels (down 1 / down 2 at 2 or 4
                      columns per thread, each with the separable or the general FIR loop; up 2 at 2 or 4 columns per
                      thread) and upfirdn2d_general_kernel;
* `bias_act_path`  -- hf_bias_act_f32 (csrc/hf_ops.cu): bias_act_plane_kernel, bias_act_kernel<true> (flat float4)
                      and bias_act_kernel<false> (scalar), each with or without a second grid-stride iteration;
* `fspace_path`    -- fspace_blend_kernel (csrc/hf_glue_ops.cu): float4 columns, float4 with a partial last CTA, and
                      the scalar loop (P % 4 != 0, or a tensor that is not 16-byte aligned).

Byte offsets (`x_off`, `y_off`) are those of the tensors the tests build: a view 4 bytes into a fresh allocation.
The SM count only decides the grid-stride classes; without a device it is the 132 of an H100 SXM."""
from __future__ import annotations

import zlib
from typing import NamedTuple

import numpy as np
import torch

SMS = 132


def cdiv(a, b):
    return -(-a // b)


def grid_threads(sms):
    """Threads of one `grid_for` grid (csrc/hf_common.cuh): at most 16 CTAs of 256 threads per SM."""
    return sms * 16 * 256


def seed(name):
    return zlib.crc32(name.encode())


# ------------------------------------------------------------------------------------------------ upfirdn2d
def fir_separable(k):
    """The rank-1 test of upfirdn2d_k4_bulk_kernel on the flipped 4x4 taps kr, in float32: kx = row 0 of kr,
    ky[a] = kr[a][0] / kr[0][0], separable when every |ky[a] kx[b] - kr[a][b]| <= 1e-6 |kr[a][b]| + 1e-30.  The
    compiler may evaluate ky * kx - kr with one rounding (FFMA) or two; both are computed, and a case whose decision
    depends on that is refused."""
    kr = np.asarray(k, dtype=np.float32).reshape(-1)[::-1].reshape(4, 4)
    if kr[0, 0] == 0:
        return False
    f32 = np.float32
    ky = np.array([kr[a, 0] / kr[0, 0] for a in range(4)], dtype=np.float32)
    decisions = set()
    for fused in (False, True):
        ok = True
        for a in range(4):
            for b in range(4):
                if fused:
                    d = f32(np.float64(ky[a]) * np.float64(kr[0, b]) - np.float64(kr[a, b]))
                else:
                    d = f32(f32(ky[a] * kr[0, b]) - kr[a, b])
                ok = ok and abs(d) <= f32(1e-6) * abs(kr[a, b]) + f32(1e-30)
        decisions.add(ok)
    assert len(decisions) == 1, "rank-1 test on the edge of its tolerance: the FIR loop depends on contraction"
    return decisions.pop()


def upfirdn_out(u):
    return ((u.in_h * u.up_y + u.py0 + u.py1 - u.kh) // u.down_y + 1,
            (u.in_w * u.up_x + u.px0 + u.px1 - u.kw) // u.down_x + 1)


def upfirdn_path(u, k=None):
    """hf_upfirdn2d_f32's choice for case u (csrc/hf_ops.cu, the bulk_ok / pads03 / width conditions)."""
    out_h, out_w = upfirdn_out(u)
    k4 = u.kh == 4 and u.kw == 4
    sym = u.up_x == u.up_y and u.down_x == u.down_y
    pads03 = all(0 <= p <= 3 for p in (u.px0, u.px1, u.py0, u.py1))
    bulk_ok = (k4 and sym and u.planes <= 65535 and u.in_w >= 64 and u.x_off % 16 == 0
               and (u.planes * u.in_h * u.in_w) % 4 == 0)
    fir = lambda: "sep" if fir_separable(upfirdn_taps(u) if k is None else k) else "gen"
    if bulk_ok and u.up_x == 1 and u.down_x in (1, 2) and pads03 and out_w <= 1024 and u.in_w <= 1040:
        return f"bulk_d{u.down_x}_nc{2 if out_w <= 512 else 4}_{fir()}"
    if (bulk_ok and u.up_x == 2 and u.down_x == 1 and (u.px0, u.py0, u.px1, u.py1) == (2, 2, 1, 1)
            and u.in_w <= 1024 and u.y_off % 8 == 0):
        return f"bulk_up2_nc{2 if u.in_w <= 512 else 4}"
    return "general"


UPFIRDN_PATHS = ([f"bulk_d{d}_nc{nc}_{f}" for d in (1, 2) for nc in (2, 4) for f in ("sep", "gen")]
                 + ["bulk_up2_nc2", "bulk_up2_nc4", "general"])


class Up(NamedTuple):
    name: str
    planes: int
    in_h: int
    in_w: int
    up_x: int = 1
    up_y: int = 1
    down_x: int = 1
    down_y: int = 1
    px0: int = 1
    px1: int = 1
    py0: int = 1
    py1: int = 1
    fir: str = "gen"         # gen: distinct taps; sep: outer(u, v) / 64 with dyadic ratios; sep3: u[3] = 3;
    kh: int = 4              # near: rank-1 only within the kernel's 1e-6 test
    kw: int = 4
    x_off: int = 0
    y_off: int = 0
    impulses: bool = True    # plane 0 holds impulses instead of random integers


def _distinct_taps(g, n):
    """n distinct integers in [-16, 16] / 64, none zero."""
    vals = torch.cat([torch.arange(-16, 0), torch.arange(1, 17)]).double()
    return vals[torch.randperm(32, generator=g)[:n]] / 64


def _factor(g, last):
    """4 distinct nonzero integers in [-4, 4] with the given last entry."""
    pool = [v for v in (-4, -3, -2, -1, 1, 2, 3, 4) if v != last]
    head = [pool[i] for i in torch.randperm(len(pool), generator=g)[:3].tolist()]
    return torch.tensor(head + [last], dtype=torch.float64)


def upfirdn_taps(u):
    """The case's FIR [kh, kw] in float64 (every value exact in fp32).  For `near` it is the TRUE kernel: one tap
    off the rank-1 product by a relative 2^-21 (4.8e-7), inside the bulk kernel's 1e-6 separability test."""
    g = torch.Generator().manual_seed(seed(u.name + u.fir))
    if u.fir == "gen":
        return _distinct_taps(g, u.kh * u.kw).view(u.kh, u.kw)
    assert (u.kh, u.kw) == (4, 4)
    last_u = {"sep": [1, -1, 2, -2], "near": [1, -1, 2, -2], "sep3": [3]}[u.fir]
    uu = _factor(g, last_u[int(torch.randint(0, len(last_u), (1,), generator=g))])
    vv = _factor(g, [1, -1, 2, -2, 3, -3][int(torch.randint(0, 6, (1,), generator=g))])
    k = torch.outer(uu, vv) / 64
    if u.fir == "near":
        k[1, 2] *= 1 + 2.0 ** -21            # flipped position (2, 1): neither row 0 nor column 0 of kr
    return k


def rank1_part(k):
    """What the separable loop computes for `near`: the rank-1 kernel through kr's row 0 and column 0."""
    kr = k.flip(0, 1)
    r = torch.outer(kr[:, 0] / kr[0, 0], kr[0, :])
    return r.flip(0, 1)


def _widths():
    """The column-ownership boundaries: a thread owns columns t, t + 256, ... (out_w for down 1 / 2, in_w for up 2)."""
    cases = []
    # down 1: out_w = in_w + px0 + px1 - 3
    for out_w, (px0, px1), (planes, in_h, py0, py1) in [
            (255, (1, 1), (2, 67, 1, 1)), (256, (0, 3), (3, 70, 2, 1)), (257, (2, 2), (1, 64, 0, 3)),
            (511, (3, 0), (2, 34, 1, 2)), (512, (1, 1), (2, 20, 1, 1)), (513, (0, 0), (4, 9, 3, 0)),
            (1024, (1, 1), (2, 70, 1, 1))]:
        for fir in ("sep", "gen"):
            cases.append(Up(f"d1_ow{out_w}_{fir}", planes, in_h, out_w + 3 - px0 - px1, px0=px0, px1=px1, py0=py0,
                            py1=py1, fir=fir))
    # down 2: out_w = (in_w + px0 + px1 - 4) // 2 + 1; 4 columns per thread only from out_w 513 (in_w <= 1040)
    for out_w, in_w, (px0, px1), (planes, in_h, py0, py1) in [
            (255, 510, (1, 1), (2, 67, 1, 1)), (256, 511, (2, 1), (2, 70, 0, 0)), (257, 514, (1, 1), (1, 130, 1, 2)),
            (511, 1021, (3, 0), (2, 34, 3, 3)), (512, 1024, (1, 1), (2, 66, 1, 1)),
            (513, 1028, (0, 0), (4, 9, 2, 1)), (521, 1040, (2, 2), (2, 40, 1, 1))]:
        assert (in_w + px0 + px1 - 4) // 2 + 1 == out_w
        for fir in ("sep", "gen"):
            cases.append(Up(f"d2_ow{out_w}_{fir}", planes, in_h, in_w, down_x=2, down_y=2, px0=px0, px1=px1,
                            py0=py0, py1=py1, fir=fir))
    # up 2, pad (2, 1)
    for in_w, (planes, in_h) in [(255, (2, 38)), (256, (3, 33)), (257, (1, 32)), (511, (2, 64)), (512, (2, 20)),
                                 (513, (4, 7)), (1024, (2, 35))]:
        cases.append(Up(f"up2_iw{in_w}", planes, in_h, in_w, 2, 2, px0=2, px1=1, py0=2, py1=1,
                        fir="sep" if in_w % 2 else "gen"))
    return cases


def _strips():
    """Strip and chunk edges: 64 / 32 output rows per CTA for down 1 / 2 and 32 input rows for up 2, 4-row chunks
    (6 for up 2) in 3 stages.  A full strip is 17 chunks for down 1 and 2, so each stage is reused five or six times
    and its mbarrier phase flips as often; an up-2 strip is at most 6 chunks (34 rows)."""
    return [
        Up("d1_oh1_one_chunk", 4, 4, 100, py0=0, py1=0),                       # out_h 1: 4 strip rows, 1 chunk
        Up("d1_in_h1", 4, 1, 96, py0=2, py1=1),                                 # one input row, out_h 1
        Up("d1_oh64_full_strip", 2, 65, 128, py0=1, py1=1, fir="sep"),          # 67 rows: 17 chunks, tail of 3
        Up("d1_oh130_three_strips", 2, 131, 96, py0=2, py1=0),                  # last strip: 2 rows, 2 chunks
        Up("d1_oh200_chunk_tail", 3, 201, 80, py0=1, py1=1, fir="sep"),         # last strip: 8 rows + 3
        Up("d2_oh1_one_chunk", 4, 4, 100, down_x=2, down_y=2, py0=0, py1=0),
        Up("d2_in_h1", 4, 1, 96, down_x=2, down_y=2, py0=2, py1=1),
        Up("d2_oh32_full_strip", 2, 66, 128, down_x=2, down_y=2, py0=0, py1=0, fir="sep"),
        Up("d2_oh97_four_strips", 2, 194, 96, down_x=2, down_y=2, py0=1, py1=1),
        Up("up2_in_h1", 4, 1, 64, 2, 2, px0=2, px1=1, py0=2, py1=1),
        Up("up2_in_h32_full_strip", 2, 32, 96, 2, 2, px0=2, px1=1, py0=2, py1=1),
        Up("up2_in_h75_three_strips", 2, 75, 128, 2, 2, px0=2, px1=1, py0=2, py1=1, fir="sep"),
    ]


def _plane_offsets():
    """in_h * in_w = 1, 2, 3 (mod 4) with 4 planes: planes 1..3 start inside a 16-byte word, so the widened span of
    their first chunk begins inside the previous plane."""
    cases = []
    for r, (h, w) in zip((1, 2, 3), ((5, 65), (6, 67), (7, 65))):
        assert (h * w) % 4 == r
        cases += [Up(f"d1_plane_mod4_{r}", 4, h, w, fir="sep" if r == 2 else "gen"),
                  Up(f"d2_plane_mod4_{r}", 4, h + 4, w, down_x=2, down_y=2),
                  Up(f"up2_plane_mod4_{r}", 4, h, w, 2, 2, px0=2, px1=1, py0=2, py1=1)]
    return cases


def _general():
    """One case per condition that sends a 4x4-like call to upfirdn2d_general_kernel."""
    return [
        Up("gen_x_not_16B_aligned", 2, 20, 130, x_off=4),
        Up("gen_total_not_mult4", 1, 5, 65),
        Up("gen_in_w63", 4, 12, 63),
        Up("gen_in_w1044", 2, 9, 1044, down_x=2, down_y=2),
        Up("gen_pad_m1", 2, 12, 70, px0=-1, px1=2, py0=1, py1=-1),
        Up("gen_pad_4", 2, 12, 70, px0=4, px1=0, py0=2, py1=4),
        Up("gen_k1x1", 2, 9, 70, px0=0, px1=0, py0=0, py1=0, kh=1, kw=1),
        Up("gen_k3x5", 2, 9, 70, 2, 2, px0=2, px1=3, py0=1, py1=2, kh=3, kw=5),
        Up("gen_up_x_ne_up_y", 2, 9, 70, 2, 1, px0=2, px1=1, py0=1, py1=1),
        Up("gen_down_x_ne_down_y", 2, 10, 70, down_x=1, down_y=2),
        Up("gen_up2_y_not_8B_aligned", 2, 9, 70, 2, 2, px0=2, px1=1, py0=2, py1=1, y_off=4),
        Up("gen_up2_pad_12", 2, 9, 70, 2, 2, px0=1, px1=2, py0=1, py1=2),
        Up("gen_up3_down2", 3, 11, 70, 3, 3, 2, 2, px0=2, px1=2, py0=3, py1=1),
        Up("gen_planes_65536", 65536, 1, 64, px0=1, px1=2, py0=2, py1=1, impulses=False),
        Up("gen_over_one_grid", 6, 128, 128, 3, 3, px0=2, px1=1, py0=2, py1=1),
    ]


def _bounded():
    return [Up("d1_sep3_rounded_ky", 2, 40, 300, fir="sep3"), Up("d2_sep3_rounded_ky", 2, 40, 300, 1, 1, 2, 2,
                                                                   fir="sep3"),
            Up("d1_near_rank1", 2, 40, 300, fir="near"), Up("d2_near_rank1", 2, 40, 300, 1, 1, 2, 2, fir="near")]


UPFIRDN_EXACT = _widths() + _strips() + _plane_offsets() + _general()
UPFIRDN_BOUNDED = _bounded()


def upfirdn_id(u):
    return f"{upfirdn_path(u)}-{u.name}"


# ------------------------------------------------------------------------------------------------ bias_act
def bias_act_path(n, size_b, step_b, x_off=0, y_off=0, sms=SMS):
    """hf_bias_act_f32's choice: the per-plane float4 kernel, the flat float4 kernel or the scalar one, plus
    `_stride` when a thread of the grid-stride loop runs more than one iteration."""
    aligned = (x_off | y_off) % 16 == 0
    if step_b % 4 == 0 and step_b >= 1024 and n % step_b == 0 and n // step_b <= 65535 and aligned:
        planes, quads = n // step_b, step_b // 4
        gx = max(1, min(cdiv(quads, 256), max(1, sms * 16 // planes)))
        return "plane" + ("_stride" if quads > gx * 256 else "")
    vec = step_b % 4 == 0 and n % 4 == 0 and aligned
    work = n // 4 if vec else n
    return ("flat_vec" if vec else "scalar") + ("_stride" if work > grid_threads(sms) else "")


BIAS_ACT_PATHS = [p + s for p in ("plane", "flat_vec", "scalar") for s in ("", "_stride")]


class Ba(NamedTuple):
    name: str
    shape: tuple
    bias: str = "channel"    # channel: size_b = shape[1]; none: NULL bias; odd3: size_b = 3 on more planes
    act: int = 3
    alpha: float = 0.2
    scale: float = 2 ** 0.5
    x_off: int = 0
    y_off: int = 0


BIAS_ACT = [
    Ba("nchw_b2_c4_32x32", (2, 4, 32, 32)),
    Ba("nchw_b3_c5_48x48_act1_nobias", (3, 5, 48, 48), bias="none", act=1),
    Ba("nchw_b2_c6_64x64_alpha_scale", (2, 6, 64, 64), alpha=0.1, scale=1.5),
    Ba("nchw_b2_c4_32x32_size_b3", (2, 4, 32, 32), bias="odd3", alpha=-0.5, scale=0.25),
    Ba("ncl_4x16x1024", (4, 16, 1024), act=1, scale=3.0),
    Ba("nchw_b2_c2112_2048_stride", (2, 2112, 32, 64)),
    Ba("nchw_b2_c4_8x8", (2, 4, 8, 8)),
    Ba("nchw_b2_c4_8x8_nobias", (2, 4, 8, 8), bias="none"),
    Ba("ncl_3x7x20_act1", (3, 7, 20), act=1, alpha=0.3, scale=0.5),
    Ba("ncl_1x65536x1024_planes_over_65535", (1, 65536, 1024), scale=1.0),
    Ba("nchw_64x64x24x24_stride", (64, 64, 24, 24)),
    Ba("nchw_b2_c3_5x7_odd_hw", (2, 3, 5, 7)),
    Ba("nchw_b2_c3_5x7_nobias_act1", (2, 3, 5, 7), bias="none", act=1, scale=1.25),
    Ba("nchw_b2_c4_32x32_x_unaligned", (2, 4, 32, 32), x_off=4),
    Ba("nchw_b2_c4_32x32_y_unaligned", (2, 4, 32, 32), y_off=4, alpha=0.05, scale=2.0),
    Ba("nc_6x512_2d", (6, 512)),
    Ba("nc_5x7_2d_act1", (5, 7), act=1),
    Ba("nchw_8x16x67x67_odd_stride", (8, 16, 67, 67)),
]


def bias_act_dims(c):
    n = 1
    for s in c.shape:
        n *= s
    step_b = 1
    for s in c.shape[2:]:
        step_b *= s
    size_b = {"channel": c.shape[1], "none": 0, "odd3": 3}[c.bias]
    return n, size_b, step_b


def bias_act_id(c, sms=SMS):
    n, size_b, step_b = bias_act_dims(c)
    return f"{bias_act_path(n, size_b, step_b, c.x_off, c.y_off, sms)}-{c.name}"


# ------------------------------------------------------------------------------------------------ F-space blend
def fspace_path(P, aligned=True):
    """fspace_blend_kernel's per-thread choice: float4 when the tensors are 16-byte aligned and P % 4 == 0, for the
    quads that lie inside P (`vec_tail`: a CTA whose 256 pixels are not all inside the image)."""
    if not aligned:
        return "scalar_unaligned"
    if P % 4:
        return "scalar"
    return "vec" if P % 256 == 0 else "vec_tail"


FSPACE_PATHS = ["vec", "vec_tail", "scalar", "scalar_unaligned"]


class Fs(NamedTuple):
    name: str
    C: int
    Ho: int
    Wo: int
    Hm: int
    Wm: int
    stages: int = 1
    mask: str = "int"        # int: integers 0..3; dyadic: {0, 1/4, 1/2, 3/4, 1}
    aligned: bool = True
    ref: str = "exact"       # exact: the float64 chain is exact in fp32; ffma: only the weights are (see the test)


FSPACE = [
    Fs("ratio8_256to32", 16, 32, 32, 256, 256),
    Fs("ratio4_128to32_c19", 19, 32, 32, 128, 128),
    Fs("ratio2_64to32_c6", 6, 32, 32, 64, 64),
    Fs("up2_16to32", 16, 32, 32, 16, 16),
    Fs("up2_5to10_c3", 3, 10, 10, 5, 5),
    Fs("same_size_32", 16, 32, 32, 32, 32, mask="dyadic"),
    Fs("ratio4x2_128x64_to_32x32", 16, 32, 32, 128, 64),
    Fs("ratio1x8_20x256_to_20x32_c5", 5, 20, 32, 20, 256),
    Fs("up2x_ratio2y_24x7_to_12x14", 19, 12, 14, 24, 7),
    Fs("same_size_2_stages", 16, 32, 32, 32, 32, stages=2, mask="dyadic"),
    Fs("same_size_3_stages_c19", 19, 20, 13, 20, 13, stages=3, mask="dyadic"),
    Fs("same_size_4_stages", 16, 32, 32, 32, 32, stages=4, mask="dyadic"),
    Fs("same_size_4_stages_c6_odd", 6, 9, 7, 9, 7, stages=4, mask="dyadic"),
    Fs("ratio8_2_stages", 8, 32, 32, 256, 256, stages=2, ref="ffma"),
    Fs("ratio8_4_stages_256to32", 16, 32, 32, 256, 256, stages=4, ref="ffma"),
    Fs("up2_2_stages_c3", 3, 16, 20, 8, 10, stages=2, ref="ffma"),
    Fs("up2x_ratio2y_3_stages_c19", 19, 12, 14, 24, 7, stages=3, ref="ffma"),
    Fs("ratio2_P260_tail_cta", 4, 20, 13, 40, 26),
    Fs("ratio2_P63_scalar_c5", 5, 9, 7, 18, 14),
    Fs("unaligned_ratio8", 16, 32, 32, 256, 256, aligned=False),
    Fs("unaligned_same_size_4_stages", 16, 32, 32, 32, 32, stages=4, mask="dyadic", aligned=False),
]


def fspace_id(c):
    return f"{fspace_path(c.Ho * c.Wo, c.aligned)}-{c.name}"


# ------------------------------------------------------------------------------------------------ float64 references
def upfirdn_ref(x, k, up_x, up_y, down_x, down_y, px0, px1, py0, py1):
    """x [P, H, W], k [kh, kw], float64: zero-stuff each axis, pad (negative = crop), correlate with the flipped
    taps, keep every down-th sample -- op/upfirdn2d.py's upfirdn2d_native with up / down / pad per axis."""
    p, h, w = x.shape
    z = x.new_zeros(p, h * up_y, w * up_x)
    z[:, ::up_y, ::up_x] = x
    z = torch.nn.functional.pad(z, (max(px0, 0), max(px1, 0), max(py0, 0), max(py1, 0)))
    z = z[:, max(-py0, 0):z.shape[1] - max(-py1, 0), max(-px0, 0):z.shape[2] - max(-px1, 0)]
    out = torch.nn.functional.conv2d(z[:, None], k.flip(0, 1)[None, None])[:, 0]
    return out[:, ::down_y, ::down_x]


def bicubic_ref(x, k, f, clip_round, keep=None):
    """utils/bicubic.py:36-78 in float64 on x [P, H, W]: reflect-pad H by (3f // 2, 3f - 3f // 2), the 4f-tap column
    filter with stride f, [clamp(round)], the same along W.  `keep` collects the values before each rounding."""
    pad = 3 * f
    t, b = pad // 2, pad - pad // 2
    v = torch.nn.functional.pad(x[:, None], (0, 0, t, b), mode="reflect")
    v = torch.nn.functional.conv2d(v, k.view(1, 1, -1, 1), stride=(f, 1))
    if clip_round:
        if keep is not None:
            keep.append(v.clone())
        v = v.round().clamp(0, 255)                     # torch.round: half to even, like rintf
    v = torch.nn.functional.pad(v, (t, b, 0, 0), mode="reflect")
    v = torch.nn.functional.conv2d(v, k.view(1, 1, 1, -1), stride=(1, f))
    if clip_round:
        if keep is not None:
            keep.append(v.clone())
        v = v.round().clamp(0, 255)
    return v[:, 0]


def cubic_weights(t):
    """ATen's upsample_bicubic2d coefficients (A = -0.75) of the four taps around the floor, float64 [..., 4]."""
    A = -0.75
    x0, x1, x2, x3 = t + 1, t, 1 - t, 2 - t
    return torch.stack([((A * x0 - 5 * A) * x0 + 8 * A) * x0 - 4 * A, ((A + 2) * x1 - (A + 3)) * x1 * x1 + 1,
                        ((A + 2) * x2 - (A + 3)) * x2 * x2 + 1, ((A * x3 - 5 * A) * x3 + 8 * A) * x3 - 4 * A], -1)


def bicubic_interp_ref(m, ho, wo):
    """F.interpolate(m [Hm, Wm], (ho, wo), 'bicubic', align_corners=False) in float64: source (o + 0.5) in / out - 0.5,
    four taps around its floor with indices clamped to the image."""
    hm, wm = m.shape

    def axis(n_out, n_in):
        s = (torch.arange(n_out, dtype=torch.float64) + 0.5) * (n_in / n_out) - 0.5
        f = torch.floor(s)
        idx = (f.long()[:, None] + torch.arange(-1, 3)).clamp(0, n_in - 1)
        return cubic_weights(s - f), idx

    wy, iy = axis(ho, hm)
    wx, ix = axis(wo, wm)
    g = m[iy[:, :, None, None], ix[None, None, :, :]]             # [ho, 4, wo, 4]
    return torch.einsum("yj,yjxi,xi->yx", wy, g, wx)

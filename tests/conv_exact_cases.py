"""Case table of the exact-arithmetic convolution tests (tests/test_gpu_conv_exact.py runs it on the GPU,
tests/test_conv_plan_cases_cpu.py checks without a device that it reaches every kernel variant).

`conv_plan` picks the N tile from the SM count, so the batch sizes that must fill the GPU are computed from `sms`
here; every case states the (channels per K chunk, N tile, mainloop) it is meant to run, and both tests assert it
through the plan query.  Mainloop: SHIFT = column-shift boxes (plan out[4] = activation ring slots), TAP = one
activation box per tap (out[4] = 0)."""
import ctypes as C
from typing import NamedTuple, Optional, Tuple

SHIFT, TAP = 2, 0          # plan out[4]
PLAN_FIELDS = ("k0", "n_tile", "n_n", "k3", "a_slots", "k5", "k6", "stages", "smem", "work", "grid", "kchunk")


class Enc(NamedTuple):
    """One hf_conv2d_forward call.  cin = channels of the nn.Conv2d (cin_pad = stored NHWC channels, default cin)."""
    name: str
    cin: int
    cout: int
    h: int
    w: int
    batch: int
    plan: Tuple[int, int, int]              # (kchunk, n_tile, SHIFT | TAP)
    k: int = 3
    stride: int = 1
    groups: int = 1
    cin_pad: Optional[int] = None
    y32_only: bool = False                  # SEAN's gamma || beta convolution asks for the fp32 NCHW output alone
    hot_last_row: bool = False              # large values on the last row of every sample
    min_tiles_per_cta: int = 0              # persistence cases: the plan must give each CTA at least this many tiles
    n_tiles_per_m: int = 0                  # ... and this many N tiles per M tile (0 = any)


class Gen(NamedTuple):
    """One hf_conv_forward call (ModulatedConv2d, 3x3)."""
    name: str
    cin: int
    cout: int
    h: int
    w: int
    batch: int
    up: int
    plan: Tuple[int, int, int]


def _fill(sms, tiles_per_sample, n_tiles=1, rounds=1):
    """Smallest batch with at least rounds * sms work items."""
    return -(-rounds * sms // (tiles_per_sample * n_tiles))


def encoder_cases(sms):
    two = 2 * sms + 1                       # 8x8 maps: two samples per tile, the last tile half empty
    return [
        # ---- column-shift mainloop: stride-1 3x3, 16 x 8 pixel tiles of one sample
        Enc("shift_kc32_n32", 32, 32, 16, 16, 1, (32, 32, SHIFT)),
        Enc("shift_kc32_n64_fill", 32, 64, 32, 32, _fill(sms, 8), (32, 64, SHIFT)),
        Enc("shift_kc32_n128_fill", 32, 128, 32, 32, _fill(sms, 8), (32, 128, SHIFT)),
        Enc("shift_kc64_n32_one_tile_row", 64, 32, 8, 16, 3, (64, 32, SHIFT), hot_last_row=True),
        Enc("shift_kc64_n64_h24_w48", 64, 192, 24, 48, _fill(sms, 9, 3), (64, 64, SHIFT), hot_last_row=True),
        Enc("shift_kc64_n128_h40_w80", 64, 128, 40, 80, _fill(sms, 25), (64, 128, SHIFT)),
        Enc("shift_groups2_n32", 128, 128, 16, 16, 3, (64, 32, SHIFT), groups=2),
        Enc("shift_groups2_n64_fill", 128, 128, 16, 16, _fill(sms, 2, 2), (64, 64, SHIFT), groups=2),
        Enc("shift_kc32_cin96", 96, 64, 16, 32, 2, (32, 32, SHIFT)),
        # persistent CTAs: 9 k-blocks per tile against 8 (N = 64) and 5 (N = 128) weight slots, so the ring phase
        # carries over from tile to tile; with two N tiles per M tile the weight ring is re-entered mid-phase
        Enc("persist_n64_3_tiles", 64, 64, 32, 32, _fill(sms, 8, 1, 3), (64, 64, SHIFT), min_tiles_per_cta=3),
        Enc("persist_n128_two_n_tiles", 64, 256, 32, 32, _fill(sms, 8, 2, 3), (64, 128, SHIFT), min_tiles_per_cta=3,
            n_tiles_per_m=2),
        # ---- per-tap mainloop: narrow maps (several samples per tile), stride 2, 1x1 kernels
        Enc("tap_stem_cin3_pad32", 3, 32, 8, 8, 3, (32, 32, TAP), cin_pad=32),
        Enc("tap_kc32_n64_8x8_fill", 32, 64, 8, 8, two, (32, 64, TAP)),
        Enc("tap_kc32_n128_1x1_fill", 32, 128, 16, 16, _fill(sms, 2), (32, 128, TAP), k=1),
        Enc("tap_kc64_n32_4x4_b5", 64, 32, 4, 4, 5, (64, 32, TAP)),
        Enc("tap_kc64_n32_4x4_b9", 64, 32, 4, 4, 9, (64, 32, TAP)),
        Enc("tap_kc64_n64_stride2_fill", 64, 64, 32, 32, _fill(sms, 2), (64, 64, TAP), stride=2),
        Enc("tap_kc64_n128_8x8_fill", 64, 128, 8, 8, two, (64, 128, TAP)),
        Enc("tap_groups4_stride2_b9", 128, 128, 8, 8, 9, (32, 32, TAP), stride=2, groups=4),
        Enc("tap_stride2_to_1x1_b3", 64, 64, 2, 2, 3, (64, 32, TAP), stride=2),
        Enc("tap_stride2_to_1x1_b130", 64, 64, 2, 2, 130, (64, 32, TAP), stride=2),
        Enc("tap_1x1_stride1", 64, 64, 16, 16, 3, (64, 32, TAP), k=1),
        Enc("tap_1x1_stride2", 64, 64, 16, 16, 3, (64, 32, TAP), k=1, stride=2),
        # ---- SEAN decode shapes (batch 1)
        Enc("sean_1024_8x8", 1024, 1024, 8, 8, 1, (64, 32, TAP)),
        Enc("sean_gamma_beta_8x8", 128, 2048, 8, 8, 1, (64, 32, TAP), y32_only=True),
        Enc("sean_gamma_beta_16x16", 128, 2048, 16, 16, 1, (64, 32, SHIFT), y32_only=True),
        Enc("sean_conv_s_1x1", 1024, 512, 8, 8, 1, (64, 32, TAP), k=1),
    ]


def generator_cases(sms):
    return [
        Gen("plain_shift_kc64_n32", 64, 64, 16, 16, 3, 0, (64, 32, SHIFT)),
        Gen("plain_shift_kc64_n64_fill", 64, 64, 32, 32, _fill(sms, 8), 0, (64, 64, SHIFT)),
        Gen("plain_shift_kc32_n128_fill", 32, 128, 24, 48, _fill(sms, 9), 0, (32, 128, SHIFT)),
        Gen("plain_tap_kc64_8x8", 64, 64, 8, 8, 3, 0, (64, 32, TAP)),
        Gen("plain_tap_kc32_4x4", 32, 32, 4, 4, 9, 0, (32, 32, TAP)),
        Gen("up_shift_kc64", 64, 32, 16, 16, 3, 1, (64, 128, SHIFT)),
        Gen("up_shift_kc32_h24_w32", 32, 32, 24, 32, 2, 1, (32, 128, SHIFT)),
        Gen("up_tap_kc64_8x8", 64, 64, 8, 8, 3, 1, (64, 128, TAP)),
        Gen("up_tap_kc32_4x4", 32, 32, 4, 4, 5, 1, (32, 128, TAP)),
    ]


def _as_dict(out):
    return dict(zip(PLAN_FIELDS, out))


def encoder_plan(lib, c: Enc, dtype, batch=None):
    """Plan of the launch hf_conv2d_forward makes for `c` (dict of PLAN_FIELDS), or raises with the library's message."""
    d = lib.hf_conv2d_desc(c.cin, c.cout, c.cin if c.cin_pad is None else c.cin_pad, c.k, c.stride, c.groups, dtype)
    out = (C.c_int * 12)()
    rc = lib.lib().hf_conv2d_plan_query(C.byref(d), c.batch if batch is None else batch, c.h, c.w, out)
    if rc:
        raise RuntimeError(lib.lib().hf_last_error().decode())
    return _as_dict(out)


def generator_plan(lib, c: Gen, dtype):
    d = lib.hf_conv_desc(c.cin, c.cout, 3, c.up, dtype)
    out = (C.c_int * 12)()
    rc = lib.lib().hf_conv_plan_query(C.byref(d), c.batch, c.h, c.w, out)
    if rc:
        raise RuntimeError(lib.lib().hf_last_error().decode())
    return _as_dict(out)


def triple(plan):
    return (plan["kchunk"], plan["n_tile"], plan["a_slots"])


def check_claim(c, plan, sms):
    """The case runs the kernel variant it names (and, for the persistence cases, the schedule it needs)."""
    assert triple(plan) == c.plan, (c.name, "claims", c.plan, "gets", plan)
    assert plan["grid"] == min(plan["work"], sms), (c.name, plan, sms)
    if getattr(c, "min_tiles_per_cta", 0):
        assert plan["work"] >= c.min_tiles_per_cta * plan["grid"], (c.name, plan)
        kb = 9 * (c.cin // c.groups) // plan["kchunk"]
        assert kb % plan["stages"] != 0, (c.name, "k-blocks", kb, "stages", plan["stages"])
    if getattr(c, "n_tiles_per_m", 0):
        assert plan["n_n"] == c.n_tiles_per_m, (c.name, plan)

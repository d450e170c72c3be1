"""The case table of the exact-arithmetic convolution tests reaches every kernel variant `conv_plan` can choose, and
unsupported shapes come back as error codes with a message (no device needed).

Without a device the planner assumes the 132 SMs of an H100 SXM; tests/test_gpu_conv_exact.py repeats the claim
checks with the SM count of the device it runs on."""
import ctypes as C
import itertools

import pytest

from tests import conv_exact_cases as T

SMS = 132


@pytest.fixture(scope="module")
def lib():
    from hairfastgan_b200 import build
    build.build()
    from hairfastgan_b200 import _lib
    return _lib


def _reachable_encoder_triples(lib):
    """Every (kchunk, n_tile, mainloop) the planner gives over a sweep of encoder-form shapes."""
    seen = set()
    for cin, cout, (h, w), k, stride, groups, batch in itertools.product(
            (32, 64, 96, 128), (32, 64, 128, 192, 256), ((2, 2), (4, 4), (8, 8), (8, 16), (16, 16), (32, 32), (32, 64)),
            (1, 3), (1, 2), (1, 2), (1, 3, 40, 300)):
        if (cin // groups) % 32 or (cout // groups) % 32:
            continue
        c = T.Enc("sweep", cin, cout, h, w, batch, (0, 0, 0), k=k, stride=stride, groups=groups)
        seen.add(T.triple(T.encoder_plan(lib, c, lib.HF_BF16)))
    return seen


def _covered(lib, cases, plan_fn):
    got = {}
    for c in cases:
        for dtype in (lib.HF_BF16, lib.HF_F16):
            p = plan_fn(lib, c, dtype)
            T.check_claim(c, p, SMS)
            assert p["smem"] <= 232448 and p["stages"] >= 2, (c.name, p)
        got.setdefault(c.plan, []).append(c.name)
    return got


def test_encoder_cases_cover_every_kernel_variant(lib):
    reachable = _reachable_encoder_triples(lib)
    # two K chunk widths x three N tiles x two mainloops; a planner that learns a new tile or mainloop shows up here
    assert reachable == set(itertools.product((32, 64), (32, 64, 128), (T.SHIFT, T.TAP))), sorted(reachable)
    covered = _covered(lib, T.encoder_cases(SMS), T.encoder_plan)
    missing = sorted(reachable - set(covered))
    assert not missing, f"no exact-arithmetic case runs (kchunk, n_tile, mainloop) = {missing}"


def test_coverage_check_notices_a_removed_case(lib):
    """Without its only N = 128 per-tap case at 32-channel chunks the table no longer covers that kernel."""
    cases = [c for c in T.encoder_cases(SMS) if c.plan != (32, 128, T.TAP)]
    assert len(cases) < len(T.encoder_cases(SMS))
    assert (32, 128, T.TAP) in _reachable_encoder_triples(lib) - set(_covered(lib, cases, T.encoder_plan))


def test_encoder_cases_use_every_requested_form(lib):
    cases = T.encoder_cases(SMS)
    assert any(c.groups > 1 and c.plan[2] == T.SHIFT for c in cases) and any(c.groups > 1 and c.plan[2] == T.TAP
                                                                              for c in cases)
    assert any(c.cin_pad and c.cin_pad > c.cin for c in cases)
    assert {(c.k, c.stride) for c in cases} == {(1, 1), (1, 2), (3, 1), (3, 2)}
    assert any(c.n_tiles_per_m == 2 and c.min_tiles_per_cta >= 3 for c in cases)
    shift = [c for c in cases if c.plan[2] == T.SHIFT]
    assert {8, 24, 40} <= {c.h for c in shift} and {16, 48, 80} <= {c.w for c in shift}
    # part-empty last tiles on the maps that pack several samples into one tile
    for h, batches in ((4, {5, 9}), (8, {3}), (2, {3, 130})):
        assert batches <= {c.batch for c in cases if c.h == h and c.w == h}, (h, batches)
    # the filled N = 128 / 64 tiles stay cheap: at most 64 input channels per group
    for c in cases:
        if "fill" in c.name:
            assert c.cin // c.groups <= 64, c.name


def test_generator_cases_cover_plain_and_upsample_on_both_mainloops(lib):
    covered = _covered(lib, T.generator_cases(SMS), T.generator_plan)
    forms = {(c.plan[0], c.plan[2], c.up) for c in T.generator_cases(SMS)}
    assert forms == set(itertools.product((32, 64), (T.SHIFT, T.TAP), (0, 1))), sorted(forms)
    assert {32, 64, 128} <= {p[1] for p, names in covered.items()}
    assert all(c.plan[1] == 128 for c in T.generator_cases(SMS) if c.up)      # four parities in one 128-column tile


def test_generator_and_encoder_queries_agree_on_the_mainloop_field(lib):
    """out[4] is the activation ring depth of the column-shift mainloop in both queries; out[0] stays 0."""
    for r, want in ((8, T.TAP), (16, T.SHIFT), (64, T.SHIFT)):
        g = T.generator_plan(lib, T.Gen("g", 64, 64, r, r, 2, 0, (0, 0, 0)), lib.HF_BF16)
        e = T.encoder_plan(lib, T.Enc("e", 64, 64, r, r, 2, (0, 0, 0)), lib.HF_BF16)
        assert g["a_slots"] == e["a_slots"] == want and g["k0"] == e["k0"] == 0
        assert (g["kchunk"], g["stages"], g["smem"]) == (e["kchunk"], e["stages"], e["smem"])


# (cin, cout, cin_pad, k, stride, groups, H, W, message fragment)
REJECTED = [
    (64, 64, 64, 3, 1, 1, 16, 24, b"not divisible by tile"),            # W = 24: not a multiple of the 16-wide tile
    (64, 64, 64, 3, 1, 1, 16, 12, b"tile width must divide 128"),       # W = 12
    (64, 64, 64, 3, 1, 1, 12, 16, b"not divisible by tile"),            # H = 12 with W = 16 (8-row tiles)
    (64, 64, 64, 3, 2, 1, 15, 16, b"stride 2 needs even"),              # stride 2 with odd H
    (96, 64, 96, 3, 1, 2, 16, 16, b"multiple of 32 per group"),         # 48 input channels per group
    (64, 48, 64, 3, 1, 1, 16, 16, b"cout=48 must be a multiple of 32"),
]


@pytest.mark.parametrize("cin,cout,cin_pad,k,stride,groups,h,w,msg", REJECTED)
def test_unsupported_shapes_are_error_codes(lib, cin, cout, cin_pad, k, stride, groups, h, w, msg):
    hdl = lib.lib()
    d = lib.hf_conv2d_desc(cin, cout, cin_pad, k, stride, groups, lib.HF_BF16)
    out = (C.c_int * 12)(*([-7] * 12))
    assert hdl.hf_conv2d_plan_query(C.byref(d), 2, h, w, out) == -1
    assert msg in hdl.hf_last_error(), hdl.hf_last_error()
    assert list(out) == [-7] * 12                                        # nothing written on failure


def test_generator_query_rejections(lib):
    hdl = lib.lib()
    out = (C.c_int * 12)()
    d = lib.hf_conv_desc(64, 64, 3, 0, lib.HF_BF16)
    assert hdl.hf_conv_plan_query(C.byref(d), 2, 16, 24, out) == -1 and b"not divisible" in hdl.hf_last_error()
    assert hdl.hf_conv_plan_query(C.byref(d), 0, 16, 16, out) == -1 and b"bad shape" in hdl.hf_last_error()
    d = lib.hf_conv_desc(64, 64, 1, 1, lib.HF_BF16)                     # upsample needs the 3x3 kernel
    assert hdl.hf_conv_plan_query(C.byref(d), 2, 16, 16, out) == -1 and b"upsample" in hdl.hf_last_error()
    assert hdl.hf_conv2d_plan_query(None, 2, 16, 16, out) == -1 and b"null descriptor" in hdl.hf_last_error()
    d2 = lib.hf_conv2d_desc(64, 64, 64, 3, 1, 1, lib.HF_BF16)
    assert hdl.hf_conv2d_plan_query(C.byref(d2), 2, 16, 16, None) == -1 and b"null output" in hdl.hf_last_error()
    # Upsampling with groups (or stride 2) cannot be asked for: hf_conv_desc has no groups / stride and hf_conv2d_desc
    # has no upsample, so conv_plan's guard against the combination is unreachable through the C ABI.
    assert not {"groups", "stride"} & {f for f, _ in lib.hf_conv_desc._fields_}
    assert "upsample" not in {f for f, _ in lib.hf_conv2d_desc._fields_}

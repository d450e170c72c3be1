"""The case tables of tests/test_gpu_ops_exact.py reach every dispatch path of hf_upfirdn2d_f32, hf_bias_act_f32 and
fspace_blend_kernel, the Python restatements of those paths still match the host conditions in the sources, and the
float64 references agree with independent implementations (no device needed)."""
import os
import re

import torch
import torch.nn.functional as F

from tests import ops_exact_cases as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _source(name):
    return re.sub(r"\s+", " ", open(os.path.join(ROOT, "hairfastgan_b200", "csrc", name)).read())


def test_restated_host_conditions_match_the_sources():
    """The restatements in tests/ops_exact_cases.py copy these conditions; an edit here must be made there too."""
    ops, glue = _source("hf_ops.cu"), _source("hf_glue_ops.cu")
    for cond in [
        "const bool pads03 = px0 >= 0 && py0 >= 0 && px1 >= 0 && py1 >= 0 && px0 <= 3 && px1 <= 3 && py0 <= 3 && "
        "py1 <= 3;",
        "const bool bulk_ok = k4 && sym && planes <= 65535 && in_w >= 64 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 "
        "&& ((size_t)planes * in_h * in_w) % 4 == 0;",
        "if (bulk_ok && up_x == 1 && down_x == 1 && pads03 && out_w <= 1024 && in_w <= 1040) { if (out_w <= 512)",
        "} else if (bulk_ok && up_x == 1 && down_x == 2 && pads03 && out_w <= 1024 && in_w <= 1040) { if (out_w <= 512)",
        "} else if (bulk_ok && up_x == 2 && down_x == 1 && px0 == 2 && py0 == 2 && px1 == 1 && py1 == 1 && in_w <= 1024 "
        "&& (reinterpret_cast<uintptr_t>(y) & 7) == 0) { if (in_w <= 512)",
        "separable = separable && fabsf(ky[a] * kx[b] - kr[a * 4 + b]) <= 1e-6f * fabsf(kr[a * 4 + b]) + 1e-30f;",
        "if (step_b % 4 == 0 && step_b >= 1024 && n % step_b == 0 && n / step_b <= 65535 && step_b / 4 < (int64_t)2000000000"
        " && ((((uintptr_t)x | (uintptr_t)y) & 15) == 0)) {",
        "const int gx = std::max(1, std::min(cdiv(quads, 256), std::max(1, num_sms() * 16 / planes)));",
        "const bool vec = (step_b % 4 == 0) && (n % 4 == 0) && ((((uintptr_t)x | (uintptr_t)y) & 15) == 0);",
    ]:
        assert cond in ops, cond
    for cond in ["const bool vec = a.aligned && (P % 4 == 0) && (p0 + lane4 + 3 < P);",
                 "a.aligned = (bits & 15) == 0;"]:
        assert cond in glue, cond
    assert "return (int)std::min<int64_t>((n + 255) / 256, (int64_t)num_sms() * 16);" in _source("hf_common.cuh")


def _covered(ids):
    return {i.split("-", 1)[0] for i in ids}


def test_upfirdn_cases_reach_every_kernel():
    paths = _covered(map(T.upfirdn_id, T.UPFIRDN_EXACT))
    assert paths == set(T.UPFIRDN_PATHS), sorted(set(T.UPFIRDN_PATHS) - paths)
    assert {T.upfirdn_path(u) for u in T.UPFIRDN_BOUNDED} == {"bulk_d1_nc2_sep", "bulk_d2_nc2_sep"}


def test_coverage_check_notices_a_removed_case():
    cases = [u for u in T.UPFIRDN_EXACT if T.upfirdn_path(u) != "bulk_d2_nc4_gen"]
    assert len(cases) < len(T.UPFIRDN_EXACT)
    assert "bulk_d2_nc4_gen" in set(T.UPFIRDN_PATHS) - _covered(map(T.upfirdn_id, cases))


def test_upfirdn_cases_sit_on_every_column_boundary():
    """out_w 255 / 256 / 257 / 511 / 512 (2 columns per thread) and 513 plus the widest (4 columns) for down 1 and
    down 2, each with both FIR loops; in_w at the same boundaries for up 2."""
    got = {}
    for u in T.UPFIRDN_EXACT:
        p = T.upfirdn_path(u)
        width = u.in_w if p.startswith("bulk_up2") else T.upfirdn_out(u)[1]
        got.setdefault(p, set()).add(width)
    for d, top in ((1, 1024), (2, 521)):
        for fir in ("sep", "gen"):
            assert {255, 256, 257, 511, 512} <= got[f"bulk_d{d}_nc2_{fir}"], (d, fir)
            assert {513, top} <= got[f"bulk_d{d}_nc4_{fir}"], (d, fir)
    assert {255, 256, 257, 511, 512} <= got["bulk_up2_nc2"] and {513, 1024} <= got["bulk_up2_nc4"]


def test_upfirdn_cases_reach_the_pipeline_edges():
    bulk = [u for u in T.UPFIRDN_EXACT if T.upfirdn_path(u) != "general"]
    for d in (1, 2):
        rows = {T.upfirdn_out(u)[0] for u in bulk if u.up_x == 1 and u.down_x == d}
        strip = 64 if d == 1 else 32
        assert 1 in rows and any(r % strip for r in rows) and any(r >= strip for r in rows), (d, rows)
        # a full strip: DOWN * RS + HALO rows in 4-row chunks = 17 chunks, so each of the 3 stages flips its phase
        assert -(-(d * strip + (3 if d == 1 else 2)) // 4) >= 7
        assert any(u.in_h == 1 for u in bulk if u.up_x == 1 and u.down_x == d)
    assert any(u.in_h == 1 for u in bulk if u.up_x == 2) and any(u.in_h > 32 for u in bulk if u.up_x == 2)
    for kind in ("d1", "d2", "up2"):
        mods = {u.in_h * u.in_w % 4 for u in bulk if u.name.startswith(kind) and u.planes > 1}
        assert mods == {0, 1, 2, 3}, (kind, mods)


def test_upfirdn_general_triggers_one_each():
    gen = {u.name: u for u in T.UPFIRDN_EXACT if u.name.startswith("gen_")}
    assert all(T.upfirdn_path(u) == "general" for u in gen.values())
    # each trigger alone: undoing it gives back a bulk kernel
    undo = {"gen_x_not_16B_aligned": dict(x_off=0), "gen_total_not_mult4": dict(planes=4),
            "gen_in_w63": dict(in_w=64), "gen_in_w1044": dict(in_w=1040), "gen_pad_m1": dict(px0=1, py1=1),
            "gen_pad_4": dict(px0=3, py1=3), "gen_up_x_ne_up_y": dict(up_y=2, py0=2),
            "gen_down_x_ne_down_y": dict(down_x=2), "gen_up2_y_not_8B_aligned": dict(y_off=0),
            "gen_up2_pad_12": dict(px0=2, px1=1, py0=2, py1=1), "gen_planes_65536": dict(planes=65535)}
    for name, fix in undo.items():
        assert T.upfirdn_path(gen[name]._replace(**fix)) != "general", name
    assert gen["gen_over_one_grid"].planes * T.upfirdn_out(gen["gen_over_one_grid"])[0] * \
        T.upfirdn_out(gen["gen_over_one_grid"])[1] > T.grid_threads(T.SMS)
    assert {(u.kh, u.kw) for u in gen.values()} >= {(1, 1), (3, 5), (4, 4)}


def test_fir_restatement_and_tap_designs():
    for u in T.UPFIRDN_EXACT + T.UPFIRDN_BOUNDED:
        k = T.upfirdn_taps(u)
        assert torch.equal(k.float().double(), k)
        if u.kh == u.kw == 4:
            assert T.fir_separable(k) == (u.fir != "gen"), u.name
        if u.fir == "gen":
            assert k.unique().numel() == k.numel(), u.name
        if u.fir in ("sep", "near"):                    # dyadic ratios: the separable loop is exact
            kr = T.rank1_part(k).flip(0, 1)
            assert torch.equal(kr[:, 0] / kr[0, 0], (kr[:, 0] / kr[0, 0]).float().double())
        if u.fir == "near":
            rel = ((k - T.rank1_part(k)).abs() / k.abs()).max()
            assert 4e-7 < rel < 1e-6 and (k != T.rank1_part(k)).sum() == 1


def test_bias_act_cases_reach_every_path():
    ids = [T.bias_act_id(c) for c in T.BIAS_ACT]
    assert _covered(ids) == set(T.BIAS_ACT_PATHS), sorted(set(T.BIAS_ACT_PATHS) - _covered(ids))
    nobias = {T.bias_act_id(c).split("-")[0].replace("_stride", "") for c in T.BIAS_ACT if c.bias == "none"}
    assert nobias == {"plane", "flat_vec", "scalar"}
    assert {c.act for c in T.BIAS_ACT} == {1, 3} and {len(c.shape) for c in T.BIAS_ACT} == {2, 3, 4}
    assert any(c.shape[0] > 1 and c.bias == "odd3" for c in T.BIAS_ACT)
    assert any((c.alpha, c.scale) != (0.2, 2 ** 0.5) for c in T.BIAS_ACT)
    assert any(c.x_off % 16 for c in T.BIAS_ACT) and any(c.y_off % 16 for c in T.BIAS_ACT)
    assert any(T.bias_act_dims(c)[0] // T.bias_act_dims(c)[2] > 65535 for c in T.BIAS_ACT)


def test_fspace_cases_reach_every_path_and_form():
    ids = [T.fspace_id(c) for c in T.FSPACE]
    assert _covered(ids) == set(T.FSPACE_PATHS)
    ratios = {(c.Hm / c.Ho, c.Wm / c.Wo) for c in T.FSPACE}
    assert {(8, 8), (4, 4), (2, 2), (0.5, 0.5), (1, 1)} <= ratios and any(a != b for a, b in ratios)
    assert {c.stages for c in T.FSPACE} == {1, 2, 3, 4}
    assert any(c.C % 4 for c in T.FSPACE) and any(c.C % 16 and not c.C % 4 for c in T.FSPACE)
    assert any(c.stages == 4 and c.ref == "ffma" and c.Hm == 256 for c in T.FSPACE)


def test_upfirdn_reference_matches_the_oracle():
    """Per-axis restatement == oracle.stylegan2_oracle.upfirdn2d_ref (one up / down / pad for both axes)."""
    from oracle import stylegan2_oracle as O
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, 9, 11, generator=g).double()
    k = torch.randn(4, 4, generator=g).double()
    for up, down, pad in [(1, 1, (1, 1)), (2, 1, (2, 1)), (1, 2, (1, 1)), (3, 2, (2, 3)), (1, 1, (-1, 1))]:
        ref = O.upfirdn2d_ref(x, k, up, down, pad).reshape(6, *O.upfirdn2d_ref(x, k, up, down, pad).shape[2:])
        mine = T.upfirdn_ref(x.reshape(6, 9, 11), k, up, up, down, down, pad[0], pad[1], pad[0], pad[1])
        assert torch.allclose(mine, ref, rtol=0, atol=1e-12), (up, down, pad)
    # x and y independent: transposing the input and the taps swaps the axes' parameters
    a = T.upfirdn_ref(x[0], k, 2, 1, 1, 2, 2, 1, 0, 3)
    b = T.upfirdn_ref(x[0].transpose(1, 2), k.t(), 1, 2, 2, 1, 0, 3, 2, 1)
    assert torch.allclose(a, b.transpose(1, 2), rtol=0, atol=1e-12)


def test_bicubic_reference_matches_the_oracle():
    from oracle import glue_oracle as GO
    g = torch.Generator().manual_seed(4)
    x = torch.rand(1, 3, 40, 56, generator=g) * 255
    for f in (1, 2, 3, 4, 8):
        k = GO.bicubic_taps(f).double()
        for clip in (False, True):
            ref = GO.bicubic_downsample_ref(x, f, clip).double()
            mine = T.bicubic_ref(x[0].double(), k, f, clip)[None]
            assert torch.allclose(mine, ref, rtol=0, atol=1.0 if clip else 1e-4), (f, clip)
            if clip:                                   # the oracle rounds fp32 values: ties may differ by one
                assert (mine != ref).float().mean() < 1e-2


def test_bicubic_interp_reference_matches_torch():
    """Exact against F.interpolate(bicubic) in float64 on dyadic masks at the dyadic ratios of the cases, and within
    1e-13 on random masks at any ratio (summation order)."""
    g = torch.Generator().manual_seed(5)
    for c in T.FSPACE:
        m = torch.randint(0, 4, (c.Hm, c.Wm), generator=g).double() / 4
        want = F.interpolate(m[None, None], (c.Ho, c.Wo), mode="bicubic", align_corners=False)[0, 0]
        assert torch.equal(T.bicubic_interp_ref(m, c.Ho, c.Wo), want), c.name
    for hm, wm, ho, wo in [(50, 70, 20, 12), (7, 9, 23, 5), (256, 256, 32, 32)]:
        m = torch.rand(hm, wm, generator=g, dtype=torch.float64)
        want = F.interpolate(m[None, None], (ho, wo), mode="bicubic", align_corners=False)[0, 0]
        assert (T.bicubic_interp_ref(m, ho, wo) - want).abs().max() < 1e-13

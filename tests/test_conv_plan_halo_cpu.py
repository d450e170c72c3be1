"""Plan of the wgmma convolution for the generator layers (no device needed): the stride-1 3x3 layers whose tile is
16 pixels wide and one sample high load one activation box per column shift, which leaves room for a weight ring of
at least 4 slots at n_tile 128; the small layers keep one activation + weight box per k-block (3 slots)."""
import ctypes as C

import pytest

LAYERS = [(512, 512, 4, 0), (512, 512, 4, 1), (512, 512, 8, 0), (512, 512, 8, 1), (512, 512, 16, 0),
          (512, 512, 16, 1), (512, 512, 32, 0), (512, 512, 32, 1), (512, 512, 64, 0), (512, 256, 64, 1),
          (256, 256, 128, 0), (256, 128, 128, 1), (128, 128, 256, 0), (128, 64, 256, 1), (64, 64, 512, 0),
          (64, 32, 512, 1), (32, 32, 1024, 0)]


@pytest.fixture(scope="module")
def lib():
    from hairfastgan_b200 import build
    build.build()
    from hairfastgan_b200 import _lib
    return _lib


def _plan(lib, cin, cout, r, up, batch, dtype):
    d = lib.hf_conv_desc(cin, cout, 3, up, dtype)
    out = (C.c_int * 12)()
    assert lib.lib().hf_conv_plan_query(C.byref(d), batch, r, r, out) == 0, lib.lib().hf_last_error()
    return dict(zip(("halo", "n_tile", "n_n", "G", "na", "pitch", "res", "stages", "smem", "work", "grid", "kchunk"),
                    out))


@pytest.mark.parametrize("batch", [1, 3, 96])
def test_weight_ring_depth_by_path(lib, batch):
    for cin, cout, r, up in LAYERS:
        for dtype in (lib.HF_BF16, lib.HF_F16):
            p = _plan(lib, cin, cout, r, up, batch, dtype)
            assert p["smem"] <= 232448
            if p["n_tile"] != 128:
                continue
            if r >= 16:          # column-shift boxes: 2 x 20 KB activation slots + 16 KB weight slots
                assert p["stages"] >= 4, (cin, cout, r, up, p)
            else:                # 8-pixel-wide tiles: 32 KB (activation + weight) slots
                assert p["stages"] == 3, (cin, cout, r, up, p)


def test_column_shift_smem_layout(lib):
    """512->512 @64^2: 2 activation slots of (8 + 2) x 16 x 64 x 2 B, five 16 KB weight slots."""
    p = _plan(lib, 512, 512, 64, 0, 96, lib.HF_BF16)
    fixed = 1024 + 2 * 64 * 132 * 4 + 2 * 16384 + 2 * 64 * 4 * 4 + 2 * (8 + 2) * 8
    assert (p["stages"], p["smem"]) == (5, fixed + 2 * 20480 + 5 * 16384)

"""GPU parity of the wgmma ModulatedConv2d / StyledConv / ToRGB path (through hf_conv_forward /
hf_torgb_forward) against the CPU oracle and the reference-generated golden vectors."""
import os

import numpy as np
import pytest
import torch

from oracle import stylegan2_oracle as O
from tests.gpu_util import TOL_SINGLE, dtype_name, record, rel_err

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture(scope="module")
def M():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import hairfastgan_b200.model as M
    return M


def _load_case(golden_dir, name):
    g = np.load(os.path.join(golden_dir, "modules.npz"))
    p = {k.split("__p__")[1]: torch.from_numpy(g[k]) for k in g.files if k.startswith(name + "__p__")}
    return g, p


@pytest.mark.parametrize("name,cin,cout,up", [("plain_64_48_r8", 64, 48, False), ("up_64_32_r8", 64, 32, True),
                                              ("plain_32_32_r16", 32, 32, False)])
def test_styled_conv_golden(M, golden_dir, name, cin, cout, up):
    if cout % 32:
        pytest.skip("tensor-core path needs Cout % 32 == 0 (every generator layer satisfies this)")
    g, p = _load_case(golden_dir, name)
    m = M.StyledConv(cin, cout, 3, 512, upsample=up).cuda()
    m.load_state_dict(p, strict=True)
    x = torch.from_numpy(g[name + "__x"]).cuda()
    st = torch.from_numpy(g[name + "__style"]).cuda()
    nz = torch.from_numpy(g[name + "__noise"]).cuda()
    tol = TOL_SINGLE[dtype_name()]
    e, rms = rel_err(m.conv(x, st), torch.from_numpy(g[name + "__modconv"]))
    record("modconv_golden_" + name, rel_max_err=e, ref_rms=rms)
    assert e < tol, e
    e, rms = rel_err(m(x, st, noise=nz), torch.from_numpy(g[name + "__styled"]))
    record("styled_golden_" + name, rel_max_err=e, ref_rms=rms)
    assert e < tol, e


def _rand_styled(M, cin, cout, up, seed):
    torch.manual_seed(seed)
    m = M.StyledConv(cin, cout, 3, 512, upsample=up)
    m.noise.weight.data.normal_(0, 0.3)
    m.activate.bias.data.normal_(0, 0.3)
    m.conv.modulation.bias.data.add_(0.1 * torch.randn(cin))
    return m


# every (Cin, Cout, R_in, up) shape class of the 1024^2 generator (SURVEY Appendix A), small batch
LAYER_SHAPES = [
    (512, 512, 4, False, 3), (512, 512, 4, True, 3), (512, 512, 8, False, 2), (512, 512, 16, True, 1),
    (512, 512, 32, False, 1), (512, 256, 64, True, 1), (256, 256, 128, False, 1), (256, 128, 128, True, 1),
    (128, 128, 256, False, 1), (128, 64, 256, True, 1), (64, 64, 512, False, 1), (64, 32, 512, True, 1),
    (32, 32, 1024, False, 1),
]


@pytest.mark.parametrize("cin,cout,r,up,batch", LAYER_SHAPES)
def test_styled_conv_layer_shapes_vs_oracle(M, cin, cout, r, up, batch):
    m = _rand_styled(M, cin, cout, up, seed=cin + r)
    g = torch.Generator().manual_seed(r)
    x = torch.randn(batch, cin, r, r, generator=g)
    st = torch.randn(batch, 512, generator=g)
    ro = 2 * r if up else r
    nz = torch.randn(batch, 1, ro, ro, generator=g)
    p = {k: v for k, v in m.state_dict().items()}
    ref = O.styled_conv_ref(x, st, p, "", nz, up)
    y = m.cuda()(x.cuda(), st.cuda(), noise=nz.cuda())
    assert y.shape == ref.shape
    e, rms = rel_err(y, ref)
    record(f"styled_{cin}_{cout}_r{r}_up{int(up)}", rel_max_err=e, ref_rms=rms)
    assert e < TOL_SINGLE[dtype_name()], e


def test_config1_modconv512_golden(M, golden_dir):
    """BASELINE.json configs[0]: ModulatedConv2d 512ch@64^2 B=1, inputs re-derived from seed 0."""
    g = np.load(os.path.join(golden_dir, "config1_modconv512.npz"))
    torch.manual_seed(0)
    m = M.ModulatedConv2d(512, 512, 3, 512)
    m.modulation.weight.data.normal_()
    x = torch.randn(1, 512, 64, 64); st = torch.randn(1, 512)
    assert np.allclose(m.weight[0, ::64, ::64].detach().numpy(), g["weight_sub"])
    y = m.cuda()(x.cuda(), st.cuda())
    ref = torch.from_numpy(g["y_sub"])
    e, rms = rel_err(y[:, ::8, ::4, ::4], ref)
    record("config1_modconv512", rel_max_err=e, ref_rms=rms)
    assert e < TOL_SINGLE[dtype_name()], e


def test_noise_broadcast_and_random(M):
    """noise of batch 1 broadcasts (registered buffers, model.py:426-427); noise=None draws from torch's
    generator at the same point as the reference (model.py:288-291)."""
    m = _rand_styled(M, 64, 64, False, 1).cuda()
    x = torch.randn(3, 64, 16, 16, device="cuda"); st = torch.randn(3, 512, device="cuda")
    nz = torch.randn(1, 1, 16, 16, device="cuda")
    a = m(x, st, noise=nz)
    b = m(x, st, noise=nz.expand(3, 1, 16, 16).contiguous())
    assert torch.equal(a, b)
    torch.manual_seed(7)
    c = m(x, st)
    torch.manual_seed(7)
    nz2 = x.new_empty(3, 1, 16, 16).normal_()
    assert torch.equal(c, m(x, st, noise=nz2))


def test_to_rgb(M, golden_dir):
    g, p = _load_case(golden_dir, "torgb")
    m = M.ToRGB(64, 512).cuda()
    m.load_state_dict(p, strict=True)
    x = torch.from_numpy(g["torgb__x"]).cuda(); st = torch.from_numpy(g["torgb__style"]).cuda()
    sk = torch.from_numpy(g["torgb__skip"]).cuda()
    assert float((m(x, st, sk).cpu() - torch.from_numpy(g["torgb__y_skip"])).abs().max()) < 1e-4
    assert float((m(x, st, None).cpu() - torch.from_numpy(g["torgb__y_noskip"])).abs().max()) < 1e-4


def test_determinism(M):
    m = _rand_styled(M, 128, 128, False, 2).cuda()
    x = torch.randn(2, 128, 64, 64, device="cuda"); st = torch.randn(2, 512, device="cuda")
    nz = torch.randn(2, 1, 64, 64, device="cuda")
    assert torch.equal(m(x, st, noise=nz), m(x, st, noise=nz))

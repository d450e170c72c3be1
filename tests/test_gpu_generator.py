"""GPU parity of Generator.forward (hf_generator_forward) -- every partial range swap() uses --
against the CPU oracle, the golden vectors produced by the unmodified reference, and size-independent
properties at the full BASELINE configuration (1024^2, B=4)."""
import os

import numpy as np
import pytest
import torch

from oracle import stylegan2_oracle as O
from tests.gpu_util import TOL_RGB, TOL_SINGLE, dtype_name, record, rel_err

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture(scope="module")
def M():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import hairfastgan_b200.model as M
    return M


@pytest.fixture(scope="module")
def gen256(M):
    g = M.Generator(256, 512, 8)
    g.load_state_dict(O.synth_generator_params(size=256, seed=0), strict=True)
    return g.cuda().eval()


def _cuda_list(ts):
    return [t.cuda() for t in ts]


def test_generator256_golden_all_ranges(M, gen256, golden_dir):
    g = np.load(os.path.join(golden_dir, "generator256.npz"))
    lat = torch.from_numpy(g["latent"]).cuda()
    noise = _cuda_list(O.synth_noise(256, batch=2, seed=3))
    tol, tol1 = TOL_RGB[dtype_name()], TOL_SINGLE[dtype_name()] * 3

    img, none = gen256([lat], input_is_latent=True, noise=noise)
    assert none is None and img.shape == (2, 3, 256, 256)
    e, rms = rel_err(img[:, :, ::4, ::4], torch.from_numpy(g["full__image"]))
    record("gen256_full", rel_max_err=e, ref_rms=rms, abs_max_err=e * rms)
    assert e < tol, e

    f, s = gen256([lat], input_is_latent=True, noise=noise, start_layer=0, end_layer=3)
    assert f.shape == (2, 512, 32, 32) and s.shape == (2, 3, 32, 32)
    e, _ = rel_err(f[:, ::8], torch.from_numpy(g["r0_3__out"])); assert e < tol1, e
    e, _ = rel_err(s, torch.from_numpy(g["r0_3__skip"])); assert e < tol, e

    g2 = torch.Generator().manual_seed(4)
    lin16 = torch.randn(2, 512, 16, 16, generator=g2).cuda()
    f, s = gen256([lat], input_is_latent=True, noise=noise, start_layer=3, end_layer=3, layer_in=lin16)
    e, _ = rel_err(f[:, ::8], torch.from_numpy(g["r3_3__out"])); assert e < tol1, e
    e, _ = rel_err(s, torch.from_numpy(g["r3_3__skip"])); assert e < tol, e

    lin32 = torch.randn(2, 512, 32, 32, generator=g2).cuda()
    img, _ = gen256([lat], input_is_latent=True, noise=noise, start_layer=4, end_layer=8, layer_in=lin32)
    e, rms = rel_err(img[:, :, ::4, ::4], torch.from_numpy(g["r4_end__image"]))
    record("gen256_r4_end", rel_max_err=e, ref_rms=rms)
    assert e < tol, e

    lin64 = torch.randn(2, 512, 64, 64, generator=g2).cuda()
    img, _ = gen256([lat], input_is_latent=True, noise=noise, start_layer=5, end_layer=8, layer_in=lin64)
    e, _ = rel_err(img[:, :, ::4, ::4], torch.from_numpy(g["r5_end__image"])); assert e < tol, e

    img, _ = gen256([lat[:1]], input_is_latent=True, randomize_noise=False)
    e, _ = rel_err(img[:, :, ::4, ::4], torch.from_numpy(g["bufnoise__image"])); assert e < tol, e

    z = torch.from_numpy(g["z"]).cuda()
    assert float((gen256.get_latent(z).cpu() - torch.from_numpy(g["mapping__w"])).abs().max()) < 1e-3


def test_generator_skip_argument_and_end0(M, gen256):
    """forward(skip=...) with start_layer>0 (model.py:546-547) and the end_layer=0 early exit (:537)."""
    p = O.synth_generator_params(size=256, seed=0)
    g = torch.Generator().manual_seed(9)
    lat = torch.randn(1, 14, 512, generator=g)
    noise = O.synth_noise(256, batch=1, seed=5)
    lin = torch.randn(1, 512, 8, 8, generator=g); sk = torch.randn(1, 3, 8, 8, generator=g)
    rf, rs = O.generator_ref(p, lat, noise, 2, 2, layer_in=lin, skip=sk)
    f, s = gen256([lat.cuda()], input_is_latent=True, noise=_cuda_list(noise), start_layer=2, end_layer=2,
                  layer_in=lin.cuda(), skip=sk.cuda())
    assert rel_err(f, rf)[0] < TOL_SINGLE[dtype_name()] * 3 and rel_err(s, rs)[0] < TOL_RGB[dtype_name()]
    rf, rs = O.generator_ref(p, lat, noise, 0, 0)
    f, s = gen256([lat.cuda()], input_is_latent=True, noise=_cuda_list(noise), start_layer=0, end_layer=0)
    assert f.shape == (1, 512, 4, 4) and s.shape == (1, 3, 4, 4)
    assert rel_err(f, rf)[0] < TOL_SINGLE[dtype_name()] and rel_err(s, rs)[0] < TOL_RGB[dtype_name()]


def test_generator_random_noise_order_matches_reference(M, gen256):
    """randomize_noise=True draws one N(0,1) tensor per executed StyledConv, in execution order, from
    torch's CUDA generator (model.py:288-291): reproduce the draws and compare to the explicit path."""
    lat = torch.randn(2, 14, 512, device="cuda")
    torch.manual_seed(3407)
    a, _ = gen256([lat], input_is_latent=True)
    torch.manual_seed(3407)
    noise = [lat.new_empty(2, 1, 4, 4).normal_()]
    for i in range(3, 9):
        for _ in range(2):
            noise.append(lat.new_empty(2, 1, 2 ** i, 2 ** i).normal_())
    b, _ = gen256([lat], input_is_latent=True, noise=noise)
    assert torch.equal(a, b)


def test_generator1024_golden_and_batch_properties(M, golden_dir):
    """BASELINE configs[1]: 1024^2 generator.  B=1 against the reference golden; B=4 through
    size-independent properties: run-to-run determinism (bit for bit) and batch independence (sample i of a
    B=4 run == the same sample run alone, up to the fp32 re-association of the ToRGB partial sums, whose
    grouping follows the N-tile width chosen for the batch)."""
    g = np.load(os.path.join(golden_dir, "generator1024.npz"))
    gen = M.Generator(1024, 512, 8)
    gen.load_state_dict(O.synth_generator_params(size=1024, seed=0), strict=True)
    gen = gen.cuda().eval()
    lat = torch.randn(1, 18, 512, generator=torch.Generator().manual_seed(0)).cuda()
    noise = _cuda_list(O.synth_noise(1024, batch=1, seed=1))
    img, _ = gen([lat], input_is_latent=True, noise=noise)
    assert img.shape == (1, 3, 1024, 1024)
    e, rms = rel_err(img[:, :, ::16, ::16], torch.from_numpy(g["image_sub"]))
    e2, _ = rel_err(img[:, :, 511:513], torch.from_numpy(g["image_rows"]))
    record("gen1024_full_b1", rel_max_err=max(e, e2), ref_rms=rms, abs_max_err=max(e, e2) * rms,
           ref_absmax=float(g["image_absmax"]))
    assert max(e, e2) < TOL_RGB[dtype_name()], (e, e2)

    lat4 = torch.randn(4, 18, 512, generator=torch.Generator().manual_seed(1)).cuda()
    lat4[0] = lat[0]
    img4, _ = gen([lat4], input_is_latent=True, noise=noise)      # shared [1,1,R,R] noise broadcasts
    img4b, _ = gen([lat4], input_is_latent=True, noise=noise)
    assert torch.equal(img4, img4b)
    assert float((img4[0] - img[0]).abs().max()) < 1e-4
    one, _ = gen([lat4[3:4]], input_is_latent=True, noise=noise)
    assert float((img4[3] - one[0]).abs().max()) < 1e-4


# north_star: "max-abs on generator RGB".  Stated ABSOLUTE tolerance on a unit-range image (RGB in [-1, 1], what a
# trained generator emits): bf16 operands 1.5e-2, fp16 operands 2e-3.
TOL_RGB_ABS_UNIT = {"bf16": 1.5e-2, "fp16": 2e-3}


def test_generator1024_unit_range_rgb_max_abs(M, golden_dir):
    """The reference golden of the synthetic 1024^2 generator spans +-8.9; the image is LINEAR in the ToRGB weights
    and biases (rgb = sum over layers of Up(W_rgb (s' x) + b), model.py:356-365), so scaling all of them by
    alpha = 1 / max|golden| gives exactly alpha * golden from the reference -- a unit-range image with a known
    answer, on which the max-abs error is asserted in absolute terms."""
    g = np.load(os.path.join(golden_dir, "generator1024.npz"))
    alpha = 1.0 / float(g["image_absmax"])
    params = O.synth_generator_params(size=1024, seed=0)
    for k in params:
        if k.startswith("to_rgb") and (k.endswith("conv.weight") or k.endswith(".bias") and params[k].ndim == 4):
            params[k] = params[k] * alpha
    gen = M.Generator(1024, 512, 8)
    gen.load_state_dict(params, strict=True)
    gen = gen.cuda().eval()
    lat = torch.randn(1, 18, 512, generator=torch.Generator().manual_seed(0)).cuda()
    noise = _cuda_list(O.synth_noise(1024, batch=1, seed=1))
    img, _ = gen([lat], input_is_latent=True, noise=noise)
    ref_sub, ref_rows = torch.from_numpy(g["image_sub"]) * alpha, torch.from_numpy(g["image_rows"]) * alpha
    assert float(ref_sub.abs().max()) <= 1.0 + 1e-6
    err = max(float((img[:, :, ::16, ::16].cpu() - ref_sub).abs().max()),
              float((img[:, :, 511:513].cpu() - ref_rows).abs().max()))
    record("gen1024_unit_range_abs", abs_max_err=err, range="[-1,1]")
    assert err < TOL_RGB_ABS_UNIT[dtype_name()], err


def test_fse_generator_variant_golden(M, golden_dir):
    """SURVEY 8 row a12: the FeatureStyleEncoder generator copy (features_in at idx 5, feature_scale=1,
    return_features=True) -- the call Trainer.get_image makes (trainer.py:295)."""
    import hairfastgan_b200.fse_model as FM
    g = np.load(os.path.join(golden_dir, "generator256_fse.npz"))
    gen = FM.Generator(256, 512, 8)
    gen.load_state_dict(O.synth_generator_params(size=256, seed=0), strict=True)
    gen = gen.cuda().eval()
    lat = torch.from_numpy(np.load(os.path.join(golden_dir, "generator256.npz"))["latent"]).cuda()
    noise = _cuda_list(O.synth_noise(256, batch=2, seed=3))
    fea = torch.randn(2, 512, 16, 16, generator=torch.Generator().manual_seed(6)).cuda()
    img, outs = gen([lat], input_is_latent=True, noise=noise, return_features=True,
                    features_in=[None] * 5 + [fea] + [None] * 12, feature_scale=1.0)
    assert len(outs) == int(g["n_outs"])
    tol, tol1 = TOL_RGB[dtype_name()], TOL_SINGLE[dtype_name()] * 3
    e, rms = rel_err(img[:, :, ::4, ::4], torch.from_numpy(g["image"]))
    record("gen256_fse_variant", rel_max_err=e, ref_rms=rms)
    assert e < tol, e
    assert float((outs[0][:, ::64].cpu() - torch.from_numpy(g["out0"])).abs().max()) < 1e-6
    for key, sl in [("out4", (slice(None), slice(None, None, 16))), ("out5", (slice(None), slice(None, None, 16))),
                    ("out6", (slice(None), slice(None, None, 16), slice(None, None, 2), slice(None, None, 2))),
                    ("out_last", (slice(None), slice(None, None, 16), slice(None, None, 8), slice(None, None, 8)))]:
        idx = {"out4": 4, "out5": 5, "out6": 6, "out_last": -1}[key]
        e, _ = rel_err(outs[idx][sl], torch.from_numpy(g[key]))
        assert e < tol1, (key, e)
    # plain call without features must equal the main Generator
    img2, none = gen([lat], input_is_latent=True, noise=noise)
    assert none is None
    with pytest.raises(RuntimeError, match="feature_scale == 1.0"):
        gen([lat], input_is_latent=True, noise=noise, features_in=[None] * 5 + [fea] + [None] * 12, feature_scale=0.5)


def test_consume_noise_advances_rng_like_a_forward():
    """The opt-in FSE fast path (fse_fast.py, SURVEY 8f-2) skips a full forward but must leave the random stream
    where the reference would: consume_noise() == the draws of forward(randomize_noise=True)."""
    import hairfastgan_b200.fse_model as FM
    torch.manual_seed(0)
    gen = FM.Generator(256, 512, 8).cuda().eval()
    lat = torch.randn(3, gen.n_latent, 512, device="cuda")
    torch.manual_seed(123)
    gen([lat], input_is_latent=True, return_features=True)             # random noise, like Trainer.get_image
    after_forward = torch.randn(1000, device="cuda")
    torch.manual_seed(123)
    gen.consume_noise(3)
    after_skip = torch.randn(1000, device="cuda")
    assert torch.equal(after_forward, after_skip)
    torch.manual_seed(123)                                              # control: without the draws the stream differs
    assert not torch.equal(after_forward, torch.randn(1000, device="cuda"))


def test_generator_cuda_graph_replay_keeps_outputs_and_rng(M, gen256):
    """graphs.py on the generator: call 1 eager, call 2 captures (17 normal_() draws inside the graph), later calls
    replay.  Under a fixed seed every call must give the eager image bit for bit AND leave torch's CUDA generator where
    the eager forward leaves it (the next draw is identical); partial ranges with layer_in likewise."""
    from hairfastgan_b200 import graphs
    lat = torch.randn(2, 14, 512, device="cuda")
    os.environ["HAIRFAST_CUDA_GRAPHS"] = "0"
    try:
        torch.manual_seed(3407)
        want, _ = gen256([lat], input_is_latent=True)
        after_want = torch.randn(64, device="cuda")
        lin = torch.randn(2, 512, 16, 16, device="cuda")
        torch.manual_seed(11)
        want_part = gen256([lat], input_is_latent=True, start_layer=3, end_layer=4, layer_in=lin)
    finally:
        os.environ.pop("HAIRFAST_CUDA_GRAPHS")
    gen256.__dict__.pop("_hf_graphs", None)
    s0 = graphs.stats()
    for _ in range(4):
        torch.manual_seed(3407)
        got, _ = gen256([lat], input_is_latent=True)
        after = torch.randn(64, device="cuda")
        assert torch.equal(got, want) and torch.equal(after, after_want)
    for _ in range(3):
        torch.manual_seed(11)
        feat, skip = gen256([lat], input_is_latent=True, start_layer=3, end_layer=4, layer_in=lin)
        assert torch.equal(feat, want_part[0]) and torch.equal(skip, want_part[1])
    s1 = graphs.stats()
    assert s1["captures"] >= s0["captures"] + 2 and s1["replays"] >= s0["replays"] + 5 and s1["failed"] == s0["failed"]
    lat2 = torch.randn(2, 14, 512, device="cuda")                 # same signature, other data
    torch.manual_seed(3407)
    other, _ = gen256([lat2], input_is_latent=True)
    assert not torch.equal(other, want)

"""GPU bring-up diagnostics for the wgmma conv kernel: runs a ladder of ModulatedConv2d cases from
a bare 1x1 GEMM to the full fused StyledConv and prints where (which channel group / pixel rows) the
result departs from the CPU oracle.  Writes gpurun_out/diag.txt.  Test infrastructure."""
import os
import sys
import traceback

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
torch.set_grad_enabled(False)
from oracle import stylegan2_oracle as O   # noqa: E402
import hairfastgan_b200.model as M         # noqa: E402

OUT = os.path.join(ROOT, "gpurun_out")
os.makedirs(OUT, exist_ok=True)
log = open(os.path.join(OUT, "diag.txt"), "w")


def P(*a):
    s = " ".join(str(x) for x in a)
    print(s)
    log.write(s + "\n")
    log.flush()


def case(name, cin, cout, r, k, up, batch, styled):
    try:
        torch.manual_seed(1)
        if styled:
            m = M.StyledConv(cin, cout, k, 512, upsample=up)
            m.noise.weight.data.fill_(0.5); m.activate.bias.data.normal_(0, 0.3)
            conv = m.conv
        else:
            m = conv = M.ModulatedConv2d(cin, cout, k, 512, upsample=up)
        x = torch.randn(batch, cin, r, r); st = torch.randn(batch, 512)
        ro = 2 * r if up else r
        nz = torch.randn(batch, 1, ro, ro)
        if styled:
            ref = O.styled_conv_ref(x, st, dict(m.state_dict()), "", nz, up)
        else:
            ref = O.modulated_conv2d_ref(x, st, conv.weight.data, conv.modulation.weight.data,
                                         conv.modulation.bias.data, True, up,
                                         conv.blur.kernel if up else None)
        m = m.cuda()
        y = m(x.cuda(), st.cuda(), noise=nz.cuda()) if styled else m(x.cuda(), st.cuda())
        torch.cuda.synchronize()
        y = y.cpu()
        rms = float(ref.pow(2).mean().sqrt())
        err = (y - ref).abs()
        P(f"[{name}] cin={cin} cout={cout} r={r} k={k} up={int(up)} B={batch} styled={int(styled)}: "
          f"max_err/rms={float(err.max()) / rms:.4g}  mean_err/rms={float(err.mean()) / rms:.4g}  "
          f"y_rms={float(y.pow(2).mean().sqrt()):.4g} ref_rms={rms:.4g} nan={int(torch.isnan(y).sum())}")
        if float(err.max()) / rms > 0.05:
            # localise: by 32-channel group, by output row band, by batch
            by_c = err.amax(dim=(0, 2, 3)).view(-1, 32).amax(1) / rms
            P("   by 32-ch group:", [round(float(v), 3) for v in by_c])
            by_y = err.amax(dim=(0, 1, 3)) / rms
            P("   by out row    :", [round(float(v), 2) for v in by_y[:32]])
            by_x = err.amax(dim=(0, 1, 2)) / rms
            P("   by out col    :", [round(float(v), 2) for v in by_x[:32]])
            P("   by batch      :", [round(float(v), 3) for v in err.amax(dim=(1, 2, 3)) / rms])
            # is it a scaled / permuted version?
            c = float((y * ref).sum() / (ref.pow(2).sum() + 1e-9))
            P(f"   <y,ref>/<ref,ref> = {c:.4f}")
    except Exception:
        P(f"[{name}] EXCEPTION\n" + traceback.format_exc())


P("device:", torch.cuda.get_device_name(0), "dtype env:", os.environ.get("HAIRFAST_DTYPE", "bf16"))
case("gemm1x1_64", 64, 64, 16, 1, False, 1, False)        # pure GEMM, one K chunk, one tile
case("gemm1x1_128", 128, 64, 16, 1, False, 1, False)      # two K chunks
case("gemm1x1_32", 32, 32, 16, 1, False, 1, False)        # SWIZZLE_64B path
case("conv3_64", 64, 64, 16, 3, False, 1, False)          # taps + zero padding via TMA OOB
case("conv3_64_r32", 64, 64, 32, 3, False, 2, False)      # several M tiles + batch
case("conv3_256n", 64, 256, 16, 3, False, 1, False)       # wide N
case("conv3_512", 512, 512, 8, 3, False, 2, False)        # TB=2 tile, many K blocks (pipeline wrap)
case("conv3_r4", 512, 512, 4, 3, False, 3, False)         # TB=8 tile, ragged batch
case("styled_64", 64, 64, 16, 3, False, 2, True)          # epilogue: noise/bias/lrelu
case("up_64_32", 64, 32, 8, 3, True, 2, False)            # polyphase
case("up_styled_128_64", 128, 64, 32, 3, True, 1, True)
case("conv3_32_r64", 32, 32, 64, 3, False, 1, True)       # SW64 + taps
# halo-kernel modes: resident weights + rounds (G>1), SW64 rounds, streamed weights with G=2, ragged last round
case("res_g4", 64, 64, 256, 3, False, 2, True)
case("res_up_g2", 64, 32, 256, 3, True, 1, True)
case("res_g8_sw64", 32, 32, 512, 3, False, 1, True)
case("stream_g2", 128, 128, 256, 3, False, 1, True)
case("stream_up_256", 128, 64, 128, 3, True, 3, True)
# CTA-pair kernel (cta_group::2): N tile 256, streamed weights
case("pair_512", 512, 512, 64, 3, False, 4, True)
case("pair_up_256_128", 256, 128, 64, 3, True, 3, True)
case("pair_256_b1", 256, 256, 128, 3, False, 1, False)
P("done")

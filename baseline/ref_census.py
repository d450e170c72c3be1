"""The hot-path census of one `swap()` (SURVEY Appendix B) on the STOCK reference modules -- the comparator arms of
bench.py.  Same call list as bench.py's own step, but through the unmodified classes of the built reference:
`models.stylegan2.model.Generator` (F.conv2d(groups=B) / conv_transpose2d through cuDNN + the two JIT kernels,
models/stylegan2/model.py:238-279), `Encoder4Editing`, `fs_encoder_v2`, `FeatureEncoderMult`, `FeatureiResnet`, `BiSeNet`.

    python baseline/ref_census.py --device cuda --triples T --steps K --warmup W     # reference_gpu leg (fp32/TF32)
    python baseline/ref_census.py --device cpu  --steps K --warmup W [--threads N]   # `bench.py --impl reference`

* cuda: the T triples' calls batched exactly like bench.py batches its own (3T / T / 2T per call), CUDA events, L2 flush
  between steps.
* cpu: every DISTINCT call of the census once at B=1 (full, 0->3, 3->3, 4->8, 5->8 generator ranges, e4e, FSE,
  FeatureEncoderMult, FeatureiResnet, BiSeNet 512^2 and 1024^2) and the per-triple time = sum(count x time): the whole
  census, not a FLOP-scaled part of it (CPU time is linear in the batch).  All host threads, count stated.
One JSON line on stdout.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time
import types

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from baseline import refenv, synth_checkpoints  # noqa: E402

# (name, count per triple) of the distinct calls; batch factors for the batched GPU form are in gpu_calls()
CENSUS = [("gen_full", 5), ("gen_0_3", 5), ("gen_3_3", 3), ("gen_4_8", 1), ("gen_5_8", 1), ("e4e", 5), ("fse", 3),
          ("pp_enc", 2), ("pp_res", 1), ("seg_512", 3), ("seg_1024", 2)]


def build(device, work):
    import torch
    torch.set_grad_enabled(False)
    os.environ.setdefault("TORCH_HOME", os.path.join(work, "torch_home"))
    from models.stylegan2.model import Generator
    gen = Generator(1024, 512, 8)
    gen.load_state_dict(synth_checkpoints.generator_state(0), strict=True)

    def tamed(mod, seed):
        mod.load_state_dict(synth_checkpoints._tame({k: v.clone() for k, v in mod.state_dict().items()}, seed))
        return mod
    from models.Net import iresnet50, FeatureEncoderMult
    arc = os.path.join(work, "arcface_synth.pth")
    torch.manual_seed(2)
    torch.save(synth_checkpoints._tame(synth_checkpoints._cpu_sd(iresnet50()), 2), arc)
    from models.encoder4editing.models.encoders.psp_encoders import Encoder4Editing
    torch.manual_seed(4)
    e4e = tamed(Encoder4Editing(50, "ir_se", types.SimpleNamespace(stylegan_size=1024)), 4)
    fse_dir = os.path.join(refenv.ref_root(), "models", "FeatureStyleEncoder")
    if fse_dir not in sys.path:
        sys.path.insert(0, fse_dir)
    from nets.feature_style_encoder import fs_encoder_v2
    torch.manual_seed(5)
    fse = tamed(fs_encoder_v2(n_styles=18, opts=types.SimpleNamespace(arcface_model_path=arc), stride=(2, 2)), 5)
    from models.Encoders import FeatureiResnet
    torch.manual_seed(12)
    pp_enc = tamed(FeatureEncoderMult(fs_layers=[9], opts=types.SimpleNamespace(arcface_model_path=arc)), 12)
    pp_res = tamed(FeatureiResnet([[1024, 2], [768, 2], [512, 2]]), 13)
    import torchvision
    hub = os.path.join(os.environ["TORCH_HOME"], "hub", "checkpoints")
    os.makedirs(hub, exist_ok=True)
    if not os.path.exists(os.path.join(hub, "resnet18-5c106cde.pth")):
        torch.manual_seed(13)
        torch.save(torchvision.models.resnet18().state_dict(), os.path.join(hub, "resnet18-5c106cde.pth"))
    from models.CtrlHair.external_code.face_parsing.model import BiSeNet
    torch.manual_seed(6)
    seg = BiSeNet(n_classes=19)
    nets = {"gen": gen, "e4e": e4e, "fse": fse, "pp_enc": pp_enc, "pp_res": pp_res, "seg": seg}
    return {k: v.to(device).eval() for k, v in nets.items()}


def make_calls(nets, device, T, batched):
    """name -> (callable, per-call batch multiplier).  batched=True: one call per census row at its batched size."""
    import torch
    g = torch.Generator().manual_seed(100)
    gen = nets["gen"]

    def lat(b):
        return torch.randn(b, 18, 512, generator=g).to(device)

    def img(b, r):
        return (torch.rand(b, 3, r, r, generator=g) * 2 - 1).to(device)
    calls = []
    if batched:
        # bench.py census(T): (0,8,3T) (3,3,3T,16) (0,3,3T) (0,8,T) (0,3,2T) (0,8,T) (4,8,T,32) (5,8,T,64)
        for (s, e, b, r) in [(0, 8, 3 * T, None), (3, 3, 3 * T, 16), (0, 3, 3 * T, None), (0, 8, T, None),
                             (0, 3, 2 * T, None), (0, 8, T, None), (4, 8, T, 32), (5, 8, T, 64)]:
            la = lat(b)
            li = None if r is None else torch.randn(b, 512, r, r, generator=g).to(device)
            calls.append((f"gen_{s}_{e}_B{b}", lambda la=la, li=li, s=s, e=e: gen(
                [la], input_is_latent=True, start_layer=s, end_layer=e, layer_in=li)))
        xs = {n: img(n * T, 256) for n in (3, 2, 1)}
        calls += [("e4e_3T", lambda: nets["e4e"](xs[3])), ("e4e_2T", lambda: nets["e4e"](xs[2])),
                  ("fse_3T", lambda: nets["fse"](xs[3])),
                  ("pp_enc_a", lambda: nets["pp_enc"](xs[1])), ("pp_enc_b", lambda: nets["pp_enc"](xs[1]))]
        xr = torch.randn(T, 1024, 64, 64, generator=g).to(device)
        calls.append(("pp_res", lambda: nets["pp_res"](xr)))
        s512, s1024 = img(3 * T, 512), img(T, 1024)
        calls += [("seg_512_3T", lambda: nets["seg"](s512)), ("seg_1024_a", lambda: nets["seg"](s1024)),
                  ("seg_1024_b", lambda: nets["seg"](s1024))]
        return calls
    l1 = lat(1)
    li = {r: torch.randn(1, 512, r, r, generator=g).to(device) for r in (16, 32, 64)}
    x256, x512, x1024 = img(1, 256), img(1, 512), img(1, 1024)
    xr = torch.randn(1, 1024, 64, 64, generator=g).to(device)
    return [
        ("gen_full", lambda: gen([l1], input_is_latent=True)),
        ("gen_0_3", lambda: gen([l1], input_is_latent=True, start_layer=0, end_layer=3)),
        ("gen_3_3", lambda: gen([l1], input_is_latent=True, start_layer=3, end_layer=3, layer_in=li[16])),
        ("gen_4_8", lambda: gen([l1], input_is_latent=True, start_layer=4, end_layer=8, layer_in=li[32])),
        ("gen_5_8", lambda: gen([l1], input_is_latent=True, start_layer=5, end_layer=8, layer_in=li[64])),
        ("e4e", lambda: nets["e4e"](x256)), ("fse", lambda: nets["fse"](x256)),
        ("pp_enc", lambda: nets["pp_enc"](x256)), ("pp_res", lambda: nets["pp_res"](xr)),
        ("seg_512", lambda: nets["seg"](x512)), ("seg_1024", lambda: nets["seg"](x1024)),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", choices=["cpu", "cuda"], required=True)
    ap.add_argument("--triples", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--work", default=None)
    a = ap.parse_args()
    real_stdout = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)                                   # the reference prints while it loads; keep stdout for the JSON line
    work = a.work or tempfile.mkdtemp(prefix="hf_census_")
    os.makedirs(work, exist_ok=True)
    refenv.activate(overlay=False, chdir=False)
    import torch
    threads = a.threads or os.cpu_count()            # bench.py passes the physical core count
    torch.set_num_threads(threads)                  # torchrun exports OMP_NUM_THREADS=1: do not inherit it silently
    dev = torch.device(a.device)
    nets = build(dev, work)
    counts = dict(CENSUS)
    out = {"device": a.device, "steps": a.steps, "warmup": a.warmup,
           "generator_class": type(nets["gen"]).__module__, "torch_threads": torch.get_num_threads()}
    if a.device == "cpu":
        calls = make_calls(nets, dev, 1, batched=False)
        per_step = []
        last = {}
        for it in range(a.warmup + a.steps):
            tot = 0.0
            for name, fn in calls:
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                last[name] = dt
                tot += counts[name] * dt
            if it >= a.warmup:
                per_step.append(tot)
        s = sum(per_step) / len(per_step)
        out.update({"triples_per_s": 1.0 / s, "s_per_triple": s, "per_call_s": {k: round(v, 4) for k, v in last.items()},
                    "cores": threads,
                    "sample": "every distinct call of the SURVEY App. B census once at B=1 on the stock reference "
                              "modules (CPU branches), per-triple time = sum(count x time): full census, "
                              f"{threads} threads"})
    else:
        T = a.triples
        calls = make_calls(nets, dev, T, batched=True)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        tf32 = bool(torch.backends.cudnn.allow_tf32)
        ms_steps, per = [], {}
        for it in range(a.warmup + a.steps):
            flush.fill_(1)
            evs = []
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record()
            prev = e0
            for name, fn in calls:
                fn()
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                evs.append((name, prev, e))
                prev = e
            torch.cuda.synchronize()
            if it >= a.warmup:
                ms_steps.append(e0.elapsed_time(prev))
                per = {n: round(s_.elapsed_time(e_), 3) for n, s_, e_ in evs}
        ms = sum(ms_steps) / len(ms_steps)
        out.update({"triples": T, "ms_per_step": ms, "triples_per_s": T / (ms * 1e-3), "per_call_ms": per,
                    "cudnn_allow_tf32": tf32, "cudnn_benchmark": bool(torch.backends.cudnn.benchmark),
                    "device_name": torch.cuda.get_device_name(0),
                    "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                    "arith": "fp32 storage, cuDNN TF32 convolutions (torch default), fp32 F.linear"})
    real_stdout.write(json.dumps(out) + "\n")
    real_stdout.flush()


if __name__ == "__main__":
    main()

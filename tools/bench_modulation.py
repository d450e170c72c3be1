"""Time HairFast's latent modulation stacks: the stock reference's RotateModel / ClipBlendingModel / PostProcessModel
forwards against hairfastgan_b200.modulation, same GPU, same modules (the reference classes holding
``oracle.modulation_oracle.synth_params``; needs the reference built under oracle/_ref, baseline/refenv.py).  CLIP and
PostProcess's encoders are replaced by identities on both sides, so only the stacks are timed.

    python tools/bench_modulation.py [--reps 20] [--warmup 3] [--swap N] [--out result.json]

* B = 1 (as swap() calls them) and B = 32; CUDA events around each call, a 256 MiB L2 flush between calls, the median;
* kernel launches per call: stock from torch.profiler, ours from hf_total_launch_count, and our memsets from
  torch.profiler;
* the 16-bit weight bytes one call streams over our call time, against the 3.35 TB/s of HBM3;
* our per-kernel times from one torch.profiler run (the chain kernel among them);
* --swap N: full_swap_ms of baseline/run_swap.py, overlay_all and overlay_modulation alternated N times each;
* the card name, power limit and SM clock are read in the same run (nvidia-smi queries only).
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
HBM_TBS = 3.35


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else {}


def weight_bytes(layers: int, stacks: int) -> int:
    from hairfastgan_b200.modulation import CONFIGS, DIM
    inp, middle = CONFIGS[layers]
    return 2 * stacks * (10 * middle * inp + 10 * DIM * middle + 5 * DIM * DIM)


def models(dev):
    import torch
    from torch import nn
    from baseline import refenv
    refenv.activate(overlay=False, chdir=False)
    import models.Encoders as E
    from oracle import modulation_oracle as O
    rot = E.RotateModel()
    rot.modulation_module_list.load_state_dict(O.stack_state_dict(O.synth_params(31, 6)))
    bl = E.ClipBlendingModel()
    bl.modulation_module_list.load_state_dict(O.stack_state_dict(O.synth_params(32, 12)))
    bl.get_image_embed = lambda image: image
    pp = E.PostProcessModel.__new__(E.PostProcessModel)
    nn.Module.__init__(pp)
    pp.to_latent_1 = nn.ModuleList([E.ModulationModule(18, i == 4) for i in range(5)])
    pp.to_latent_2 = nn.ModuleList([E.ModulationModule(18, i == 4) for i in range(5)])
    pp.to_latent_1.load_state_dict(O.stack_state_dict(O.synth_params(33, 18)))
    pp.to_latent_2.load_state_dict(O.stack_state_dict(O.synth_params(34, 18)))
    pp.pixelnorm = E.PixelNorm()
    pp.to_feature = nn.Identity()
    pp = pp.to(dev)
    pp.latent_avg = 0.5 * torch.randn(18, 512, device=dev)
    pp.encoder_face = lambda x: (x, [x[:, :1]])
    return E, rot.to(dev).eval(), bl.to(dev).eval(), pp.eval()


def calls(E, rot, bl, pp, batch, dev):
    """name -> (layers, stacks, stock call, our call)"""
    import torch
    from hairfastgan_b200 import modulation as M
    g = torch.Generator(device=dev).manual_seed(batch)
    w1, w2 = (torch.randn(batch, 18, 512, device=dev, generator=g) for _ in range(2))
    lf, lc = (torch.randn(batch, 12, 512, device=dev, generator=g) for _ in range(2))
    ef, ec = (torch.randn(batch, 512, device=dev, generator=g) for _ in range(2))
    sf, sh = (torch.randn(batch, 18, 512, device=dev, generator=g) for _ in range(2))
    return {"rotate": (6, 1, lambda: E.RotateModel.forward(rot, w2[:, :6], w1[:, :6]),
                       lambda: M.rotate_forward(rot, w2[:, :6], w1[:, :6])),
            "blending": (12, 1, lambda: E.ClipBlendingModel.forward(bl, lf, lc, ef, ec),
                         lambda: M.blending_forward(bl, lf, lc, ef, ec)),
            "postprocess": (18, 2, lambda: E.PostProcessModel.forward(pp, sf, sh)[0],
                            lambda: M.postprocess_forward(pp, sf, sh)[0])}


def time_ms(fn, reps, warmup, flush):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def profile(fn):
    """(kernel count, memset count, {kernel name: device ms}) of one call."""
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    device = [e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    memsets = sum("Memset" in e.name for e in device)
    kernels = [e for e in device if "Memset" not in e.name and "Memcpy" not in e.name]
    per = {}
    for e in kernels:
        m = re.search(r"(\w+)\s*[<(]", e.name.replace("(anonymous namespace)", ""))
        name = m.group(1) if m else e.name
        per[name] = per.get(name, 0.0) + e.device_time_total / 1e3
    return len(kernels), memsets, per


def swap_runs(n: int) -> dict:
    work = os.environ.get("HAIRFAST_WORK", "/tmp/hairfast_work")
    res = {"overlay_all": [], "overlay_modulation": []}
    with tempfile.TemporaryDirectory() as tmp:
        for i in range(n):
            for mode in (("overlay_all", "overlay_modulation") if i % 2 == 0 else
                         ("overlay_modulation", "overlay_all")):
                out = os.path.join(tmp, f"{mode}.pt")
                subprocess.run([sys.executable, os.path.join(ROOT, "baseline", "run_swap.py"), "--mode", mode, "--work",
                                work, "--out", out, "--reps", "3", "--warmup", "1"], check=True, capture_output=True)
                import torch
                s = torch.load(out, weights_only=False)["summary"]
                res[mode].append(statistics.median(t["gpu_ms"] for t in s["timings"]))
    return {m: {"runs_ms": v, "median_ms": statistics.median(v), "spread_ms": max(v) - min(v)} for m, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--swap", type=int, default=0, help="alternate the two swap arms this many times each")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_modulation.py needs a GPU"
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    from hairfastgan_b200 import _lib, nn16
    E, rot, bl, pp = models(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    res = {"card": card(), "dtype": "fp16" if nn16.default_dtype() == _lib.HF_F16 else "bf16", "calls": {}}
    for batch in (1, 32):
        for name, (layers, stacks, stock, ours) in calls(E, rot, bl, pp, batch, dev).items():
            ours()
            stock_ms, ours_ms = time_ms(stock, a.reps, a.warmup, flush), time_ms(ours, a.reps, a.warmup, flush)
            n_stock, _, _ = profile(stock)
            n0 = _lib.lib().hf_total_launch_count()
            ours()
            n_ours = _lib.lib().hf_total_launch_count() - n0
            _, memsets, kernels = profile(ours)
            wb = weight_bytes(layers, stacks)
            res["calls"][f"{name}_b{batch}"] = {
                "stock_ms": stock_ms, "ours_ms": ours_ms, "speedup": stock_ms / ours_ms,
                "stock_kernels": n_stock, "ours_launches": n_ours, "ours_memsets": memsets, "weight_MB": wb / 1e6,
                "weight_GBps": wb / ours_ms / 1e6, "weight_share_of_hbm": wb / ours_ms / 1e9 / HBM_TBS,
                "ours_kernel_ms": kernels}
            print(name, batch, json.dumps(res["calls"][f"{name}_b{batch}"]), flush=True)
    if a.swap:
        res["swap"] = swap_runs(a.swap)
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

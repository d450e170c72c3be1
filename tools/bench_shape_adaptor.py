"""Time CtrlHair's shape adaptor: the stock reference's get_hair_face_code / get_new_shape against
hairfastgan_b200.shape_adaptor, same GPU, one reference ``Generator(cfg)`` of config 054 holding
``oracle.shape_adaptor_oracle.synth_params(7)`` (needs the reference built under oracle/_ref, baseline/refenv.py).

    python tools/bench_shape_adaptor.py [--reps 20] [--warmup 3] [--swap] [--out result.json]

* CUDA events around each call, a 256 MiB L2 flush between calls, warm-up calls first, the median reported;
* algorithmic GFLOP per call (the layer-0 lookup counted at its convolution FLOPs) and the TFLOP/s they give;
* the split-K GEMM's kernel time from one torch.profiler run, and the weight bytes its layers stream over it (GB/s
  against the 3.35 TB/s of HBM3: these layers are bound by their weight bytes);
* our kernel launches per call;
* --swap: full_swap_ms of baseline/run_swap.py for the overlay_sean_full and overlay_all arms;
* the card name, power limit and SM clock are read in the same run (nvidia-smi queries only).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)


def encoder_flops(n_mask: int, out_dim: int) -> float:
    from hairfastgan_b200.shape_adaptor import ENC_CH, POS_CHANNELS
    f, cin, r = 0.0, n_mask + POS_CHANNELS, 128
    for c in ENC_CH:
        f += 2.0 * r * r * c * cin * 16
        cin, r = c, r // 2
    return f + 2.0 * 4 * ENC_CH[-1] * out_dim


def decoder_flops(in_dim: int, n_out: int) -> float:
    from hairfastgan_b200.shape_adaptor import DEC_CH
    f, cin, r = 2.0 * in_dim * 4 * DEC_CH[0], DEC_CH[0], 4
    for c in DEC_CH:
        f += 2.0 * r * r * c * cin * 9
        cin, r = c, r * 2
    return f + 2.0 * 256 * 256 * n_out * cin * 9


def gemm_weight_bytes() -> int:
    """16-bit weight bytes of the split-K GEMM layers of one get_hair_face_code + get_new_shape."""
    from hairfastgan_b200 import shape_adaptor as S
    n = 0
    for net, d in S.NETWORK_SHAPES.items():
        for k, shape in d.items():
            if not k.endswith("weight") or k.startswith("std_out_layer") or k == "layers.0.conv.weight":
                continue
            if "decoder" in net and k.startswith("layers.") and int(k.split(".")[1]) // 2 >= S.DEC_GEMM_LAYERS:
                continue
            if k.startswith("out_layer.conv"):
                continue
            size = 1
            for s in shape:
                size *= s
            n += 2 * size
    return n


def card_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"nvidia_smi": q.stdout.strip()}


def timed(fn, reps: int, warmup: int, flush) -> float:
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--swap", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from baseline import refenv
    refenv.activate(overlay=False, chdir=False)
    from models.CtrlHair.shape_branch import solver
    from hairfastgan_b200 import _lib, shape_adaptor as S
    from oracle import shape_adaptor_oracle as O
    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    gen = O.reference_generator()
    gen.load_state_dict(O.synth_params(7))
    gen = gen.to(dev).eval()
    mask = O.label_cases()["face"].to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    res = {"card": card_info()}
    stock_codes = solver.get_hair_face_code(gen, mask.clone())
    ours_codes = S.get_hair_face_code(gen, mask.clone())
    res["codes_max_abs_diff"] = max(float((x - y).abs().max()) for x, y in zip(stock_codes, ours_codes))
    stock_lab = solver.get_new_shape(gen, *stock_codes)
    ours_lab = S.get_new_shape(gen, *stock_codes)
    res["label_agreement"] = float((stock_lab == ours_lab).float().mean())
    f_code = encoder_flops(1, 16) + encoder_flops(18, 1024)
    f_shape = decoder_flops(1040, 1) + decoder_flops(1024, 18)
    for name, stock, ours, flops in [
            ("get_hair_face_code", lambda: solver.get_hair_face_code(gen, mask.clone()),
             lambda: S.get_hair_face_code(gen, mask.clone()), f_code),
            ("get_new_shape", lambda: solver.get_new_shape(gen, *stock_codes),
             lambda: S.get_new_shape(gen, *stock_codes), f_shape)]:
        ts, to = timed(stock, a.reps, a.warmup, flush), timed(ours, a.reps, a.warmup, flush)
        n0 = _lib.lib().hf_total_launch_count()
        ours()
        launches = _lib.lib().hf_total_launch_count() - n0
        res[name] = {"stock_ms": ts, "ours_ms": to, "speedup": ts / to, "gflop": flops / 1e9,
                     "stock_tflops": flops / ts / 1e9, "ours_tflops": flops / to / 1e9, "our_kernel_launches": launches}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        S.get_new_shape(gen, *S.get_hair_face_code(gen, mask.clone()))
        torch.cuda.synchronize()
    gemm_us = sum(e.device_time_total for e in prof.key_averages() if "shape_gemm_kernel" in e.key)
    wb = gemm_weight_bytes()
    res["splitk_gemm"] = {"kernel_us": gemm_us, "weight_bytes": wb, "weight_GBps": wb / gemm_us / 1e3,
                          "share_of_3.35TBps": wb / gemm_us / 1e3 / 3350.0}
    if a.swap:
        work = os.environ.get("HAIRFAST_WORK", "/tmp/hairfast_work")
        for mode in ("overlay_sean_full", "overlay_all"):
            out = os.path.join(tempfile.mkdtemp(), f"{mode}.pt")
            subprocess.run([sys.executable, os.path.join(ROOT, "baseline", "run_swap.py"), "--mode", mode, "--work",
                            work, "--out", out, "--reps", "4", "--warmup", "1"], check=True, capture_output=True)
            t = torch.load(out, weights_only=False)["summary"]["timings"]
            res[f"swap_{mode}_ms"] = statistics.median(x["gpu_ms"] for x in t)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

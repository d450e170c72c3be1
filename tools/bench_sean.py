"""Time SEAN's decode_sean (and, with --encode, encode_sean): the stock reference against hairfastgan_b200.sean, same
GPU, same synthetic weights; decode B = 1, encode B = 2 (what Alignment.align_images passes, models/Alignment.py:128).

    python tools/bench_sean.py [--reps 20] [--warmup 3] [--encode] [--swap] [--out result.json]

* both decodes run on ONE reference ``Pix2PixModel(SEAN_OPT)`` built by the reference's own code from a checkpoint
  holding ``oracle.sean_oracle.synth_sean_params(5)`` (needs the reference built under oracle/_ref, baseline/refenv.py);
* CUDA events around each call, a 256 MiB L2 flush between calls, warm-up calls first, the median reported;
* our per-stage split from one torch.profiler run: style tables, label maps + one-hot lookups, convolutions, ACE apply,
  other (upsample, conv_img);
* achieved TFLOP/s against the algorithmic FLOPs of the decode, the lookup-replaced convolutions counted at their
  convolution FLOPs (the rule of bench.py's roofline);
* --encode: the same timing of encode_sean, its algorithmic FLOPs (the ConvTranspose2d counted at its algorithmic
  FLOPs, a quarter of what its four-parity form runs) and the max difference of the codes;
* --swap: full_swap_ms / out_of_scope_ms of baseline/run_swap.py for the overlay, overlay_sean and overlay_sean_full
  arms;
* the card name, power limit and SM clock are read in the same run (nvidia-smi queries only).
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)


def decode_flops() -> float:
    """Algorithmic FLOPs of one decode (2 per MAC)."""
    from oracle import sean_oracle as SO
    f = 2 * 19 * 1024 * 9 * 8 * 8                                   # fc
    for _, fin, fout, r, rgb in SO.BLOCKS:
        hw = r * r
        fmid = min(fin, fout)
        for _, c in SO.block_aces(fin, fout):
            f += 2 * 19 * 128 * 9 * hw + 2 * 128 * 2 * c * 9 * hw   # mlp_shared, mlp_gamma || mlp_beta
            if rgb:
                f += 2 * 512 * 2 * c * 9 * hw + 19 * 2 * 512 * 512  # conv_gamma || conv_beta, fc_mu
        f += 2 * fin * fmid * 9 * hw + 2 * fmid * fout * 9 * hw     # conv_0, conv_1
        if fin != fout:
            f += 2 * fin * fout * hw                                # conv_s
    return f + 2 * 64 * 3 * 9 * 256 * 256                          # conv_img


def encode_flops(batch: int = 2) -> float:
    """Algorithmic FLOPs of one encode_sean call (2 per MAC): the five Zencoder convolutions (architecture.py:154-175)."""
    f = 2 * 3 * 32 * 9 * 256 ** 2 + 2 * 32 * 64 * 9 * 128 ** 2 + 2 * 64 * 128 * 9 * 64 ** 2
    f += 2 * 128 * 256 * 9 * 64 ** 2                               # ConvTranspose2d: 9 taps per input pixel
    f += 2 * 256 * 512 * 9 * 128 ** 2
    return batch * f


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {}


def time_calls(fn, reps, warmup, flush):
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
    return statistics.median(ms), ms


def stage_split(fn):
    """Kernel time per stage (ms) of one call, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    stages = {"tables": 0.0, "lut": 0.0, "convs": 0.0, "ace_apply": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        if ev.device_type != torch.autograd.DeviceType.CUDA and not getattr(ev, "self_device_time_total", 0):
            continue
        t = getattr(ev, "self_device_time_total", 0) / 1e3
        n = ev.key
        if "sean_fc_mu" in n or "sean_table" in n:
            stages["tables"] += t
        elif "sean_onehot" in n or "sean_labels" in n:
            stages["lut"] += t
        elif "conv_wgmma" in n:
            stages["convs"] += t
        elif "sean_ace" in n:
            stages["ace_apply"] += t
        elif t > 0:
            stages["other"] += t
    return {k: round(v, 4) for k, v in stages.items()}


def swap_arms(work):
    res = {}
    env = {k: v for k, v in os.environ.items() if k not in ("HAIRFAST_DTYPE", "HAIRFAST_ENC_DTYPE")}
    for mode in ("overlay", "overlay_sean", "overlay_sean_full"):
        out = os.path.join(tempfile.mkdtemp(), mode + ".pt")
        cmd = [sys.executable, os.path.join(ROOT, "baseline", "run_swap.py"), "--mode", mode, "--work", work,
               "--out", out, "--reps", "3", "--warmup", "1"]
        p = subprocess.run(cmd, capture_output=True, text=True, env=env)
        if p.returncode:
            raise RuntimeError(f"run_swap {mode} failed:\n{p.stderr[-3000:]}")
        s = json.loads(p.stdout.strip().splitlines()[-1])
        t = s["timings"]
        res[mode] = {"full_swap_ms": statistics.median(x["gpu_ms"] for x in t),
                     "out_of_scope_ms": statistics.median(x["out_of_scope_ms"] for x in t)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--encode", action="store_true", help="also time encode_sean")
    ap.add_argument("--swap", action="store_true")
    ap.add_argument("--work", default="/tmp/hairfast_work")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    out_path = os.path.abspath(a.out) if a.out else None     # refenv.activate changes the working directory

    from baseline import refenv
    if not refenv.available():
        raise SystemExit("bench_sean: the reference is not built under oracle/_ref (oracle/build_ref.py)")
    refenv.activate(overlay=False)                # cwd = reference root: load_average_feature reads a relative path
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sean: needs a CUDA device")
    torch.set_grad_enabled(False)
    import models.sean_codes.models.pix2pix_model as P
    from hairfastgan_b200 import sean as S
    from oracle import sean_oracle as SO

    tmp = tempfile.mkdtemp()
    opt = copy.copy(P.SEAN_OPT)
    opt.checkpoints_dir = tmp
    os.makedirs(os.path.join(tmp, opt.name))
    torch.save(SO.synth_sean_params(5), os.path.join(tmp, opt.name, "latest_net_G.pth"))
    model = P.Pix2PixModel(opt)
    model.eval()
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(3)
    labels = torch.randint(0, 19, (1, 1, 16, 16), generator=g).repeat_interleave(16, 2).repeat_interleave(16, 3)
    target_mask = labels.float().to(dev)
    code = (torch.randn(1, 19, 512, generator=g) * 0.5).to(dev)
    flush = torch.empty(256 * 2 ** 20, dtype=torch.uint8, device=dev)

    with torch.inference_mode():
        torch.manual_seed(0)
        ref_img = P.decode_sean(model, code, target_mask)
        torch.manual_seed(0)
        our_img = S.decode_sean(model, code, target_mask)
        diff = float((our_img - ref_img).abs().max())
        stock_ms, stock_all = time_calls(lambda: P.decode_sean(model, code, target_mask), a.reps, a.warmup, flush)
        ours_ms, ours_all = time_calls(lambda: S.decode_sean(model, code, target_mask), a.reps, a.warmup, flush)
        stages = stage_split(lambda: S.decode_sean(model, code, target_mask))
    flops = decode_flops()
    res = {"gpu": gpu_info(), "dtype": "fp16" if S.nn16.default_dtype() == 1 else "bf16",
           "stock_decode_ms": round(stock_ms, 3), "ours_decode_ms": round(ours_ms, 3),
           "speedup": round(stock_ms / ours_ms, 2), "stock_ms_all": [round(x, 3) for x in stock_all],
           "ours_ms_all": [round(x, 3) for x in ours_all], "ours_stage_kernel_ms": stages,
           "algorithmic_gflop": round(flops / 1e9, 1), "ours_tflops": round(flops / ours_ms / 1e9, 1),
           "stock_tflops": round(flops / stock_ms / 1e9, 1), "max_abs_vs_stock": diff}
    if a.encode:
        images = (torch.rand(2, 3, 256, 256, generator=g) * 2 - 1).to(dev)
        enc_labels = torch.randint(0, 19, (2, 1, 16, 16), generator=g).repeat_interleave(16, 2).repeat_interleave(16, 3)
        enc_labels = enc_labels.float().to(dev)
        with torch.inference_mode():
            ref_codes = P.encode_sean(model, images, enc_labels)
            our_codes = S.encode_sean(model, images, enc_labels)
            stock_e, stock_e_all = time_calls(lambda: P.encode_sean(model, images, enc_labels), a.reps, a.warmup, flush)
            ours_e, ours_e_all = time_calls(lambda: S.encode_sean(model, images, enc_labels), a.reps, a.warmup, flush)
        ef = encode_flops(2)
        res["encode"] = {"batch": 2, "stock_encode_ms": round(stock_e, 3), "ours_encode_ms": round(ours_e, 3),
                         "speedup": round(stock_e / ours_e, 2), "stock_ms_all": [round(x, 3) for x in stock_e_all],
                         "ours_ms_all": [round(x, 3) for x in ours_e_all], "algorithmic_gflop": round(ef / 1e9, 2),
                         "ours_tflops": round(ef / ours_e / 1e9, 1), "stock_tflops": round(ef / stock_e / 1e9, 1),
                         "codes_max_abs_vs_stock": float((our_codes - ref_codes).abs().max()),
                         "codes_max_abs_ref": float(ref_codes.abs().max())}
    if a.swap:
        res["swap"] = swap_arms(os.path.abspath(a.work))
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

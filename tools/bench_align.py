"""Time the FFHQ face alignment after the landmarks: the stock reference's CPU ``align_face`` (PIL / numpy / scipy)
against hairfastgan_b200.face_align on the GPU, on seeded synthetic images at user sizes with fixed landmarks (the
reference's dlib is replaced by oracle/align_oracle.FakeDlib, so only the warp is timed).

    python tools/bench_align.py [--reps 30] [--cpu-reps 5] [--warmup 3] [--swap] [--out result.json]

* cases: 1024^2 with a large face (the padding branch), 2000x1500, and 4800^2 with shrink = 2;
* stock: the unmodified reference align_face (built under oracle/_ref, baseline/refenv.py) on a PIL image,
  return_tensors=False, median of --cpu-reps calls after one warm-up, with the host's thread counts stated;
* ours: align_from_landmarks from the uint8 upload to the uint8 download (host clock around work that ends in a
  device synchronise), median of --reps calls after --warmup; the device time alone from CUDA events; the output is
  checked equal to the stock one;
* the kernel breakdown of one call per case from a separate torch.profiler run;
* --swap: baseline/run_swap.py's aligned swap, reference_align against overlay_align, one process each;
* the card name and power limit are read in the same run (nvidia-smi queries only).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

# name -> (height, width, eye midpoint, inter-ocular px, roll)
CASES = {"1024_pad": (1024, 1024, (512, 440), 420, 0.0),
         "2000x1500": (1500, 2000, (1010, 700), 300, 6.0),
         "4800_shrink": (4800, 4800, (2400, 2250), 1100, 0.0)}


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--cpu-reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--swap", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import numpy as np
    import PIL.Image
    import torch
    from oracle import align_oracle as O
    from hairfastgan_b200 import face_align as FA
    assert torch.cuda.is_available(), "bench_align.py needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "torch_threads": torch.get_num_threads(), "cpu_count": os.cpu_count(),
           "omp_num_threads": os.environ.get("OMP_NUM_THREADS"), "cases": {}}

    stock = None
    from baseline import refenv
    if refenv.available():
        refenv.activate(overlay=False, chdir=False)
        import utils.shape_predictor as sp
        if not hasattr(PIL.Image, "ANTIALIAS"):
            PIL.Image.ANTIALIAS = PIL.Image.LANCZOS
        stock = sp

    for name, (h, w, mid, io, roll) in CASES.items():
        img = O.synth_image(h, w, seed=len(name) + h, cell=64)
        lm = O.synth_landmarks(mid, io, roll)
        g = FA.geometry(lm, (w, h))
        row = {"size": [w, h], "inter_ocular": io, "shrink": g.shrink, "crop": g.crop, "pad": g.pad}
        ref = None
        if stock is not None:
            fake = O.FakeDlib([lm])
            stock.dlib = fake
            pil = PIL.Image.fromarray(img)
            ts = []
            for i in range(1 + a.cpu_reps):
                t0 = time.perf_counter()
                ref = np.asarray(stock.align_face([pil], fake.predictor, return_tensors=False)[0])
                if i:
                    ts.append((time.perf_counter() - t0) * 1e3)
            row["stock_cpu_ms"] = statistics.median(ts)
            row["stock_cpu_ms_all"] = [round(t, 1) for t in ts]
        ts, dts = [], []
        for i in range(a.warmup + a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            src = torch.from_numpy(img).to(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = FA.align_from_landmarks(src, lm)
            e1.record()
            host = out.cpu().numpy()
            torch.cuda.synchronize()
            if i >= a.warmup:
                ts.append((time.perf_counter() - t0) * 1e3)
                dts.append(e0.elapsed_time(e1))
        row["ours_upload_to_download_ms"] = statistics.median(ts)
        row["ours_device_ms"] = statistics.median(dts)
        row["ours_ms_min_max"] = [round(min(ts), 3), round(max(ts), 3)]
        if ref is not None:
            row["equal_to_stock"] = bool(np.array_equal(host, ref))
            row["speedup"] = row["stock_cpu_ms"] / row["ours_upload_to_download_ms"]
        res["cases"][name] = row
        print(name, json.dumps(row), flush=True)

    # kernel breakdown: one call per case in a separate profiled run
    from torch.profiler import ProfilerActivity, profile
    for name, (h, w, mid, io, roll) in CASES.items():
        img = O.synth_image(h, w, seed=len(name) + h, cell=64)
        lm = O.synth_landmarks(mid, io, roll)
        src = torch.from_numpy(img).to(dev)
        FA.align_from_landmarks(src, lm)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            FA.align_from_landmarks(src, lm)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                k = ev.name.split("(")[0].replace("void ", "")
                kern[k] = kern.get(k, 0.0) + ev.device_time_total / 1e3
        res["cases"][name]["kernels_ms"] = {k: round(v, 4) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
        print(name, "kernels", json.dumps(res["cases"][name]["kernels_ms"]), flush=True)

    if a.swap:
        work = os.environ.get("HAIRFAST_WORK", "/tmp/hairfast_work")
        res["swap"] = {}
        for mode in ("reference_align", "overlay_align"):
            with tempfile.TemporaryDirectory() as d:
                out = os.path.join(d, "r.pt")
                p = subprocess.run([sys.executable, os.path.join(ROOT, "baseline", "run_swap.py"), "--mode", mode,
                                    "--work", work, "--out", out, "--reps", "3", "--warmup", "1"],
                                   capture_output=True, text=True, timeout=1800)
                if p.returncode:
                    raise RuntimeError(p.stderr[-3000:])
                s = torch.load(out, weights_only=False)["summary"]
            res["swap"][mode] = {"wall_ms": [round(t["wall_ms"], 1) for t in s["timings"]],
                                 "gpu_ms": [round(t["gpu_ms"], 1) for t in s["timings"]]}
            print(mode, json.dumps(res["swap"][mode]), flush=True)

    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Time the float64 feature path (kernel family 12) against the float32 one on bench.py's workload.

    python scripts/bench_f64.py [--clips 1000] [--steps 5] [--warmup 2] [--out DIR]

Workload: bench.py's -- CLIPS synthetic 16 kHz mono int16 10 s clips, window / step 50 / 25 ms (800 / 400 samples).  Each
step is one call of feature_extraction_batch (68 rows) or mid_feature_extraction_batch (1 s / 1 s mid-term windows), clip
statistics included, with the clips resident in HBM; the float64 and float32 calls alternate inside one process and each
is timed with CUDA events around a synchronised call.  A separate torch.profiler pass gives the time of every kernel of one
call of each path.  Prints one JSON line: the card's name and power limit, the median step times, frames/s, the kernel
times, and the largest per-row difference between the two paths' short-term features (float32 widened).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (its workload constants and clip generator)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=bench.CLIPS_PER_GPU)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_f64.py needs a CUDA device")
    from pyaudioanalysis_b200 import batch as BT

    dev = torch.device("cuda", 0)
    clips = bench.synth_device_batch(torch, args.clips, 1234, dev)
    fs, w, s = bench.FS, bench.WINDOW, bench.STEP
    calls = {
        "st_f32": lambda: BT.feature_extraction_batch(clips, fs, w, s),
        "st_f64": lambda: BT.feature_extraction_batch(clips, fs, w, s, dtype=torch.float64),
        "mid_f32": lambda: BT.mid_feature_extraction_batch(clips, fs, fs, fs, w, s),
        "mid_f64": lambda: BT.mid_feature_extraction_batch(clips, fs, fs, fs, w, s, dtype=torch.float64),
    }
    for _ in range(args.warmup):
        for f in calls.values():
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(args.steps):
        for k, f in calls.items():                  # float32 and float64 alternate
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    step_ms = {k: statistics.median(v) for k, v in times.items()}
    frames = args.clips * bench.FRAMES_PER_CLIP

    # kernel times of one call of each path
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for k in ("st_f32", "st_f64", "mid_f64"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            calls[k]()
            torch.cuda.synchronize()
        rows = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0)
            if t > 0 and "memcpy" not in e.key.lower() and "memset" not in e.key.lower():
                rows[e.key.split("(")[0][:60]] = round(t / 1000.0, 3)
        kernels[k] = rows
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "kernels_%s.txt" % k), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=20))

    a = calls["st_f64"]().double()
    b = calls["st_f32"]().double()
    per_row = (a - b).abs().amax(dim=(0, 2))
    row = int(per_row.argmax())
    scale = a.abs().amax(dim=(0, 2))
    print(json.dumps({
        "gpu": card(),
        "workload": "%d x 10 s 16 kHz int16 clips, 50 / 25 ms, 68 rows; mid-term 1 s / 1 s" % args.clips,
        "step_ms": {k: round(v, 3) for k, v in step_ms.items()},
        "frames_per_s": {k: round(frames / (v / 1000.0)) for k, v in step_ms.items()},
        "kernel_ms": kernels,
        "max_row_diff": {"row": row, "abs": float(per_row[row]), "row_max_abs": float(scale[row])},
        "max_row_rel_diff": float((per_row / scale.clamp_min(1e-300)).max()),
        "steps": args.steps,
    }))


if __name__ == "__main__":
    main()

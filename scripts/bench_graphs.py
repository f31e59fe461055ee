#!/usr/bin/env python
"""Time the feature path called eagerly against a replay of it captured in a CUDA graph.

    python scripts/bench_graphs.py [--batches 1,8,64] [--iters 200] [--warmup 20]

Workload: B synthetic 16 kHz mono int16 10 s clips per call (bench.py's generator), B = 1, 8 and 64, resident in HBM,
through clip statistics, short-term features (50 / 25 ms, 68 rows), mid-term pooling (1 s / 1 s), the long-term mean
and beat extraction: the steps of directory_feature_extraction.  The eager arm calls the batch functions; the graph arm
replays one ``torch.cuda.CUDAGraph`` captured from the same calls.  After warm-up, each arm runs ITERS calls back to back;
the host wall clock around them, ending in a synchronise, gives the time per call, and CUDA events around them the device
time.  The arms alternate twice and the outputs of the last call of each are compared bit for bit.  Prints the card's name
and power limit, then one JSON line per batch size.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402  (its workload constants and clip generator)

MID = 1.0, 1.0                      # mid-term window / step, seconds


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def step(pkg, x):
    """One call of the workload on the current stream: (short-term features, mid-term, long-term mean, beat)."""
    fs, w, s = bench.FS, bench.WINDOW, bench.STEP
    ratio, stepr = pkg.batch.mid_ratios(MID[0] * fs, MID[1] * fs, w, s)
    norm = pkg.clip_stats(x)
    st = pkg.feature_extraction_batch(x, fs, w, s, norm=norm)
    mid = pkg.mid_pool_batch(st, ratio, stepr)
    return st, mid, pkg.long_term_mean_batch(mid), pkg.beat_extraction_batch(st, s / fs)


def timed(torch, call, iters):
    """(host ms per call around a final synchronise, device ms per call from CUDA events)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a.record()
    for _ in range(iters):
        call()
    b.record()
    torch.cuda.synchronize()
    host = (time.perf_counter() - t0) * 1e3 / iters
    return host, a.elapsed_time(b) / iters


def bits(t):
    a = np.ascontiguousarray(t.cpu().numpy())
    return a.view({4: np.int32, 8: np.int64}[a.dtype.itemsize])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import pyaudioanalysis_b200 as pkg
    assert torch.cuda.is_available(), "needs a CUDA device"
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    for B in (int(v) for v in args.batches.split(",")):
        x = bench.synth_device_batch(torch, B, 0, torch.device("cuda"))
        out = {"eager": None}
        for _ in range(args.warmup):
            out["eager"] = step(pkg, x)
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step(pkg, x)
        torch.cuda.current_stream().wait_stream(side)
        with torch.cuda.graph(g):
            out["graph"] = step(pkg, x)
        for _ in range(args.warmup):
            g.replay()
        res = {"eager": [], "graph": []}
        for _ in range(2):
            res["eager"].append(timed(torch, lambda: out.__setitem__("eager", step(pkg, x)), args.iters))
            res["graph"].append(timed(torch, g.replay, args.iters))
        same = all(np.array_equal(bits(a), bits(b)) for a, b in zip(out["eager"], out["graph"]))
        host = {k: min(h for h, _ in v) for k, v in res.items()}
        dev = {k: min(d for _, d in v) for k, v in res.items()}
        print(json.dumps({"clips": B, "clip_seconds": bench.CLIP_SAMPLES / bench.FS, "iters": args.iters,
                          "eager_host_ms": round(host["eager"], 4), "graph_host_ms": round(host["graph"], 4),
                          "eager_device_ms": round(dev["eager"], 4), "graph_device_ms": round(dev["graph"], 4),
                          "host_speedup": round(host["eager"] / host["graph"], 3), "bit_identical": same,
                          "runs_ms": {k: [[round(h, 4), round(d, 4)] for h, d in v] for k, v in res.items()}}), flush=True)
        del g
    return 0


if __name__ == "__main__":
    sys.exit(main())

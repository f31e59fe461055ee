"""Wall-clock time of directory_feature_extraction on folders of 1000 generated 16 kHz mono PCM16 files, decode
included, and of the config-4 pooling (1 x 68 x 143 999 frames, ratio 39 / 40) -> one JSON line per measurement.

    python scripts/bench_folders.py --make DIR                 # (a) 2-20 s, (b) 10 s +- 0-50 samples, (c) exactly 10 s
    python scripts/bench_folders.py --time DIR [--root PKG_ROOT] [--out FEATURES.npz] [--padding 0.25]

``--root`` imports pyaudioanalysis_b200 from another tree (e.g. an older build, to alternate runs of two versions in
one session); ``--out`` saves each folder's feature matrix so two versions' outputs can be compared; ``--padding`` sets
the chunk planner's padding bound (this tree only).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 16000
FOLDERS = {"a": "uniform 2-20 s", "b": "10 s +- 0-50 samples", "c": "exactly 10 s"}


def make(path):
    from scipy.io import wavfile
    for key, seed in (("a", 1), ("b", 2), ("c", 3)):
        d = os.path.join(path, key)
        os.makedirs(d, exist_ok=True)
        rng = np.random.default_rng(seed)
        if key == "a":
            lens = rng.integers(2 * FS, 20 * FS + 1, size=1000)
        elif key == "b":
            lens = 10 * FS + rng.integers(-50, 51, size=1000)
        else:
            lens = np.full(1000, 10 * FS)
        base = np.clip(np.round(3000.0 * rng.standard_normal(20 * FS + 64)), -32768, 32767).astype(np.int16)
        for i, n in enumerate(lens):
            off = int(rng.integers(0, 64))
            wavfile.write(os.path.join(d, "f%04d.wav" % i), FS, base[off:off + int(n)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--make")
    ap.add_argument("--time")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--out")
    ap.add_argument("--padding", type=float)
    ap.add_argument("--folders", default="abc")
    a = ap.parse_args()
    if a.make:
        make(a.make)
        return
    sys.path.insert(0, os.path.abspath(a.root))
    sys.path.insert(1, ROOT)
    import torch
    import pyaudioanalysis_b200 as pkg
    from pyaudioanalysis_b200.batch import mid_pool_batch
    import bench
    torch.cuda.set_device(0)
    pkg.MidTermFeatures.VERBOSE = False
    if a.padding is not None:
        pkg.MidTermFeatures._MAX_PADDING = a.padding
    gpu = {"name": torch.cuda.get_device_name(0), "power_limit_w": bench.ClockSampler(0).power_limit_w()}
    tag = {"root": os.path.abspath(a.root), "padding": a.padding, "gpu": gpu}
    # warm-up: CUDA context, plans, first launches
    pkg.MidTermFeatures.directory_feature_extraction(os.path.join(a.time, "c"), 1.0, 1.0, 0.05, 0.05, compute_beat=True)
    saved = {}
    for key in a.folders:
        t0 = time.perf_counter()
        feats, files, _ = pkg.MidTermFeatures.directory_feature_extraction(os.path.join(a.time, key), 1.0, 1.0, 0.05, 0.05,
                                                                           compute_beat=True)
        dt = time.perf_counter() - t0
        saved[key] = feats
        print(json.dumps(dict(tag, folder=key + ": " + FOLDERS[key], files=len(files), s=dt)), flush=True)
    if a.out:
        np.savez(a.out, **saved)
    # config 4's pooling: 1 x 68 x 143 999 frames, ratio 39, step 40
    g = torch.Generator(device="cuda")
    g.manual_seed(4)
    st = torch.randn((1, 68, 143999), generator=g, device="cuda")
    for _ in range(5):
        mid_pool_batch(st, 39, 40)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        mid_pool_batch(st, 39, 40)
    e1.record()
    torch.cuda.synchronize()
    call_ms = e0.elapsed_time(e1) / 200
    from torch.profiler import profile, ProfilerActivity         # the kernel's own time, in a run of its own
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(200):
            mid_pool_batch(st, 39, 40)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "mid_pool_kernel" in e.key]
    kernel_us = (getattr(ev[0], "device_time", None) or ev[0].cuda_time) if ev else None
    print(json.dumps(dict(tag, config="4: mid_pool_batch 1 x 68 x 143999, ratio 39 / 40", call_ms=call_ms,
                          kernel_us=kernel_us)), flush=True)


if __name__ == "__main__":
    main()

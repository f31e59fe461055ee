"""Wall-clock time of directory_feature_extraction on folders of 1000 generated files, decode included, and of the
config-4 pooling (1 x 68 x 143 999 frames, ratio 39 / 40) -> one JSON line per measurement.

    python scripts/bench_folders.py --make DIR       # 16 kHz mono PCM16: (a) 2-20 s, (b) 10 s +- 0-50 samples, (c) 10 s;
                                                     # (d) 44.1 kHz stereo PCM16, 2-10 s; (e) 16 kHz, 2-20 s, the other
                                                     # WAV flavours in turn (8 / 24 / 32-bit, float32 / 64, mono / stereo)
    python scripts/bench_folders.py --time DIR [--root PKG_ROOT] [--out FEATURES.npz] [--padding 0.25] [--folders abcde]
                                    [--warm c] [--profile]

``--root`` imports pyaudioanalysis_b200 from another tree (e.g. an older build, to alternate runs of two versions in
one session); ``--out`` saves each folder's feature matrix so two versions' outputs can be compared; ``--padding`` sets
the chunk planner's padding bound (this tree only); ``--warm`` is the folder of the untimed first call.  Every line
carries the process's peak resident memory so far (run one folder per process to compare builds).  ``--profile`` runs
the timed folders again under torch.profiler and prints the WAV decode kernel's time beside the H2D copies.

(d) runs with 0.02 / 0.01 s short-term windows (882 / 441 samples: the per-frame kernel) as a stereo collection at
44.1 kHz would; the other folders with 0.05 / 0.05 s.
"""
import argparse
import json
import os
import resource
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 16000
FOLDERS = {"a": "uniform 2-20 s", "b": "10 s +- 0-50 samples", "c": "exactly 10 s",
           "d": "44.1 kHz stereo PCM16, uniform 2-10 s", "e": "16 kHz, other WAV flavours in turn, uniform 2-20 s"}
WINDOWS = {"d": (1.0, 1.0, 0.02, 0.01)}
OTHER_FLAVOURS = [(name, ch) for name in ("u8", "s16", "s24", "s32", "f32", "f64") for ch in (1, 2)
                  if (name, ch) not in (("s16", 1), ("s16", 2))]


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
    sys.path.insert(0, ROOT)
    from tests import wavgen
    d = os.path.join(path, "d")
    os.makedirs(d, exist_ok=True)
    rng = np.random.default_rng(4)
    fs = 44100
    base = np.clip(np.round(3000.0 * rng.standard_normal((10 * fs + 64, 2))), -32768, 32767).astype(np.int16)
    for i, n in enumerate(rng.integers(2 * fs, 10 * fs + 1, size=1000)):
        off = int(rng.integers(0, 64))
        wavfile.write(os.path.join(d, "f%04d.wav" % i), fs, base[off:off + int(n)])
    d = os.path.join(path, "e")
    os.makedirs(d, exist_ok=True)
    rng = np.random.default_rng(5)
    bases = [wavgen.signal(name, ch, 20 * FS + 64, 50 + k, FS) for k, (name, ch) in enumerate(OTHER_FLAVOURS)]
    for i, n in enumerate(rng.integers(2 * FS, 20 * FS + 1, size=1000)):
        k = i % len(OTHER_FLAVOURS)
        off = int(rng.integers(0, 64))
        wavgen.write(os.path.join(d, "f%04d.wav" % i), FS, bases[k][off:off + int(n)], OTHER_FLAVOURS[k][0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--make")
    ap.add_argument("--time")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--out")
    ap.add_argument("--padding", type=float)
    ap.add_argument("--folders", default="abc")
    ap.add_argument("--warm", default="c")
    ap.add_argument("--profile", action="store_true")
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
    pkg.MidTermFeatures.directory_feature_extraction(os.path.join(a.time, a.warm), *WINDOWS.get(a.warm, (1.0, 1.0, 0.05, 0.05)),
                                                     compute_beat=True)
    saved = {}
    for key in a.folders:
        t0 = time.perf_counter()
        feats, files, _ = pkg.MidTermFeatures.directory_feature_extraction(os.path.join(a.time, key),
                                                                           *WINDOWS.get(key, (1.0, 1.0, 0.05, 0.05)),
                                                                           compute_beat=True)
        dt = time.perf_counter() - t0
        saved[key] = feats
        print(json.dumps(dict(tag, folder=key + ": " + FOLDERS[key], files=len(files), s=dt,
                              max_rss_mb=resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024)), flush=True)
    if a.out:
        np.savez(a.out, **saved)
    if a.profile:
        from torch.profiler import profile, ProfilerActivity
        for key in a.folders:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                pkg.MidTermFeatures.directory_feature_extraction(os.path.join(a.time, key),
                                                                 *WINDOWS.get(key, (1.0, 1.0, 0.05, 0.05)), compute_beat=True)
                torch.cuda.synchronize()
            rows = {}
            for e in prof.key_averages():
                if "decode_kernel" in e.key or "Memcpy HtoD" in e.key:
                    total = getattr(e, "device_time_total", None) or e.cuda_time_total
                    rows[e.key] = {"count": e.count, "total_us": total}
            print(json.dumps(dict(tag, profile=key + ": " + FOLDERS[key], events=rows)), flush=True)
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

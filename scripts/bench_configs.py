"""Timings of the BASELINE.json configs other than configs[1] (which is bench.py) -> one JSON line each.
Parity at these sizes is tests/test_gpu_configs.py; this script only measures.

    python scripts/bench_configs.py > configs.jsonl
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                              # noqa: E402
import pyaudioanalysis_b200 as pkg                        # noqa: E402
from pyaudioanalysis_b200.batch import mid_pool_batch, mid_ratios, clip_stats   # noqa: E402
from pyaudioanalysis_b200._lib import Plan               # noqa: E402

PEAK = bench.hbm_peak()[0]


def emit(d):
    print(json.dumps(d), flush=True)


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def noise(b, n, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    out = torch.empty((b, n), dtype=torch.int16, device="cuda")
    for i in range(0, b, 8):
        k = min(8, b - i)
        out[i:i + k] = (3000.0 * torch.randn((k, n), generator=g, device="cuda")).round().clamp(-32768, 32767).to(torch.int16)
    return out


def wall(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def ragged_config3():
    """Config 3 as a ragged batch: one spectrogram_batch / chromagram_batch call with lengths= against one call per clip
    (the only way before lengths= existed); kernel time with the clip statistics done beforehand, wall time with them."""
    fs, w, s, B = 44100, 882, 441, 64
    lengths = np.random.default_rng(3).integers(30 * fs, 60 * fs + 1, size=B)
    sig = noise(B, int(lengths.max()), 33)
    lens = torch.from_numpy(lengths).cuda()
    norm = clip_stats(sig, lens)
    views = [sig[b:b + 1, :int(n)] for b, n in enumerate(lengths)]
    norms = [clip_stats(v) for v in views]
    res = {"config": "3 ragged: %d clips @44.1 kHz, 20/10 ms, lengths uniform in 30-60 s (seed 3)" % B,
           "samples": int(lengths.sum())}
    for name, fn in (("spectrogram", pkg.spectrogram_batch), ("chromagram", pkg.chromagram_batch)):
        res[name + "_ragged_kernel_ms"] = timed(lambda: fn(sig, fs, w, s, norm=norm, lengths=lens), reps=5)
        res[name + "_per_clip_kernel_ms"] = timed(lambda: [fn(v, fs, w, s, norm=nv) for v, nv in zip(views, norms)], reps=3)
        res[name + "_ragged_wall_ms"] = wall(lambda: fn(sig, fs, w, s, lengths=lens))
        res[name + "_per_clip_wall_ms"] = wall(lambda: [fn(v, fs, w, s) for v in views])
    res["gpu"] = {"name": torch.cuda.get_device_name(0), "power_limit_w": bench.ClockSampler(0).power_limit_w()}
    emit(res)


def main():
    torch.cuda.set_device(0)
    pkg.ShortTermFeatures.PRINT_SPECTROGRAM_SHAPE = False
    # ---- config 1: doremi.wav through the NumPy drop-in (one clip, host in / host out, wall clock)
    g = np.load(os.path.join(ROOT, "tests", "golden", "doremi.npz"))
    x = g["x"]
    pkg.ShortTermFeatures.feature_extraction(x, 16000, 800, 400)
    t0 = time.perf_counter()
    for _ in range(20):
        F, _ = pkg.ShortTermFeatures.feature_extraction(x, 16000, 800, 400)
    dt = (time.perf_counter() - t0) / 20
    emit({"config": "1: doremi.wav 50/25 ms via ShortTermFeatures.feature_extraction (NumPy in/out, wall clock)", "ms": dt * 1e3,
          "frames": int(F.shape[1]), "frames_per_s": F.shape[1] / dt})

    # ---- config 3: 64 x 60 s @44.1 kHz, 20/10 ms: spectrogram + chromagram + feature_extraction
    B3, N3, w3, s3 = 64, 2646000, 882, 441
    c3 = noise(B3, N3, 3)
    T3 = (N3 - w3) // s3 + 1
    ms_fe = timed(lambda: pkg.feature_extraction_batch(c3, 44100, w3, s3), reps=3)
    ms_sp = timed(lambda: pkg.spectrogram_batch(c3, 44100, w3, s3), reps=3)
    ms_ch = timed(lambda: pkg.chromagram_batch(c3, 44100, w3, s3), reps=3)
    # the kernels alone (clip statistics computed once, outputs preallocated)
    n3 = clip_stats(c3)
    o_fe = torch.empty((B3, 68, T3), device="cuda")
    o_sp = torch.empty((B3, T3, 441), device="cuda")
    k_fe = timed(lambda: pkg.feature_extraction_batch(c3, 44100, w3, s3, norm=n3, out=o_fe), reps=5)
    k_sp = timed(lambda: pkg.spectrogram_batch(c3, 44100, w3, s3, norm=n3, out=o_sp), reps=5)
    k_ch = timed(lambda: pkg.chromagram_batch(c3, 44100, w3, s3, norm=n3), reps=5)
    del o_fe, o_sp
    alg = B3 * (2 * N3 + 4 * (T3 * 441 + (T3 - 1) * 12 + 13 * T3))
    emit({"config": "3: %d x 60 s @44.1 kHz, 20/10 ms" % B3, "frames_per_clip": T3, "feature_extraction_ms": ms_fe, "spectrogram_ms": ms_sp,
          "chromagram_ms": ms_ch, "feature_extraction_frames_per_s": B3 * T3 / (ms_fe * 1e-3), "spectrogram_rows_per_s": B3 * T3 / (ms_sp * 1e-3),
          "chromagram_rows_per_s": B3 * T3 / (ms_ch * 1e-3), "spectrogram_GBps": B3 * (2 * N3 + 4 * T3 * 441) / (ms_sp * 1e-3) / 1e9,
          "spectrogram_frac_of_hbm_peak": B3 * (2 * N3 + 4 * T3 * 441) / (ms_sp * 1e-3) / 1e9 / PEAK,
          "kernel_only_ms": {"feature_extraction": k_fe, "spectrogram": k_sp, "chromagram": k_ch},
          "kernel_only_spectrogram_GBps": B3 * (2 * N3 + 4 * T3 * 441) / (k_sp * 1e-3) / 1e9,
          "kernel_only_spectrogram_frac_of_hbm_peak": B3 * (2 * N3 + 4 * T3 * 441) / (k_sp * 1e-3) / 1e9 / PEAK,
          "kernel_only_feature_extraction_frames_per_s": B3 * T3 / (k_fe * 1e-3),
          "combined_algorithmic_GBps": alg / ((ms_sp + ms_ch + ms_fe) * 1e-3) / 1e9, "hbm_peak_GBps": PEAK})
    del c3
    ragged_config3()

    # ---- config 4: mid_feature_extraction over a 1 h recording, mt 1.0/1.0 s, st 50/25 ms
    N4 = 57600000
    c4 = noise(1, N4, 4)
    ratio, stepr = mid_ratios(16000, 16000, 800, 400)

    def mid():
        st = pkg.feature_extraction_batch(c4, 16000, 800, 400)
        return mid_pool_batch(st, ratio, stepr), st
    ms4 = timed(mid, reps=5)
    m, st = mid()
    T4 = st.shape[2]
    emit({"config": "4: mid_feature_extraction, 1 h @16 kHz, mt 1.0/1.0 s, st 50/25 ms (device resident)", "ms": ms4, "st_frames": int(T4),
          "mid_windows": int(m.shape[2]), "st_frames_per_s": T4 / (ms4 * 1e-3), "x_realtime": 3600.0 / (ms4 * 1e-3),
          "algorithmic_GBps": (2 * N4 + 4 * 68 * T4 + 4 * 136 * m.shape[2]) / (ms4 * 1e-3) / 1e9, "hbm_peak_GBps": PEAK})
    beat_inputs = [("4: 1 h @16 kHz, st 50/25 ms", st)]
    del c4, m

    # ---- other windows on the config-2 batch, per kernel kind
    cg = noise(1000, 160000, 5)
    norm = clip_stats(cg)
    for w, s in ((800, 400), (1024, 512), (512, 256), (640, 320), (960, 480), (480, 240), (320, 160), (400, 160), (600, 300), (2048, 1024)):
        T = (160000 - w) // s + 1
        out = torch.empty((1000, 68, T), device="cuda")
        row = {"config": "other windows: 1000 x 10 s @16 kHz", "window": w, "step": s, "frames": 1000 * T}
        for kind in (2, 3, 1, 0):
            pl = Plan(16000, w, s).prefer_kernel(kind)
            if pl.kernel_kind() != kind:
                continue
            ms = timed(lambda: pkg.feature_extraction_batch(cg, 16000, w, s, out=out, norm=norm, plan=pl), reps=3, warm=1)
            row["ms_kernel_%d" % kind] = ms
            row["frames_per_s_kernel_%d" % kind] = 1000 * T / (ms * 1e-3)
        emit(row)
    # ---- kernel 0 alone (HBM-bound)
    ms0 = timed(lambda: clip_stats(cg), reps=20)
    emit({"config": "kernel 0 (clip statistics) on 1000 x 10 s", "ms": ms0, "GBps": cg.numel() * 2 / (ms0 * 1e-3) / 1e9, "hbm_peak_GBps": PEAK,
          "frac": cg.numel() * 2 / (ms0 * 1e-3) / 1e9 / PEAK})

    # ---- kernel 4 (beat extraction) on config 2's and config 4's short-term features, beside the host function on the
    # same features (one pass over every clip, wall clock)
    beat_inputs.insert(0, ("2: 1000 x 10 s @16 kHz, st 50/25 ms", pkg.feature_extraction_batch(cg, 16000, 800, 400)))
    for name, st in beat_inputs:
        ms_k = timed(lambda: pkg.beat_extraction_batch(st, 0.025), reps=20, warm=3)
        st_h = st.cpu().numpy()
        t0 = time.perf_counter()
        for b in range(st_h.shape[0]):
            pkg.MidTermFeatures.beat_extraction(st_h[b].astype(np.float64), 0.025)
        ms_h = (time.perf_counter() - t0) * 1e3
        emit({"config": "beat extraction, " + name, "clips": int(st.shape[0]), "frames": int(st.shape[2]), "kernel_ms": ms_k,
              "host_beat_extraction_ms": ms_h, "host_over_kernel": ms_h / ms_k,
              "gpu": {"name": torch.cuda.get_device_name(0), "power_limit_w": bench.ClockSampler(0).power_limit_w()}})


if __name__ == "__main__":
    main()

"""The clipped-frame chromagram kernel -> one JSON line per measurement (the ragged config 3 is in bench_configs.py).

    python scripts/bench_rows.py                           # this build
    python scripts/bench_rows.py --ab path/to/other/tree   # plus config 3's equal-length row kernels and the clipped
                                                           # chromagram rows, alternated with another checkout whose
                                                           # library is built

Every line carries the card's name and power limit.  Kernel times are CUDA events around calls whose clip statistics
are prepared beforehand; the clipped-frame kernel's own time comes from torch.profiler (CUDA activity).
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.environ.get("B200AA_AB_TREE", ROOT))     # --ab: the package (and its library) of the other checkout
import bench                                              # noqa: E402
import pyaudioanalysis_b200 as pkg                        # noqa: E402
from pyaudioanalysis_b200.batch import clip_stats         # noqa: E402


def gpu():
    return {"name": torch.cuda.get_device_name(0), "power_limit_w": bench.ClockSampler(0).power_limit_w()}


def emit(d):
    d["gpu"] = gpu()
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


def clipped_frames(n, w, s):
    """Clipped chromagram frames of a clip of n samples, 0 when the clip is refused (a clipped frame shorter than w // 2)."""
    cl = [n - p for p in range(w, n - s, s) if p + w > n]
    return 0 if (cl and min(cl) < w // 2) or n - s - w < 0 else len(cl)


def clipped_kernel_alone():
    from torch.profiler import ProfilerActivity, profile
    for fs, w, s, B, lo, hi in ((16000, 800, 200, 1000, 9 * 16000, 10 * 16000), (16000, 16000, 8000, 64, 20 * 16000, 30 * 16000)):
        rng = np.random.default_rng(w + s)
        lengths = []
        while len(lengths) < B:              # every clip with clipped frames the chromagram computes
            n = int(rng.integers(lo, hi))
            if clipped_frames(n, w, s):
                lengths.append(n)
        sig = noise(B, max(lengths), 7)
        lens = torch.tensor(lengths, dtype=torch.int64, device="cuda")
        norm = clip_stats(sig, lens)
        for _ in range(2):
            pkg.chromagram_batch(sig, fs, w, s, norm=norm, lengths=lens)
        torch.cuda.synchronize()
        reps = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                pkg.chromagram_batch(sig, fs, w, s, norm=norm, lengths=lens)
            torch.cuda.synchronize()
        us = {}
        for ev in prof.key_averages():
            for key in ("clipped_chroma_kernel", "st_solo_kernel", "st_fast_kernel", "st_generic_kernel"):
                if key in ev.key:
                    us[key] = us.get(key, 0.0) + ev.device_time_total / reps
        emit({"config": "clipped-frame kernel, %d clips @%d Hz, window %d / step %d" % (B, fs, w, s),
              "clipped_frames": int(sum(clipped_frames(n, w, s) for n in lengths)),
              "clipped_kernel_us": us.get("clipped_chroma_kernel"), "row_kernel_us": {k: v for k, v in us.items() if k != "clipped_chroma_kernel"}})


def ab_one(out_path):
    """This build's config-3 equal-length row kernels and its chromagram of clips with clipped last frames."""
    fs, w, s, B, N = 44100, 882, 441, 64, 2646000
    c3 = noise(B, N, 3)
    n3 = clip_stats(c3)
    o_sp = torch.empty((B, (N - w) // s + 1, w // 2), device="cuda")
    res = {"tree": os.environ.get("B200AA_AB_TREE", ROOT),
           "config3_spectrogram_kernel_ms": timed(lambda: pkg.spectrogram_batch(c3, fs, w, s, norm=n3, out=o_sp), reps=5),
           "config3_chromagram_kernel_ms": timed(lambda: pkg.chromagram_batch(c3, fs, w, s, norm=n3), reps=5)}
    del c3, o_sp
    from oracle import st_oracle as O
    outs = {"doremi": pkg.ShortTermFeatures.chromagram(np.load(os.path.join(ROOT, "tests", "golden", "doremi.npz"))["x"], 16000, 800, 400)[0],
            "chroma_clipped": pkg.ShortTermFeatures.chromagram(O.synth_clip(22, 16300, 16000), 16000, 800, 400)[0]}
    for fs_, w_, s_, n_ in [(16000, 800, 400, 40000), (44100, 882, 441, 50000), (16000, 800, 800, 24000), (16000, 800, 200, 16400),
                            (16000, 400, 160, 16000), (8000, 600, 300, 12000), (44100, 882, 882, 30000), (44100, 882, 300, 20001)]:
        clips = np.stack([O.synth_clip(60 + i, n_, fs_) for i in range(3)])
        outs["row_kernels_%d_%d_%d_%d" % (fs_, w_, s_, n_)] = pkg.chromagram_batch(torch.from_numpy(clips).cuda(), fs_, w_, s_).cpu().numpy()
    np.savez(out_path, **outs)
    print(json.dumps(res), flush=True)


def ab(other):
    out_dir = tempfile.mkdtemp(prefix="bench_rows_")     # the two builds' outputs, compared below
    files = {}
    for rnd in range(3):
        for name, lib in (("other", other), ("this", None)):
            env = dict(os.environ)
            env.pop("B200AA_AB_TREE", None)
            if lib:
                env["B200AA_AB_TREE"] = os.path.abspath(lib)
            path = os.path.join(out_dir, "rows_ab_%s.npz" % name)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--ab-one", path], env=env, capture_output=True, text=True)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            d = json.loads(line[-1]) if line else {"error": (r.stderr or r.stdout)[-600:]}
            d.update({"round": rnd, "build": name})
            emit(d)
            files[name] = path
    a, b = np.load(files["other"]), np.load(files["this"])
    diff = {k: float(np.max(np.abs(a[k].astype(np.float64) - b[k]))) for k in a.files}
    emit({"config": "chromagram rows with clipped last frames: largest |this - other build|", "max_abs_diff": diff,
          "rows_differing": {k: int(np.any(a[k] != b[k], axis=-1).sum()) for k in a.files}})
    shutil.rmtree(out_dir)


if __name__ == "__main__":
    torch.cuda.set_device(0)
    pkg.ShortTermFeatures.PRINT_SPECTROGRAM_SHAPE = False
    if "--ab-one" in sys.argv:
        ab_one(sys.argv[sys.argv.index("--ab-one") + 1])
        sys.exit(0)
    clipped_kernel_alone()
    if "--ab" in sys.argv:
        ab(sys.argv[sys.argv.index("--ab") + 1])

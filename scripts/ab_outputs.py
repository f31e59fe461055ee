"""Byte-for-byte A/B of the short-term outputs of two builds of libb200aa.so (on the GPU).

    python scripts/ab_outputs.py /path/to/other/libb200aa.so [OUT_DIR]
    python scripts/ab_outputs.py --time /path/to/other/libb200aa.so   # kernel times of the row / generic paths, alternated

Each build runs in its own process (the library is chosen at import time through B200AA_LIB) and writes every output to
OUT_DIR/<build>.npz: feature_extraction_batch with deltas on and off, spectrogram_batch and chromagram_batch equal-length
and ragged (lengths=), int16 and float32, through every kernel kind tests.kernels.plans reaches, at the (fs, window, step)
below.  Prints one JSON line: arrays compared, and the names of those whose bytes differ.  A refactor of the kernels or
their launchers should leave it empty.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = [(16000, 800, 400), (16000, 800, 200), (44100, 882, 441), (16000, 400, 160), (16000, 600, 300),
           (16000, 1024, 300), (16000, 551, 200), (16000, 20000, 10000)]


def one(path):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import pyaudioanalysis_b200 as pkg
    from tests.kernels import KIND_NAMES, plans, ragged
    rng = np.random.default_rng(20261016)
    res = {}
    for fs, w, s in CONFIGS:
        n = w + (7 * w // s) * s        # (n - w) % s == 0: the last clipped frame keeps 2s >= K samples (not refused)
        t = np.arange(n)
        x16 = np.stack([(6000 * np.sin(2 * np.pi * (110 + 37 * i) * t / fs) + rng.normal(0, 900, n)).astype(np.int16) for i in range(5)])
        lens = [n, n - 1, n - w // 3, 2 * w + s // 2, w + s + 1, w // 2]       # clipped frames, a refused clip
        for dt, x in (("i16", x16), ("f32", x16.astype(np.float32) / 32768)):
            d = torch.from_numpy(x).cuda()
            r, rl = ragged([x[i % len(x), :m] for i, m in enumerate(lens)], x.dtype)
            for i, (kind, pl) in enumerate(plans(fs, w, s)):      # i: the default plan and a preferred one may share a kind
                key = "%d_%d_%d_%s%d_%s_" % (fs, w, s, KIND_NAMES[kind], i, dt)
                for deltas in (True, False):
                    res[key + "features_%d" % deltas] = pkg.feature_extraction_batch(d, fs, w, s, deltas=deltas, plan=pl)
                res[key + "features_ragged"] = pkg.feature_extraction_batch(r, fs, w, s, lengths=rl, plan=pl)
                res[key + "spectrogram"] = pkg.spectrogram_batch(d, fs, w, s, plan=pl)
                res[key + "spectrogram_ragged"] = pkg.spectrogram_batch(r, fs, w, s, plan=pl, lengths=rl)
                res[key + "chromagram"] = pkg.chromagram_batch(d, fs, w, s, plan=pl)
                res[key + "chromagram_ragged"] = pkg.chromagram_batch(r, fs, w, s, plan=pl, lengths=rl)
    torch.cuda.synchronize()
    np.savez(path, **{k: v.cpu().numpy() for k, v in res.items()})


def time_rows():
    """--time: kernel milliseconds (median of 9 calls, CUDA events; clip statistics and spectrogram outputs prepared
    beforehand) of the generic kernel's forms, the BIG forms at a 20000-sample window, and CTA row kernels (EVEN without
    run staging at 480 / 320, run staging at 800)."""
    sys.path.insert(0, ROOT)
    import torch
    import pyaudioanalysis_b200 as pkg
    g = torch.Generator(device="cuda")
    g.manual_seed(5)

    def ms(fn):
        ts = []
        for i in range(11):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return sorted(ts[2:])[4]

    res = {}
    for fs, w, s, B, secs in ((16000, 1000, 500, 64, 30), (16000, 20000, 10000, 16, 60), (16000, 480, 244, 64, 30),
                              (16000, 320, 162, 64, 30), (16000, 800, 400, 64, 30)):
        x = torch.randint(-12000, 12000, (B, fs * secs), generator=g, device="cuda", dtype=torch.int16)
        lens = torch.randint(fs * secs // 2, fs * secs + 1, (B,), generator=g, device="cuda")
        norm, rnorm = pkg.clip_stats(x), pkg.clip_stats(x, lens)
        sp = pkg.spectrogram_batch(x, fs, w, s, norm=norm)
        key = "%d/%d " % (w, s)
        res[key + "spectrogram"] = ms(lambda: pkg.spectrogram_batch(x, fs, w, s, norm=norm, out=sp))
        res[key + "chromagram"] = ms(lambda: pkg.chromagram_batch(x, fs, w, s, norm=norm))
        if w in (1000, 20000):
            res[key + "features"] = ms(lambda: pkg.feature_extraction_batch(x, fs, w, s, norm=norm))
        if w in (20000, 320):
            res[key + "spectrogram ragged"] = ms(lambda: pkg.spectrogram_batch(x, fs, w, s, norm=rnorm, out=sp.zero_(), lengths=lens))
            res[key + "chromagram ragged"] = ms(lambda: pkg.chromagram_batch(x, fs, w, s, norm=rnorm, lengths=lens))
    print(json.dumps({"lib": os.environ.get("B200AA_LIB") or "this", "gpu": torch.cuda.get_device_name(0), "kernel_ms": res}), flush=True)


def main(other, out_dir):
    os.makedirs(out_dir, exist_ok=True)
    files = {}
    for name, lib in (("this", None), ("other", other)):
        env = dict(os.environ)
        env.pop("B200AA_LIB", None)
        if lib:
            env["B200AA_LIB"] = os.path.abspath(lib)
        files[name] = os.path.join(out_dir, name + ".npz")
        subprocess.run([sys.executable, os.path.abspath(__file__), "--one", files[name]], env=env, check=True)
    import numpy as np
    a, b = np.load(files["this"]), np.load(files["other"])
    differ = sorted(k for k in set(a.files) | set(b.files) if k not in a.files or k not in b.files or a[k].tobytes() != b[k].tobytes())
    print(json.dumps({"arrays": len(set(a.files) | set(b.files)), "differ": differ}), flush=True)
    return 1 if differ else 0


if __name__ == "__main__":
    if sys.argv[1] == "--one":
        one(sys.argv[2])
    elif sys.argv[1] == "--time-one":
        time_rows()
    elif sys.argv[1] == "--time":                # three rounds, the two builds alternated
        for _ in range(3):
            for lib in (None, sys.argv[2]):
                env = dict(os.environ)
                env.pop("B200AA_LIB", None)
                if lib:
                    env["B200AA_LIB"] = os.path.abspath(lib)
                subprocess.run([sys.executable, os.path.abspath(__file__), "--time-one"], env=env, check=True)
    else:
        sys.exit(main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "ab_outputs"))

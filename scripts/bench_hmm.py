"""Time HMM segmentation (kernel 7) through the drop-in audioSegmentation on two workloads:

  file    one 1 h 16 kHz file at a 1.0 s mid window / 0.1 s mid step (36 000 windows) with a 10-state model, through
          hmm_segmentation (read, features, decode);
  folder  evaluate_segmentation_classification_dir over 1000 generated 60 s files with .segments files (one ragged
          batch, one decode per chunk).

For each: the wall time of the drop-in (best of --reps, after one warm-up call), the device time of the decode alone
(CUDA events around hmm_decode_batch on the resident mid-term batch), and, as the CPU comparison, the NumPy
restatement of GaussianHMM.predict (tests/hmm_oracle.py: hmmlearn's density and Viterbi) on the same matrices -- hmmlearn
itself is not installed -- with its labels compared to the drop-in's in the same run.  Prints one JSON line with the
card's name and power limit, read in the same call.

    python scripts/bench_hmm.py [--files 1000] [--reps 3]
"""
import argparse
import contextlib
import glob
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def write_wav(path, x, fs):
    from tests import wavgen
    wavgen.write(path, fs, x, "s16")


def signal(rng, seconds, fs, n_classes):
    """Class-wise tones and noise in 2-6 s segments: (int16 samples, segment rows)."""
    n = seconds * fs
    x = np.zeros(n, dtype=np.float32)
    rows, a = [], 0
    order = rng.permutation(n_classes)         # every class in every file: the evaluation adds per-file confusion matrices
    while a < seconds:
        b = min(seconds, a + int(rng.integers(2, 7)))
        c = int(order[len(rows) % n_classes])
        t = np.arange((b - a) * fs, dtype=np.float32) / fs
        x[a * fs:b * fs] = 0.3 * np.sin(2 * np.pi * (110.0 * (c + 1)) * t) + 0.05 * (c % 3) * rng.standard_normal(t.size)
        rows.append("%d.0\t%d.0\tc%d" % (a, b, c))
        a = b
    x += 0.01 * rng.standard_normal(n).astype(np.float32)
    return np.clip(np.round(x * 20000), -32768, 32767).astype(np.int16), rows


def best_of(reps, fn):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
    return min(times), out


def device_decode_ms(mid, model, counts, reps):
    import torch
    from pyaudioanalysis_b200.consumers import hmm_decode_batch
    hmm_decode_batch(mid, model, counts)
    best = None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        hmm_decode_batch(mid, model, counts)
        b.record()
        b.synchronize()
        best = a.elapsed_time(b) if best is None else min(best, a.elapsed_time(b))
    return best


def host_predict(mids, hmm):
    from tests import hmm_oracle as H
    return [H.predict(m, hmm.startprob_, hmm.transmat_, hmm.means_, hmm.covars_) for m in mids]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    from pyaudioanalysis_b200 import audioSegmentation as S
    from pyaudioanalysis_b200.consumers import HmmModel
    fs = 16000
    rng = np.random.default_rng(2026)
    res = {"card": card()}
    with tempfile.TemporaryDirectory() as tmp:
        # ---- one hour, 10 states
        x, rows = signal(rng, 3600, fs, 10)
        wav = os.path.join(tmp, "hour.wav")
        write_wav(wav, x, fs)
        with open(wav.replace(".wav", ".segments"), "w") as f:
            f.write("\n".join(rows) + "\n")
        model = os.path.join(tmp, "hmm10")
        hmm, _ = S.train_hmm_from_file(wav, wav.replace(".wav", ".segments"), model, 1.0, 0.1)
        S.hmm_segmentation(wav, model)
        wall, (labels, _, _, _) = best_of(args.reps, lambda: S.hmm_segmentation(wav, model))
        mid, counts, _, _ = S._mid_batch([wav], 1.0, 0.1)
        dev = device_decode_ms(mid, HmmModel(hmm), counts, args.reps)
        feats = [mid[0, :, :counts[0]].double().cpu().numpy()]
        host, want = best_of(1, lambda: host_predict(feats, hmm))
        res["file"] = {"windows": int(counts[0]), "states": int(hmm.means_.shape[0]), "drop_in_wall_s": wall,
                       "decode_device_ms": dev, "host_restatement_s": host, "labels_equal": bool(np.array_equal(labels, want[0]))}
        print(json.dumps(res["file"]), flush=True)
        # ---- a folder of 60 s files
        folder = os.path.join(tmp, "dir")
        os.makedirs(folder)
        for k in range(args.files):
            x, rows = signal(rng, 60, fs, 10)
            write_wav(os.path.join(folder, "f%04d.wav" % k), x, fs)
            with open(os.path.join(folder, "f%04d.segments" % k), "w") as f:
                f.write("\n".join(rows) + "\n")
        with contextlib.redirect_stdout(io.StringIO()):
            S.evaluate_segmentation_classification_dir(folder, model, "hmm")
        out = io.StringIO()

        def run():
            with contextlib.redirect_stdout(out):
                S.evaluate_segmentation_classification_dir(folder, model, "hmm")
        wall, _ = best_of(args.reps, run)
        files = glob.glob(folder + os.sep + "*.wav")
        mid, counts, _, _ = S._mid_batch(files, 1.0, 0.1)
        dev = device_decode_ms(mid, HmmModel(hmm), counts, args.reps)
        got = S._decode_mids(mid, hmm, counts)
        mids = [mid[b, :, :n].double().cpu().numpy() for b, n in enumerate(counts)]
        host, want = best_of(1, lambda: host_predict(mids, hmm))
        res["folder"] = {"files": len(files), "windows": int(sum(counts)), "drop_in_wall_s": wall, "decode_device_ms": dev,
                         "host_restatement_s": host,
                         "labels_equal": all(np.array_equal(a, b) for a, b in zip(got, want))}
        print(json.dumps(res["folder"]), flush=True)
    torch.cuda.synchronize()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

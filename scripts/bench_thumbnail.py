"""Time music thumbnails (kernel 10) on the GPU against the reference's steps on the host.  Prints one JSON line per
measurement, the first naming the card and its power limit.

    python scripts/bench_thumbnail.py [--host-max 2400] [--tracks 1000] [--chunk 100]

- device: CUDA events around b200aa_music_thumbnail for one seeded standardised [T, 68] track at T = 600 / 2 400 / 7 200
  (0.5 s step, 10 s thumbnails: m = 20), the median of several calls;
- host: the reference's steps on the same matrix on this machine's CPU (one thread of NumPy / SciPy): StandardScaler and
  the cosine pdist, convolve2d(S, eye(m), 'valid'), and the Python masking loop, restated below statement by statement;
  timed up to --host-max frames;
- batch: ``music_thumbnailing_batch`` over --tracks five-minute 16 kHz tracks in chunks of --chunk, wall clock, from
  signals already on the GPU and from WAV files decoded by ``audioio.load_batch`` (files written to a temporary
  directory first, not timed)."""
import argparse
import hashlib
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    import torch
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    except OSError:
        limit = "unknown"
    return {"card": torch.cuda.get_device_name(), "power_limit": limit}


def host_steps(st, m, step):
    """music_thumbnailing's steps after the features (audioSegmentation.py:51-55, :1145-1161), timed by stage."""
    import scipy.signal
    from scipy.spatial import distance
    from sklearn.preprocessing import StandardScaler
    t0 = time.perf_counter()
    n = StandardScaler().fit_transform(st.T).T
    S = 1.0 - distance.squareform(distance.pdist(n.T, "cosine"))
    t1 = time.perf_counter()
    C = scipy.signal.convolve2d(S, np.eye(m, m), "valid")
    t2 = time.perf_counter()
    min_sm = np.min(C)
    for i in range(C.shape[0]):
        for j in range(C.shape[1]):
            if abs(i - j) < 5.0 / step or i > j:
                C[i, j] = min_sm
    t3 = time.perf_counter()
    return {"scaler_pdist_s": t1 - t0, "convolve2d_s": t2 - t1, "mask_loop_s": t3 - t2}


def device_ms(X, m, gap, reps):
    import torch
    from pyaudioanalysis_b200._lib import check, lib
    from pyaudioanalysis_b200.batch import _stream
    T = X.shape[0]
    R = T - m + 1
    frames = np.array([T], dtype=np.int64)
    limits = np.array([0, R], dtype=np.int64)
    C = torch.empty(R * R, dtype=torch.float64, device="cuda")
    idx = torch.empty(4, dtype=torch.int64, device="cuda")

    def call():
        check(lib().b200aa_music_thumbnail(ctypes.c_void_p(X.data_ptr()), X.shape[1], X.shape[1],
                                           ctypes.c_void_p(frames.ctypes.data), 1, m, gap,
                                           ctypes.c_void_p(limits.ctypes.data), None, ctypes.c_void_p(C.data_ptr()),
                                           ctypes.c_void_p(idx.data_ptr()), _stream()))
    call()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def tracks(rng, n, seconds, fs):
    """n seeded int16 tracks of one-second blocks of noise at random levels."""
    out = np.empty((n, seconds * fs), dtype=np.int16)
    for b in range(n):
        levels = rng.uniform(400, 7200, size=(seconds, 1)).astype(np.float32)
        out[b] = (rng.standard_normal(size=(seconds, fs), dtype=np.float32) * levels).astype(np.int16).ravel()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--host-max", type=int, default=2400)
    ap.add_argument("--tracks", type=int, default=1000)
    ap.add_argument("--chunk", type=int, default=100)
    args = ap.parse_args()
    import torch
    from scipy.io import wavfile
    from pyaudioanalysis_b200.audioSegmentation import standardise
    from pyaudioanalysis_b200.audioio import load_batch
    from pyaudioanalysis_b200.batch import music_thumbnailing_batch
    print(json.dumps(card()), flush=True)
    rng = np.random.default_rng(0)
    step, m = 0.5, 20
    for T in (600, 2400, 7200):
        st = rng.normal(size=(68, T)) + np.sin(np.arange(T) / rng.uniform(3, 30, size=(68, 1)))
        X = torch.from_numpy(standardise(st)).cuda()
        rec = {"T": T, "device_ms": device_ms(X, m, 5.0 / step, 20 if T < 7200 else 5)}
        if T <= args.host_max:
            rec.update(host_steps(st, m, step))
        print(json.dumps(rec), flush=True)

    fs, seconds = 16000, 300
    n_chunks = (args.tracks + args.chunk - 1) // args.chunk
    chunk = tracks(rng, args.chunk, seconds, fs)
    sig = torch.from_numpy(chunk).cuda()
    music_thumbnailing_batch(sig[:2], fs)                   # plans and the library loaded outside the timing
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_chunks):
        times, _ = music_thumbnailing_batch(sig, fs)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    print(json.dumps({"batch": "signals on the GPU", "tracks": n_chunks * args.chunk, "seconds_per_track": seconds,
                      "wall_s": wall, "times_sha1": hashlib.sha1(np.ascontiguousarray(times).tobytes()).hexdigest()}),
          flush=True)
    with tempfile.TemporaryDirectory() as d:
        paths = []
        for b in range(args.chunk):
            paths.append(os.path.join(d, "t%03d.wav" % b))
            wavfile.write(paths[-1], fs, chunk[b])
        del sig
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n_chunks):
            fs2, s2, lengths = load_batch(paths)
            times, _ = music_thumbnailing_batch(s2, fs2, lengths=lengths)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    print(json.dumps({"batch": "WAV files decoded by load_batch", "tracks": n_chunks * args.chunk,
                      "seconds_per_track": seconds, "wall_s": wall}), flush=True)


if __name__ == "__main__":
    main()

"""Time speaker diarization's silhouette stage (kernel 9 against scipy + NumPy on the host), its scaler, outlier rule and
LDA pooling (kernel 11 against scikit-learn, scipy and NumPy on the host), and ``diarize`` end to end on a synthetic 1 h
mid-term matrix with a per-stage breakdown.  Prints one JSON line per measurement.

    python scripts/bench_diarization.py [--host-max 3600] [--skip-diarize]

The silhouette stage is timed for K = 2..9 on seeded labels at M = 3 600 and 36 000 windows of D = 146 columns; scipy is
timed only up to --host-max windows (at 36 000 one count takes minutes on one core)."""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def host_means(X, labels, K):
    from scipy.spatial import distance
    A, B = np.full(K, np.nan), np.full((K, K), np.nan)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for c in range(K):
            xc = X[labels == c]
            A[c] = np.mean(distance.pdist(xc.T))
            for c2 in range(K):
                if c2 != c:
                    B[c, c2] = np.mean(distance.cdist(xc, X[labels == c2]))
    return A, B


def front_stage(rng, dev):
    """Kernel 11 against the host steps it replaces: the scaler and the outlier rule of a 1 h matrix (M = 36 000 windows
    of D = 146), and the LDA branch's pooling plus its scaler at T = 72 000 short-term frames (1 h at 50 ms, ratio 40).
    Device times include the upload of the host matrix and the copies back that diarize makes."""
    import torch
    from scipy.spatial import distance
    from sklearn.preprocessing import StandardScaler
    from pyaudioanalysis_b200 import audioSegmentation as S
    from pyaudioanalysis_b200.consumers import outlier_columns, pool_frames_batch, standard_scale_batch

    def best(fn, reps):
        out, ts = None, []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return out, min(ts) * 1e3

    def same(a, b):
        return bool(np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64)))

    feats = rng.normal(size=(146, 36000)) * np.exp(rng.normal(size=(146, 1)))

    def host_a():
        x = StandardScaler().fit_transform(feats.T)
        d = np.sum(distance.squareform(distance.pdist(x.T)), axis=0)
        return x, np.nonzero(d < 1.1 * np.mean(d))[0]

    def dev_a():
        y = standard_scale_batch(torch.from_numpy(feats).cuda().t())[0]
        return y.t().cpu().numpy().T, outlier_columns(y)[0]
    (hx, hk), host_ms = best(host_a, 3)
    best(dev_a, 2)
    (dx, dk), dev_ms = best(dev_a, 5)
    print(json.dumps({"stage": "scaler_outliers", "M": 36000, "D": 146, "host_ms": round(host_ms, 2),
                      "gpu_ms": round(dev_ms, 3), "bit_equal": same(hx, dx) and bool(np.array_equal(hk, dk)),
                      "device": dev}), flush=True)
    st = (rng.normal(size=(68, 72000)) * 3).astype(np.float32)
    post = rng.random((72000, 12))

    def host_b():
        pooled = S.pool_frames(st, 40)
        return pooled, StandardScaler().fit_transform(S._with_posteriors(pooled, [post]).T).T

    def dev_b():
        pooled_dev = pool_frames_batch(torch.from_numpy(st).cuda(), 40)
        pooled = pooled_dev.cpu().numpy()
        red = torch.cat([pooled_dev, torch.from_numpy(post.T + 1e-4).cuda()])
        return pooled, standard_scale_batch(red.t())[0].t().cpu().numpy()
    (hp, hr), host_ms = best(host_b, 1)
    best(dev_b, 2)
    (dp, dr), dev_ms = best(dev_b, 5)
    print(json.dumps({"stage": "lda_pool_scaler", "T": 72000, "ratio": 40, "host_ms": round(host_ms, 1),
                      "gpu_ms": round(dev_ms, 3), "bit_equal": same(hp, dp) and same(hr, dr), "device": dev}), flush=True)


def main():
    import torch
    from pyaudioanalysis_b200 import audioSegmentation as S
    from pyaudioanalysis_b200.consumers import cluster_distance_means
    ap = argparse.ArgumentParser()
    ap.add_argument("--host-max", type=int, default=3600)
    ap.add_argument("--skip-diarize", action="store_true")
    args = ap.parse_args()
    dev = torch.cuda.get_device_properties(0).name
    rng = np.random.default_rng(0)
    for M in (3600, 36000):
        X = rng.normal(size=(M, 146))
        t = torch.from_numpy(X).cuda()
        cluster_distance_means(t, rng.integers(0, 2, size=M), 2)         # warm-up
        torch.cuda.synchronize()
        for K in range(2, 10):
            labels = rng.integers(0, K, size=M)
            reps = 5
            t0 = time.perf_counter()
            for _ in range(reps):
                A, B = cluster_distance_means(t, labels, K)
            torch.cuda.synchronize()
            gpu_ms = (time.perf_counter() - t0) / reps * 1e3
            row = {"stage": "silhouette_means", "M": M, "D": 146, "K": K, "gpu_ms": round(gpu_ms, 3), "device": dev}
            if M <= args.host_max:
                t0 = time.perf_counter()
                hA, hB = host_means(X, labels, K)
                row["host_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                row["bit_equal"] = bool(np.array_equal(np.nan_to_num(A.cpu().numpy()), np.nan_to_num(hA)) and
                                        np.array_equal(np.nan_to_num(B.cpu().numpy()), np.nan_to_num(hB)))
            else:
                row["host_ms"] = "not measured"
            print(json.dumps(row), flush=True)
    front_stage(rng, dev)
    if args.skip_diarize:
        return
    # diarize on a synthetic 1 h matrix at the default 0.1 s step: 36 000 windows, 136 features, two seeded SVCs
    from sklearn.svm import SVC
    M, F = 36000, 136
    centres = rng.normal(size=(4, F)) * 2
    who = np.repeat(rng.integers(0, 4, size=M // 100), 100)
    mid = (centres[who] + rng.normal(size=(M, F))).T
    models = []
    for C in (10, 2):
        Xt = rng.normal(size=(40 * C, F)) + (np.arange(40 * C) % C)[:, None] * 0.3
        y = np.arange(40 * C) % C
        mean, std = Xt.mean(axis=0), Xt.std(axis=0)
        models.append((SVC(probability=True, random_state=0).fit((Xt - mean) / std, y), mean, std))
    stages = {"host_svm_s": 0.0, "host_kmeans_s": 0.0, "kernel9_s": 0.0}

    def timed(key, fn):
        def run(*a):
            t0 = time.perf_counter()
            out = fn(*a)
            torch.cuda.synchronize()
            stages[key] += time.perf_counter() - t0
            return out
        return run
    t0 = time.perf_counter()
    post = [timed("host_svm_s", S._posteriors)(mid.T, m) for m in models]
    np.random.seed(0)
    t1 = time.perf_counter()
    means = S.cluster_means_gpu
    S.cluster_means_gpu = timed("kernel9_s", means)      # diarize's default: the matrix is uploaded once, before the loop
    try:
        cls, info = S.diarize(mid, None, 0, 0.1, 0.1, 0, posteriors=post, cluster=timed("host_kmeans_s", S._kmeans),
                              details=True)
    finally:
        S.cluster_means_gpu = means
    total = time.perf_counter() - t0
    rest = (time.perf_counter() - t1) - stages["host_kmeans_s"] - stages["kernel9_s"]
    t2 = time.perf_counter()
    S._hmm_smooth(np.ascontiguousarray(np.random.default_rng(1).normal(size=(M, 148))), info["labels"][-1])
    hmm_s = time.perf_counter() - t2
    print(json.dumps({"stage": "diarize_1h", "M": M, "total_s": round(total, 2),
                      **{k: round(v, 3) for k, v in stages.items()}, "hmm_alone_s": round(hmm_s, 3),
                      "scaler_outliers_hmm_medfilt_s": round(rest, 3), "num_speakers": info["num_speakers"],
                      "device": dev}), flush=True)


if __name__ == "__main__":
    main()

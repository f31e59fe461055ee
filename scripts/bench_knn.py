"""Time b200aa_knn_classify (kernel 5) on a seeded model shaped like the reference's knn_4class (N = 15 819, F = 136, k = 13,
4 classes): one hour of 1 s windows (n = 3 600) and a folder's worth (n = 65 536).  Kernel times are CUDA events around
launches after a warm-up, scratch allocation included.  The FP64 bound is arithmetic, not a measurement: 3 n N F
operations (sub, mul, add; none can fuse) at the H100 SXM data sheet's 34 TFLOP/s FP64, i.e. 1.7e13 DADD / DMUL per s.
The host baseline is the reference's per-vector Knn.classify loop (audioTrainTest.py:33-49, restated: cdist, argsort, vote)
at n = 3 600; knn_classify_matrix's [n x N x F] temporary (62 GB there) cannot be allocated.

    python scripts/bench_knn.py [--reps 10] [--host-n 3600]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.spatial import distance

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pyaudioanalysis_b200 import consumers  # noqa: E402

FP64_OPS_PER_S = 1.7e13


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def time_kernel(model, q, reps):
    consumers.knn_classify_batch(model, q)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        consumers.knn_classify_batch(model, q)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def host_loop(feats, labels, k, q):
    """The reference's Knn.classify, one vector at a time."""
    n_classes = np.unique(labels).shape[0]
    t0 = time.perf_counter()
    for v in q:
        y_dist = distance.cdist(feats, v.reshape(1, v.shape[0]), "euclidean").T
        i_sort = np.argsort(y_dist)
        P = np.zeros((n_classes,))
        for i in range(n_classes):
            P[i] = np.nonzero(labels[i_sort[0][0:k]] == i)[0].shape[0] / float(k)
        np.argmax(P)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-n", type=int, default=3600)
    args = ap.parse_args()
    rng = np.random.default_rng(4)
    N, F, k = 15819, 136, 13
    labels = rng.integers(0, 4, size=N).astype(np.float64)
    feats = rng.normal(size=(N, F)) + labels[:, None] * 0.1
    model = consumers.KnnModel(type("Knn", (), {"features": feats, "labels": labels, "neighbors": k})())
    print("card:", card())
    rows = []
    for n in (3600, 65536):
        q = torch.from_numpy(rng.normal(size=(n, F))).cuda()
        ms = time_kernel(model, q, args.reps)
        ops = 3.0 * n * N * F
        bound_ms = ops / FP64_OPS_PER_S * 1e3
        row = {"n": n, "N": N, "F": F, "k": k, "kernel_ms": round(ms, 3), "fp64_ops": ops, "fp64_bound_ms": round(bound_ms, 3),
               "share_of_fp64_bound": round(bound_ms / ms, 3)}
        if n == 3600 and args.host_n:
            host = q[: args.host_n].cpu().numpy()
            row["host_knn_classify_loop_ms"] = round(host_loop(feats, labels, k, host) * n / host.shape[0], 1)
        rows.append(row)
        print(json.dumps(row))


if __name__ == "__main__":
    main()

"""Time the kNN model selection on the GPU (audioTrainTest.evaluate_classifier, kernel 6) against the host oracle loop
(tests/knn_cv_oracle.py: scikit-learn's train_test_split, StandardScaler and metrics per experiment, scipy's cdist and a
stable argsort per problem, i.e. the reference's loop with each problem's test rows classified as one matrix) on:

* the reference's 3_class features (tests/golden/knn_cv.npz case a: 120 x 136, 3 336 problems);
* seeded 999 x 136 and 4 998 x 136 sets of 3 classes (tests.knn_cv_oracle.seeded_features),

all with the 8 neighbour counts of extract_features_and_train and the default n_exp.  The drop-in's wall clock covers
the whole call (split draw, upload, device work, copy back and the printed report); its device part is CUDA events
around the one knn_cross_validate call, its host part the rest.  The GPU's predictions are checked against the oracle's.

    python scripts/bench_knn_cv.py [--reps 3] [--no-host]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pyaudioanalysis_b200 import audioTrainTest as at  # noqa: E402
from pyaudioanalysis_b200 import consumers  # noqa: E402
from tests import knn_cv_oracle as oracle  # noqa: E402

PARAMS = np.array([1, 3, 5, 7, 9, 11, 13, 15])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def workloads():
    g = np.load(os.path.join(ROOT, "tests", "golden", "knn_cv.npz"))
    yield "3_class", np.split(g["a_X"], np.cumsum(g["a_sizes"])[:-1])
    yield "seeded_999", oracle.seeded_features(999, (333, 333, 333), 136)
    yield "seeded_4998", oracle.seeded_features(4998, (1666, 1666, 1666), 136)


def drop_in(feats, names, seed):
    """(wall ms, device ms, return value) of one evaluate_classifier call; the device part timed with CUDA events."""
    dev = []
    inner = consumers.knn_cross_validate

    def timed(*a, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = inner(*a, **kw)
        e.record()
        e.synchronize()
        dev.append(s.elapsed_time(e))
        return out

    consumers.knn_cross_validate = timed
    try:
        np.random.seed(seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            ret = at.evaluate_classifier(feats, names, "knn", PARAMS, 1)
        wall = (time.perf_counter() - t0) * 1e3
    finally:
        consumers.knn_cross_validate = inner
    return wall, dev[0], ret


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-host", action="store_true")
    args = ap.parse_args()
    print("card:", card())
    for name, feats in workloads():
        names = ["c%d" % i for i in range(len(feats))]
        X, y = at.features_to_matrix(feats)
        n_exp = int(50000 / X.shape[0]) + 1
        drop_in(feats, names, 0)                                  # warm-up: module load, allocator
        runs = [drop_in(feats, names, 1 + r) for r in range(args.reps)]
        wall, dev = min(r[0] for r in runs), min(r[1] for r in runs)
        row = {"workload": name, "n": X.shape[0], "F": X.shape[1], "problems": len(PARAMS) * n_exp,
               "gpu_wall_ms": round(wall, 1), "gpu_device_ms": round(dev, 2), "gpu_host_ms": round(wall - dev, 1),
               "gpu_wall_ms_all": [round(r[0], 1) for r in runs]}
        if not args.no_host:
            np.random.seed(1)
            splits = at.draw_splits(X, y, len(PARAMS), n_exp, 0.90)
            ks = [int(k) for k in PARAMS for _ in range(n_exp)]
            t0 = time.perf_counter()
            preds = oracle.predict(X, y, splits, ks)
            for (_, te), pr in zip(splits, preds):
                oracle.scores(y[te], pr)
            row["host_oracle_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            pred, _ = consumers.knn_cross_validate(X, y, splits, ks)
            row["predictions_equal"] = bool(np.array_equal(pred.cpu().numpy(), np.concatenate(preds)))
            row["speedup"] = round(row["host_oracle_ms"] / wall, 1)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()

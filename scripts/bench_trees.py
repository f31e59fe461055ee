"""Time b200aa_trees_classify (kernel 8, consumers.tree_classify_batch) on seeded models shaped as the library trains them:
RandomForestClassifier(100), ExtraTreesClassifier(100), GradientBoostingClassifier(100) with 4 classes, and
RandomForestClassifier(500) (the largest n_estimators extract_features_and_train tries), all on 4 000 x 136 rows, for
3 600, 36 000 and 600 000 query rows (an hour at 1 s and 0.1 s steps, and a folder's worth).  The device column is CUDA
events around tree_classify_batch after a warm-up: the kernel, the refused-row check and, for boosting, the host link step
(the call returns once its results are ready).  The host column is batched scikit-learn predict + predict_proba on this
machine's CPU (n_jobs=None, as the library trains).  The "estimator" column is the host wall clock of
tree_classify_batch given the scikit-learn estimator itself, as classify_vectors receives it: flattening, upload, the
call and the model's release, mean of --reps calls.  Every run checks that both give the same ids and probabilities; above
--host-max rows the host runs on a seeded subset of that many rows, compared with the same rows of the device result.

    python scripts/bench_trees.py [--reps 5] [--host-max 36000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from sklearn.ensemble import ExtraTreesClassifier, GradientBoostingClassifier, RandomForestClassifier

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pyaudioanalysis_b200 import consumers  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def data(rng, n, centres):
    y = rng.integers(0, 4, size=n)
    return rng.normal(size=(n, centres.shape[1])) + centres[y], y


def time_device(model, q, reps):
    consumers.tree_classify_batch(model, q)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        ids, P = consumers.tree_classify_batch(model, q)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, ids, P


def time_estimator(est, q, reps):
    """tree_classify_batch on the plain estimator: a TreeEnsembleModel is built and released in every call."""
    consumers.tree_classify_batch(est, q)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        consumers.tree_classify_batch(est, q)
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-max", type=int, default=36000)
    args = ap.parse_args()
    print("card:", card())
    rng = np.random.default_rng(0)
    centres = rng.normal(size=(4, 136)) * 0.4
    X, y = data(rng, 4000, centres)
    specs = [("RandomForestClassifier(100)", RandomForestClassifier(100, random_state=0)),
             ("ExtraTreesClassifier(100)", ExtraTreesClassifier(100, random_state=0)),
             ("GradientBoostingClassifier(100)", GradientBoostingClassifier(n_estimators=100, random_state=0)),
             ("RandomForestClassifier(500)", RandomForestClassifier(500, random_state=0))]
    for name, est in specs:
        t0 = time.perf_counter()
        est.fit(X, y)
        fit_s = time.perf_counter() - t0
        trees = [e.tree_ for e in np.ravel(est.estimators_)]
        model = consumers.TreeEnsembleModel(est)
        info = {"model": name, "trees": len(trees), "nodes": int(sum(t.node_count for t in trees)),
                "max_depth": int(max(t.max_depth for t in trees)), "fit_s": round(fit_s, 1)}
        print(json.dumps(info))
        for n in (3600, 36000, 600000):
            Q = data(rng, n, centres)[0].astype(np.float32)
            q = torch.from_numpy(Q).cuda()
            ms, ids, P = time_device(model, q, args.reps)
            est_ms = time_estimator(est, q, args.reps)
            ids, P = model.classes[ids.cpu().numpy()], P.cpu().numpy()
            rows = np.arange(n) if n <= args.host_max else np.sort(rng.choice(n, args.host_max, replace=False))
            t0 = time.perf_counter()
            ref_ids, ref_P = est.predict(Q[rows]), est.predict_proba(Q[rows])
            host_ms = (time.perf_counter() - t0) * 1e3
            equal = bool(np.array_equal(ids[rows], ref_ids) and np.array_equal(P[rows], ref_P))
            row = {"model": name, "n": n, "device_ms": round(ms, 3), "estimator_ms": round(est_ms, 3), "host_rows": int(rows.size),
                   "host_sklearn_ms": round(host_ms, 1), "equal": equal}
            print(json.dumps(row))
            if not equal:
                sys.exit("device and host results differ")


if __name__ == "__main__":
    main()

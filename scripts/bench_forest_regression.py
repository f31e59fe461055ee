"""Time kernel 13's regression builder against scikit-learn on one host core, on rows free of ties and rows heavy with
ties:

    python scripts/bench_forest_regression.py [--n-exp 10]

1. RandomForestRegressor(n_estimators=T).fit on 1 000 x 136 rows, T = 100 and 500: GPU (forest_regressor_fit) against
   scikit-learn, each pair checked equal tree for tree;
2. evaluate_regression("randomforest", [5, 10, 25, 50, 100]) at n = 1 000 with --n-exp experiments: GPU against the
   reference's loop restated with scikit-learn (the same permutations, fits and per-row predicts), predictions compared.

Prints one JSON line per case with the card's name and power limit, read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def rows(kind, n=1000, F=136, seed=0):
    r = np.random.RandomState(seed)
    X = r.randn(n, F)
    if kind == "ties":
        X = np.round(X, 0)
        return X, r.randint(1, 6, n).astype(np.float64)
    return X, X[:, 0] + 0.5 * r.randn(n)


def reference_loop(X, y, n_exp, params):
    """evaluate_regression's randomforest loop with scikit-learn: (test predictions, training predictions) in order."""
    from sklearn.ensemble import RandomForestRegressor
    from sklearn.preprocessing import StandardScaler
    Xn = StandardScaler().fit_transform(X)
    n = y.shape[0]
    n_train = int(round(0.9 * n))
    pte, ptr = [], []
    for C in params:
        for _ in range(n_exp):
            perm = np.random.permutation(range(n))
            rf = RandomForestRegressor(n_estimators=C).fit(Xn[perm[:n_train]], y[perm[:n_train]])
            ptr.append(rf.predict(Xn[perm[:n_train]]))
            pte.append(np.array([rf.predict(Xn[i].reshape(1, -1))[0] for i in perm[n_train:]]))
    return np.concatenate(pte), np.concatenate(ptr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-exp", type=int, default=10)
    a = ap.parse_args()
    import torch
    from sklearn.ensemble import RandomForestRegressor
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.consumers import forest_regressor_fit, forest_regression_cross_validate
    from tests import forest_regression_cases as RC
    name = card()
    forest_regressor_fit(*rows("free", 50, 5), 2)         # load the library and warm the context
    for kind in ("free", "ties"):
        X, y = rows(kind)
        for T in (100, 500):
            np.random.seed(1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = forest_regressor_fit(X, y, T)
            torch.cuda.synchronize()
            t_gpu = time.perf_counter() - t0
            np.random.seed(1)
            t0 = time.perf_counter()
            ref = RandomForestRegressor(n_estimators=T).fit(X, y)
            t_cpu = time.perf_counter() - t0
            RC.compare(got, ref)
            print(json.dumps({"case": "fit", "rows": kind, "n": 1000, "F": 136, "trees": T, "gpu_s": round(t_gpu, 3),
                              "cpu_s": round(t_cpu, 3), "ratio": round(t_cpu / t_gpu, 2), "equal": True, "card": name}),
                  flush=True)
        params = [5, 10, 25, 50, 100]
        np.random.seed(2)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        splits, seeds = at.draw_regression_problems(X.shape[0], params, a.n_exp)
        pte, ptr = forest_regression_cross_validate(X, y, splits, seeds, [C for C in params for _ in range(a.n_exp)])
        pte, ptr = pte.cpu().numpy(), ptr.cpu().numpy()
        t_gpu = time.perf_counter() - t0
        np.random.seed(2)
        t0 = time.perf_counter()
        rte, rtr = reference_loop(X, y, a.n_exp, params)
        t_cpu = time.perf_counter() - t0
        equal = bool(np.array_equal(pte.view(np.uint64), rte.view(np.uint64)) and np.array_equal(ptr.view(np.uint64), rtr.view(np.uint64)))
        print(json.dumps({"case": "evaluate_regression", "rows": kind, "n": 1000, "F": 136, "n_exp": a.n_exp,
                          "params": params, "gpu_s": round(t_gpu, 3), "cpu_s": round(t_cpu, 3),
                          "ratio": round(t_cpu / t_gpu, 2), "equal": equal, "card": name}), flush=True)


if __name__ == "__main__":
    main()

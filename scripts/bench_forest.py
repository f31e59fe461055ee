"""Time forest training on the GPU (kernel 13, consumers.forest_fit) against scikit-learn's fit on this host's CPU, one
core as the library runs it (n_jobs=None), on seeded 4-class rows of 136 features (the library's mid-term feature
count): RandomForestClassifier and ExtraTreesClassifier of 100 and 500 trees on 1 000 and 10 000 rows.  The GPU column
is the host wall clock of forest_fit (host draws, upload, kernel, nodes back, estimator assembly) after one warm-up call,
mean of --reps calls; the CPU column is one scikit-learn fit.  Every timed pair is fit from the same NumPy seed and the
two forests are checked equal tree for tree.

--evaluate KIND times instead the whole model selection of evaluate_classifier(KIND, [10, 25, 50, 100, 200, 500]) on
1 000 seeded rows (51 experiments, 306 forests, 45 135 trees): the GPU column is audioTrainTest.evaluate_classifier here
(one batched forest_cross_validate), the CPU column the reference's loop restated with scikit-learn (per problem
train_test_split, StandardScaler, fit, predict), from the same seed; the predictions of every problem are compared.
Prints one JSON line per case with the card's name and power limit, read in the same call.

    python scripts/bench_forest.py [--reps 3]
    python scripts/bench_forest.py --evaluate randomforest|extratrees
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pyaudioanalysis_b200.consumers import forest_fit  # noqa: E402
from tests import forest_cases as FC  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--evaluate", choices=("randomforest", "extratrees"))
    a = ap.parse_args()
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    if not torch.cuda.is_available():
        raise SystemExit("bench_forest needs a CUDA device")
    name = card()
    if a.evaluate:
        return evaluate(a.evaluate, name)
    rng = np.random.default_rng(0)
    centres = rng.normal(scale=0.7, size=(4, 136))
    for n in (1000, 10000):
        y = rng.integers(0, 4, size=n)
        X = rng.normal(size=(n, 136)) + centres[y]
        for kind, cls in (("randomforest", RandomForestClassifier), ("extratrees", ExtraTreesClassifier)):
            for T in (100, 500):
                np.random.seed(1)
                forest_fit(X, y, T, kind)                       # warm-up
                t0 = time.perf_counter()
                for _ in range(a.reps):
                    np.random.seed(1)
                    got = forest_fit(X, y, T, kind)
                gpu = (time.perf_counter() - t0) / a.reps
                np.random.seed(1)
                t0 = time.perf_counter()
                ref = cls(n_estimators=T).fit(X, y)
                cpu = time.perf_counter() - t0
                FC.compare(got, ref)
                print(json.dumps({"kind": kind, "rows": n, "features": 136, "trees": T, "gpu_s": round(gpu, 4),
                                  "cpu_s": round(cpu, 4), "speedup": round(cpu / gpu, 2), "equal": True,
                                  "card": name}), flush=True)


def evaluate(kind, name):
    import contextlib
    import io
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    from sklearn.preprocessing import StandardScaler
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.consumers import forest_cross_validate
    from tests.knn_cv_oracle import seeded_features
    cls = RandomForestClassifier if kind == "randomforest" else ExtraTreesClassifier
    feats = seeded_features(60, (250, 250, 250, 250), 136)
    X, y = at.features_to_matrix(feats)
    params = [10, 25, 50, 100, 200, 500]
    n_exp = int(50000 / X.shape[0]) + 1
    np.random.seed(2)
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        at.evaluate_classifier(feats, ["a", "b", "c", "d"], kind, params, 1, n_exp=n_exp)
    gpu = time.perf_counter() - t0
    # the same draws again, this time keeping the predictions
    np.random.seed(2)
    splits, seeds = at.draw_forest_problems(X, params, n_exp, 0.9, kind)
    pred, _ = forest_cross_validate(X, y, splits, seeds, [p for p in params for _ in range(n_exp)], kind, n_classes=4)
    pred = pred.cpu().numpy()
    np.random.seed(2)
    off, equal = 0, True
    t0 = time.perf_counter()
    for C in params:
        for _ in range(n_exp):
            perm = np.random.permutation(X.shape[0])
            n_test = len(splits[0][1])
            te, tr = perm[:n_test], perm[n_test:]
            sc = StandardScaler().fit(X[tr])
            m = cls(n_estimators=C).fit(sc.transform(X[tr]), y[tr])
            want = m.predict(sc.transform(X[te]))
            equal &= bool(np.array_equal(pred[off:off + n_test], want.astype(int)))
            off += n_test
    cpu = time.perf_counter() - t0
    print(json.dumps({"evaluate_classifier": kind, "rows": X.shape[0], "features": 136, "params": params,
                      "experiments": n_exp, "gpu_s": round(gpu, 3), "cpu_s": round(cpu, 3),
                      "speedup": round(cpu / gpu, 2), "equal": equal, "card": name}), flush=True)


if __name__ == "__main__":
    main()

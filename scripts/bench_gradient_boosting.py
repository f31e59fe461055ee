"""Time kernel 13's gradient boosting against scikit-learn on one host core:

    python scripts/bench_gradient_boosting.py [--n-exp 2]

1. GradientBoostingClassifier(n_estimators=100).fit on a seeded 1 000 x 136, 4-class problem: GPU (train_gradient_boosting)
   against scikit-learn, checked equal tree for tree.  The GPU fit's time is split per stage into the stage call (device
   work, synchronised), the host gradient, and the rest (gradient upload, raw predictions down, train score, tree
   assembly), since every stage makes one host round trip.
2. evaluate_classifier("gradientboosting") over the reference's parameter list [10, 25, 50, 100, 200, 500] at n = 1 000
   with --n-exp experiments (the reference would take int(50000 / n) + 1 = 51): GPU only; scikit-learn's time is given
   as the single fits' time times the stage count, not measured.

Prints one JSON line per case with the card's name and power limit, read in the same call.  Fails without a GPU.
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def problem(n=1000, F=136, C=4, seed=0):
    r = np.random.RandomState(seed)
    X = r.randn(n, F)
    return X, np.argmax(X[:, :C] + r.randn(n, C), 1)


def timed_fit(X, y, T):
    """boosting_fit timed: (model, total seconds, {part: seconds}): the stage calls (synchronised), the host gradient,
    and the rest (gradient upload, raw download, train score, tree assembly)."""
    import torch
    from pyaudioanalysis_b200 import consumers
    from pyaudioanalysis_b200 import boosting as BO
    parts = {"stage_call": 0.0, "host_gradient": 0.0}
    real_lib, real_neg = consumers.lib, BO.neg_gradient

    class Timed:
        def __getattr__(self, name):
            f = getattr(real_lib(), name)
            if name != "b200aa_boosting_stage":
                return f

            def g(*a):
                torch.cuda.synchronize()
                t = time.perf_counter()
                rc = f(*a)
                torch.cuda.synchronize()
                parts["stage_call"] += time.perf_counter() - t
                return rc
            return g

    def neg(*a):
        t = time.perf_counter()
        out = real_neg(*a)
        parts["host_gradient"] += time.perf_counter() - t
        return out
    consumers.lib, BO.neg_gradient = (lambda: Timed()), neg
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m = consumers.boosting_fit(X, y, T)
        total = time.perf_counter() - t0
    finally:
        consumers.lib, BO.neg_gradient = real_lib, real_neg
    parts["copies_score_and_rest"] = total - parts["stage_call"] - parts["host_gradient"]
    return m, total, parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-exp", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark times the GPU trainer")
    from sklearn.ensemble import GradientBoostingClassifier
    from pyaudioanalysis_b200 import audioTrainTest as at
    from tests import boosting_cases as BC
    gpu = card()
    X, y = problem()
    np.random.seed(1)
    timed_fit(X[:100], y[:100], 2)                              # warm-up: library load, module, allocator
    np.random.seed(1)
    m, t_gpu, parts = timed_fit(X, y, 100)
    np.random.seed(1)
    t0 = time.perf_counter()
    ref = GradientBoostingClassifier(n_estimators=100).fit(X, y)
    t_cpu = time.perf_counter() - t0
    BC.compare(m, ref, X[:50])
    print(json.dumps({"case": "fit_1000x136_4class_100_stages", "card": gpu, "gpu_s": round(t_gpu, 3),
                      "sklearn_s": round(t_cpu, 3), "speedup": round(t_cpu / t_gpu, 1),
                      "per_stage_ms": {k: round(1e3 * v / 100, 3) for k, v in parts.items()}, "equal": True}))
    params = [10, 25, 50, 100, 200, 500]
    feats = [X[y == c] for c in range(4)]
    np.random.seed(2)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        best = at.evaluate_classifier(feats, ["a", "b", "c", "d"], "gradientboosting", params, 1, n_exp=a.n_exp)
    torch.cuda.synchronize()
    t_sel = time.perf_counter() - t0
    print(json.dumps({"case": "evaluate_classifier_gradientboosting_n1000", "card": gpu, "n_exp": a.n_exp,
                      "params": params, "gpu_s": round(t_sel, 3), "best": int(best),
                      "sklearn_s_estimate_from_fit_rate": round(t_cpu / 100 * sum(params) * a.n_exp * 0.9, 1),
                      "sklearn_note": "estimate: the 100-stage fit's time per stage x every problem's stages x 0.9 "
                                      "(training rows), not measured"}))


if __name__ == "__main__":
    main()

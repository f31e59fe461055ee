"""Golden runs of the UNMODIFIED reference's evaluate_regression with its random forest (run where the reference tree
exists):

    python -m oracle.make_golden_forest_regression_cv

The reference's evaluate_regression, train_random_forest_regression and regression_wrapper (audioTrainTest.py) are
executed from its source text with the imported scikit-learn, as in make_golden_forest_cv.py.  Writes
tests/golden/forest_regression_cv.npz; for case <c> (listed in `cases`): <c>_X and <c>_y (features and labels),
<c>_params, <c>_n_exp, <c>_seed (np.random.seed before the call), <c>_stdout (the complete printed text) and <c>_ret
(the return value: best parameter, its MSE and its baseline MSE).

Cases: (a) the default parameter list [5, 10, 25, 50, 100] on 60 rows; (b) other parameters on continuous targets with
an offset; (c) tied integer labels; (d) a tiny n of 5 (one test row).
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import sklearn.ensemble
from sklearn.preprocessing import StandardScaler

from oracle.make_golden_knn import REF, _exec_between

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "forest_regression_cv.npz")


def _reference():
    src = os.path.join(REF, "audioTrainTest.py")
    env = {"np": np, "StandardScaler": StandardScaler, "sklearn": types.SimpleNamespace(ensemble=sklearn.ensemble)}
    for start, stop in (("def regression_wrapper", "def train_knn"),
                        ("def train_random_forest_regression", "def extract_features_and_train"),
                        ("def evaluate_regression", "def print_confusion_matrix")):
        _exec_between(src, start, stop, env)
    return env


def main():
    sys.path.insert(0, ROOT)
    g, cases = {}, []

    def run(name, X, y, params, n_exp, seed):
        env = _reference()
        np.random.seed(seed)
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            ret = env["evaluate_regression"](X, y, n_exp, "randomforest", params)
        g.update({name + "_X": X, name + "_y": y, name + "_params": np.asarray(params, dtype=np.int64),
                  name + "_n_exp": np.int64(n_exp), name + "_seed": np.int64(seed),
                  name + "_stdout": np.asarray(out.getvalue()), name + "_ret": np.asarray(ret, dtype=np.float64)})
        cases.append(name)
        print(name, "returns", ret)

    r = np.random.RandomState(61)
    X = r.randn(60, 10)
    run("a", X, X[:, 0] + 0.5 * r.randn(60), [5, 10, 25, 50, 100], 2, seed=1)
    X = r.randn(80, 7)
    run("b", X, 1000.0 + X[:, 1] * 3 + r.randn(80) * 0.01, [3, 7], 3, seed=2)
    X = np.round(r.randn(70, 6), 1)
    run("c", X, r.randint(1, 6, 70).astype(np.float64), [4, 9], 3, seed=3)
    X = r.randn(5, 3)
    run("d", X, r.randn(5), [2, 6], 4, seed=4)
    g["cases"] = np.asarray(cases)
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()

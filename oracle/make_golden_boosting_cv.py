"""Golden runs of the UNMODIFIED reference's model selection for gradient boosting (run where the reference tree exists):

    python -m oracle.make_golden_boosting_cv

The reference's evaluate_classifier, group_split, train_gradient_boosting, classifier_wrapper and
print_confusion_matrix (audioTrainTest.py) are executed from its source text with the imported scikit-learn, as in
make_golden_knn_cv.py (audioTrainTest cannot be imported here: imblearn is not installed).  Writes
tests/golden/boosting_cv.npz; for case <c> (listed in `cases`): <c>_gen = (seed, F) and <c>_sizes, the rows being
tests.knn_cv_oracle.seeded_features(seed, sizes, F), with <c>_X_sum; <c>_classifier, <c>_class_names, <c>_params,
<c>_mode, <c>_n_exp, <c>_train_percentage, <c>_ids (list_of_ids, or empty); <c>_seed (np.random.seed before the call);
<c>_stdout (the complete printed text) and <c>_ret (the return value).

Cases: (a) 3 classes, params [2, 5, 10], mode 1; (b) 2 classes (the binomial loss), mode 0, train_percentage 0.7; (c)
group ids, mode 1; (d) a middle class of one row and train_percentage 0.7, so some training sets miss it and their problem
turns binary.
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import sklearn.ensemble
import sklearn.metrics
from sklearn.model_selection import GroupShuffleSplit, train_test_split
from sklearn.preprocessing import StandardScaler

from oracle.make_golden_knn import REF, _exec_between

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "boosting_cv.npz")


def _reference():
    src = os.path.join(REF, "audioTrainTest.py")
    env = {"np": np, "train_test_split": train_test_split, "StandardScaler": StandardScaler,
           "GroupShuffleSplit": GroupShuffleSplit,
           "sklearn": types.SimpleNamespace(metrics=sklearn.metrics, ensemble=sklearn.ensemble)}
    for start, stop in (("def classifier_wrapper", "def regression_wrapper"),
                        ("def train_gradient_boosting", "def train_extra_trees"),
                        ("def group_split", "def evaluate_regression"),
                        ("def print_confusion_matrix", "def pca_wrapper")):
        _exec_between(src, start, stop, env)
    return env


def main():
    sys.path.insert(0, ROOT)
    from tests.knn_cv_oracle import seeded_features
    g, cases = {}, []

    def run(name, classifier, gen, sizes, class_names, params, mode, n_exp, tp=0.90, ids=None, seed=0):
        features = seeded_features(gen[0], sizes, gen[1])
        env = _reference()
        np.random.seed(seed)
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            ret = env["evaluate_classifier"](features, class_names, classifier, params, mode, list_of_ids=ids,
                                             n_exp=n_exp, train_percentage=tp)
        g.update({name + "_gen": np.asarray(gen, dtype=np.int64), name + "_sizes": np.asarray(sizes, dtype=np.int64),
                  name + "_X_sum": np.float64(np.vstack(features).sum()), name + "_classifier": np.asarray(classifier),
                  name + "_class_names": np.asarray(class_names), name + "_params": np.asarray(params),
                  name + "_mode": np.int64(mode), name + "_n_exp": np.int64(n_exp), name + "_train_percentage": np.float64(tp),
                  name + "_ids": np.asarray(ids if ids else [], dtype=np.int64), name + "_seed": np.int64(seed),
                  name + "_stdout": np.asarray(out.getvalue()), name + "_ret": np.int64(ret)})
        cases.append(name)
        print(name, classifier, "returns", ret)

    run("a", "gradientboosting", (61, 10), (30, 25, 20), ["a", "b", "c"], [2, 5, 10], 1, 3, seed=1)
    run("b", "gradientboosting", (62, 8), (30, 28), ["speech", "music"], [3, 6], 0, 3, tp=0.7, seed=2)
    sizes = (20, 20, 20)
    run("c", "gradientboosting", (63, 6), sizes, ["x", "y", "z"], [2, 4], 1, 3, ids=[i // 5 for i in range(sum(sizes))],
        seed=3)
    run("d", "gradientboosting", (64, 6), (25, 1, 20), ["a", "rare", "c"], [2, 5], 1, 6, tp=0.7, seed=4)
    g["cases"] = np.asarray(cases)
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()

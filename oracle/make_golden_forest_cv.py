"""Golden runs of the UNMODIFIED reference's model selection for its two forests (run where the reference tree exists):

    python -m oracle.make_golden_forest_cv

The reference's evaluate_classifier, group_split, train_random_forest, train_extra_trees, classifier_wrapper and
print_confusion_matrix (audioTrainTest.py) are executed from its source text with the imported scikit-learn, as in
make_golden_knn_cv.py (audioTrainTest cannot be imported here: imblearn is not installed).  Writes
tests/golden/forest_cv.npz; for case <c> (listed in `cases`): <c>_gen = (seed, F) and <c>_sizes, the rows being
tests.knn_cv_oracle.seeded_features(seed, sizes, F), with <c>_X_sum; <c>_classifier, <c>_class_names, <c>_params,
<c>_mode, <c>_n_exp, <c>_train_percentage, <c>_ids (list_of_ids, or empty); <c>_seed (np.random.seed before the call);
<c>_stdout (the complete printed text) and <c>_ret (the return value).

Cases: (a) random forest, mode 1; (b) extra trees, mode 0, train_percentage 0.7; (c) random forest with group ids,
mode 1; (d) extra trees with a middle class of 3 rows, so some training sets miss it.
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
OUT = os.path.join(ROOT, "tests", "golden", "forest_cv.npz")


def _reference():
    src = os.path.join(REF, "audioTrainTest.py")
    env = {"np": np, "train_test_split": train_test_split, "StandardScaler": StandardScaler,
           "GroupShuffleSplit": GroupShuffleSplit,
           "sklearn": types.SimpleNamespace(metrics=sklearn.metrics, ensemble=sklearn.ensemble)}
    for start, stop in (("def classifier_wrapper", "def regression_wrapper"),
                        ("def train_random_forest", "def train_gradient_boosting"),
                        ("def train_extra_trees", "def train_svm_regression"),
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

    run("a", "randomforest", (51, 12), (40, 35, 30), ["a", "b", "c"], [10, 25, 50], 1, 4, seed=1)
    run("b", "extratrees", (52, 9), (50, 45), ["speech", "music"], [10, 25, 50], 0, 5, tp=0.7, seed=2)
    sizes = (30, 30, 30)
    run("c", "randomforest", (53, 8), sizes, ["x", "y", "z"], [10, 20], 1, 4, ids=[i // 5 for i in range(sum(sizes))],
        seed=3)
    run("d", "extratrees", (54, 6), (30, 3, 25), ["a", "rare", "c"], [10, 25], 1, 6, seed=4)
    g["cases"] = np.asarray(cases)
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()

"""Golden runs of the UNMODIFIED reference's kNN model selection (run where the reference tree exists):

    python -m oracle.make_golden_knn_cv

The reference's evaluate_classifier, group_split, features_to_matrix, print_confusion_matrix, Knn, train_knn and
classifier_wrapper (audioTrainTest.py) are executed from its source text, as in make_golden_knn.py (audioTrainTest cannot
be imported here: imblearn is not installed), with the imported scikit-learn.  Its confusion_matrix is wrapped to record
each experiment's y_test / y_pred, its StandardScaler to record the first fits, and classifier_wrapper to reject a run
with an exact tie at a test row's k-th place between different labels (the reference's unstable argsort decides there;
make_golden_knn.py's rule): the seed then moves on.  Writes tests/golden/knn_cv.npz; for case <c> (listed in `cases`):

* <c>_X [n, F] and <c>_sizes [C] (the class matrices stacked in order), or for a seeded case <c>_gen = (seed, F) with
  <c>_sizes and <c>_X_sum, the rows being tests.knn_cv_oracle.seeded_features(seed, sizes, F);
* <c>_class_names, <c>_params, <c>_mode, <c>_n_exp (as passed), <c>_train_percentage, <c>_ids (list_of_ids, or empty);
* <c>_seed: np.random.seed before the call;
* <c>_stdout: the complete printed text; <c>_ret: the return value;
* <c>_y_test / <c>_y_pred: every experiment's rows in order (int8), <c>_exp_len: rows per experiment;
* <c>_mean / <c>_scale [4, F]: the scaler of the first four experiments.

Cases: (a) the reference's pytests/test_data/3_class through its own multiple_directory_feature_extraction(..., 1.0,
1.0, 0.05, 0.05), mode 1, default n_exp; (b) the same, mode 0, n_exp 20, train_percentage 0.7; (c) the same with group
ids (file index // 6), n_exp 12; (d) seeded, a middle class of 2 rows, so some splits miss it (fewer classes in the
training rows, classes missing from y_test and y_pred); (e) seeded, 3 000 x 136, n_exp 2.
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import sklearn.metrics
from scipy.spatial import distance
from sklearn.model_selection import GroupShuffleSplit, train_test_split
from sklearn.preprocessing import StandardScaler

from oracle.make_golden_knn import REF, _ambiguous, _exec_between
from oracle.ref_import import REFERENCE_ROOT, load_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "knn_cv.npz")
THREE_CLASS = os.path.join(REFERENCE_ROOT, "pytests", "test_data", "3_class")


class Ambiguous(Exception):
    pass


def _reference(record):
    src = os.path.join(REF, "audioTrainTest.py")

    class RecordingScaler(StandardScaler):
        def fit(self, X, y=None, sample_weight=None):
            out = super().fit(X, y, sample_weight)
            record["scalers"].append((self.mean_.copy(), self.scale_.copy()))
            return out

    def confusion_matrix(y_true, y_pred, *a, **kw):
        record["cm"].append((np.asarray(y_true).copy(), np.asarray(y_pred).copy()))
        return sklearn.metrics.confusion_matrix(y_true, y_pred, *a, **kw)

    env = {"np": np, "distance": distance, "train_test_split": train_test_split, "StandardScaler": RecordingScaler,
           "GroupShuffleSplit": GroupShuffleSplit,
           "sklearn": types.SimpleNamespace(metrics=types.SimpleNamespace(confusion_matrix=confusion_matrix,
                                                                          f1_score=sklearn.metrics.f1_score))}
    for start, stop in (("class Knn", "def classifier_wrapper"), ("def classifier_wrapper", "def regression_wrapper"),
                        ("def train_knn", "def train_svm"), ("def group_split", "def evaluate_regression"),
                        ("def print_confusion_matrix", "def pca_wrapper")):
        _exec_between(src, start, stop, env)
    wrapper = env["classifier_wrapper"]

    def checked_wrapper(classifier, classifier_type, test_sample):
        d = distance.cdist(classifier.features, test_sample.reshape(1, -1), "euclidean")[:, 0]
        if _ambiguous(d, classifier.labels, classifier.neighbors):
            raise Ambiguous()
        return wrapper(classifier, classifier_type, test_sample)

    env["classifier_wrapper"] = checked_wrapper
    return env


def _three_class():
    _, M, _ = load_reference()
    dirs = [os.path.join(THREE_CLASS, d) for d in sorted(os.listdir(THREE_CLASS))]
    with contextlib.redirect_stdout(io.StringIO()):
        features, class_names, files = M.multiple_directory_feature_extraction(dirs, 1.0, 1.0, 0.05, 0.05)
    features = [np.asarray(f, dtype=np.float64) for f in features]
    assert all(np.isfinite(f).all() for f in features)
    return features, list(class_names), [f for fl in files for f in fl]


def main():
    sys.path.insert(0, ROOT)
    from tests.knn_cv_oracle import seeded_features
    g, cases = {}, []
    params = np.array([1, 3, 5, 7, 9, 11, 13, 15])

    def run(name, features, class_names, mode, n_exp=-1, tp=0.90, ids=None, seed=0, gen=None):
        while True:
            record = {"cm": [], "scalers": []}
            env = _reference(record)
            np.random.seed(seed)
            out = io.StringIO()
            try:
                with contextlib.redirect_stdout(out):
                    ret = env["evaluate_classifier"](features, class_names, "knn", params, mode, list_of_ids=ids,
                                                     n_exp=n_exp, train_percentage=tp)
                break
            except Ambiguous:
                print(name, "seed", seed, "has an ambiguous k-th place; next seed")
                seed += 1
        X = np.vstack(features)
        if gen is None:
            g[name + "_X"] = X
        else:
            g[name + "_gen"] = np.asarray(gen, dtype=np.int64)
            g[name + "_X_sum"] = np.float64(X.sum())
        g.update({name + "_sizes": np.array([len(f) for f in features], dtype=np.int64),
                  name + "_class_names": np.asarray(class_names), name + "_params": params,
                  name + "_mode": np.int64(mode), name + "_n_exp": np.int64(n_exp), name + "_train_percentage": np.float64(tp),
                  name + "_ids": np.asarray(ids if ids else [], dtype=np.int64), name + "_seed": np.int64(seed),
                  name + "_stdout": np.asarray(out.getvalue()), name + "_ret": np.int64(ret),
                  name + "_y_test": np.concatenate([t for t, _ in record["cm"]]).astype(np.int8),
                  name + "_y_pred": np.concatenate([p for _, p in record["cm"]]).astype(np.int8),
                  name + "_exp_len": np.array([t.size for t, _ in record["cm"]], dtype=np.int64),
                  name + "_mean": np.stack([m for m, _ in record["scalers"][:4]]),
                  name + "_scale": np.stack([s for _, s in record["scalers"][:4]])})
        cases.append(name)
        print(name, X.shape, "experiments", len(record["cm"]), "seed", seed, "returns", ret)

    features, class_names, files = _three_class()
    run("a", features, class_names, 1, seed=1)
    run("b", features, class_names, 0, n_exp=20, tp=0.7, seed=2)
    run("c", features, class_names, 1, n_exp=12, ids=[i // 6 for i in range(len(files))], seed=3)
    run("d", seeded_features(41, (30, 2, 25), 6), ["a", "rare", "c"], 1, n_exp=30, seed=4)
    run("e", seeded_features(42, (1000, 1000, 1000), 136), ["x", "y", "z"], 1, n_exp=2, seed=5, gen=(42, 136))
    g["cases"] = np.asarray(cases)
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()

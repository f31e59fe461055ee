"""The kNN cross-validation oracle: the reference's evaluate_classifier loop (audioTrainTest.py:631-699) restated with
scikit-learn's own train_test_split / GroupShuffleSplit, StandardScaler and metrics, and the stable-sort Knn oracle of
tests/knn_oracle.py.  It equals the reference wherever the reference's (unstable) argsort gives a defined result."""
import numpy as np
import sklearn.metrics
from sklearn.model_selection import GroupShuffleSplit, train_test_split
from sklearn.preprocessing import StandardScaler

from tests.knn_oracle import knn_oracle


def seeded_features(seed, sizes, n_feats, shift=0.35):
    """Class matrices of standard normal rows, class i shifted by i * shift (numpy's Generator streams are stable)."""
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((m, n_feats)) + i * shift for i, m in enumerate(sizes)]


def reference_splits(n, n_params, n_exp, train_percentage=0.90, list_of_ids=None):
    """(train, test) row indices per (param, experiment), params outer, drawn by scikit-learn exactly as the reference
    draws them from NumPy's global RNG."""
    rows = np.arange(n)
    if list_of_ids:
        gss = GroupShuffleSplit(n_splits=n_exp, train_size=.8)
        return [(tr, te) for tr, te in gss.split(rows, rows, list_of_ids)] * n_params
    return [tuple(train_test_split(rows, test_size=1 - train_percentage)) for _ in range(n_params * n_exp)]


def predict(X, y, splits, ks):
    """Knn(X_train, y_train, k).classify of every test row of every split, StandardScaler-standardised (a list of arrays)."""
    out = []
    for (tr, te), k in zip(splits, ks):
        sc = StandardScaler().fit(X[tr])
        ids, _ = knn_oracle(sc.transform(X[tr]), y[tr], int(k), sc.transform(X[te]))
        out.append(ids)
    return out


def counts(y, splits, preds, n_classes):
    """[P, C, C] counts of (y_test, y_pred) per problem."""
    c = np.zeros((len(splits), n_classes, n_classes), dtype=np.int64)
    for p, ((_, te), pr) in enumerate(zip(splits, preds)):
        np.add.at(c[p], (y[te].astype(np.int64), np.asarray(pr, dtype=np.int64)), 1)
    return c


def scores(y_test, y_pred):
    """The reference's per-experiment confusion_matrix and macro f1_score (:682-683)."""
    return (sklearn.metrics.confusion_matrix(y_test, y_pred),
            sklearn.metrics.f1_score(y_test, y_pred, average='macro'))


def golden_features(g, c):
    sizes = g[c + "_sizes"]
    if c + "_gen" in g.files:
        seed, F = (int(v) for v in g[c + "_gen"])
        feats = seeded_features(seed, tuple(int(s) for s in sizes), F)
        assert np.vstack(feats).sum() == g[c + "_X_sum"], c
        return feats
    return np.split(g[c + "_X"], np.cumsum(sizes)[:-1])


def golden_args(g, c):
    ids = g[c + "_ids"].tolist() or None
    return (list(g[c + "_class_names"]), g[c + "_params"], int(g[c + "_mode"]), ids, int(g[c + "_n_exp"]),
            float(g[c + "_train_percentage"]))

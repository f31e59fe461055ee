"""The stable-sort kNN oracle: scipy's cdist, np.argsort(kind="stable") and the vote of the reference's Knn.classify
(audioTrainTest.py:33-49).  It equals Knn.classify wherever the reference's own (unstable) argsort gives a defined result,
and breaks an exact tie at the k-th place by the lower training index, as b200aa_knn_classify does."""
import numpy as np
from scipy.spatial.distance import cdist


def knn_oracle(feats, labels, k, queries, chunk=256):
    """(ids int64 [n], P float64 [n, C]) for the rows of `queries` [n, F] (float64)."""
    feats = np.asarray(feats, dtype=np.float64)
    labels = np.asarray(labels)
    queries = np.asarray(queries, dtype=np.float64).reshape(-1, feats.shape[1])
    n_classes = np.unique(labels).shape[0]
    ids = np.zeros(queries.shape[0], dtype=np.int64)
    P = np.zeros((queries.shape[0], n_classes))
    for a in range(0, queries.shape[0], chunk):
        d = cdist(queries[a:a + chunk], feats, "euclidean")
        near = labels[np.argsort(d, axis=1, kind="stable")[:, :k]]
        for i in range(n_classes):
            P[a:a + chunk, i] = (near == i).sum(axis=1) / float(k)
    ids[:] = np.argmax(P, axis=1)
    return ids, P


def slots_of(labels):
    """The class each training row votes for: its label when that is an integer in [0, C), else -1."""
    labels = np.asarray(labels, dtype=np.float64)
    C = np.unique(labels).shape[0]
    ok = (labels == np.floor(labels)) & (labels >= 0) & (labels < C)
    return np.where(ok, labels, -1).astype(np.int64), C

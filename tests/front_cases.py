"""Shared inputs and oracles of kernel 11's tests (test_front_cpu.py, test_gpu_front.py): the value bank of the scaler,
the row counts around NumPy's pairwise leaves, and scikit-learn / scipy / NumPy statements of the three steps."""
import warnings

import numpy as np
from scipy.spatial import distance
from sklearn.preprocessing import StandardScaler

# row counts: one row, around the 8-wide leaf, the 128-term leaf, and NumPy's 8192-element buffer
NS = (1, 7, 8, 9, 127, 128, 129, 8191, 8193)


def value_bank(rng, n, D):
    """A C-contiguous float64 [n, D] of adversarial columns: +-0, subnormals, scales from 1e-300 to 1e300, a constant
    column, columns just either side of the constant-feature test, and seeded normal data."""
    X = rng.normal(size=(n, D))
    pick = [
        lambda: np.where(rng.random(n) < 0.5, 0.0, -0.0),
        lambda: rng.normal(size=n) * 5e-324 * 1e3,
        lambda: rng.normal(size=n) * 1e-300,
        lambda: rng.normal(size=n) * 1e300,
        lambda: np.full(n, rng.normal() * 10.0 ** rng.integers(-20, 20)),
        lambda: 1.0 + rng.integers(-2, 3, n) * 2.0 ** -52,             # a few ulps around 1: near the constant test
        lambda: 1e8 + rng.integers(-1, 2, n) * 2.0 ** -26,
        lambda: 3.0 + rng.normal(size=n) * 1e-9,
        lambda: rng.normal(size=n) * 1e150 + 1e160,
    ]
    for j in range(D):
        if j % 3 != 2:
            X[:, j] = pick[(j * 7 + n) % len(pick)]()
    return X


def with_nans(rng, X, share=0.2, all_nan_col=None):
    """X with NaN in about `share` of the rows of every other column, and one all-NaN column."""
    X = X.copy()
    n, D = X.shape
    for j in range(0, D, 2):
        X[rng.random(n) < share, j] = np.nan
    if all_nan_col is not None and D > all_nan_col:
        X[:, all_nan_col] = np.nan
    return X


def sk_scale(X):
    """(Y, mean_, scale_) of StandardScaler().fit_transform(X), X at the caller's layout."""
    s = StandardScaler()
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        Y = s.fit_transform(X)
    return Y, s.mean_, s.scale_


def column_major(X):
    """The same values as a column-major (F-ordered) array, the transpose of a C-contiguous [D, n] one."""
    return np.ascontiguousarray(X.T).T


def outlier_rule(Xn):
    """audioSegmentation.py:861-865 on the normalised [M, D] matrix: (i_non_outliers, dist_all)."""
    with np.errstate(all="ignore"):
        dist_all = np.sum(distance.squareform(distance.pdist(Xn.T)), axis=0)
        return np.nonzero(dist_all < 1.1 * np.mean(dist_all))[0], dist_all


def pool_loop(st, ratio):
    """:884-906 as the reference writes it: per feature row, the mean then the std of every window of `ratio` frames
    starting at each frame, cut at the end."""
    st = np.asarray(st, dtype=np.float64)
    F, T = st.shape
    red = np.zeros((2 * F, T))
    for f in range(F):
        for i in range(T):
            w = st[f][i:min(i + ratio, T)]
            red[f, i] = np.mean(w)
            red[F + f, i] = np.std(w)
    return red


def pool_bank(rng, F, T):
    """A float32 [F, T] short-term matrix: seeded normal rows at several scales, a constant row, a row of +-0."""
    st = (rng.normal(size=(F, T)) * 10.0 ** rng.integers(-3, 4, (F, 1))).astype(np.float32)
    st[0] = 2.5
    if F > 1:
        st[1] = np.where(rng.random(T) < 0.5, 0.0, -0.0)
    return st

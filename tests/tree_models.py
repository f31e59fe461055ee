"""Seeded scikit-learn tree ensembles and adversarial query banks for the kernel-8 tests (tests/test_trees_cpu.py,
tests/test_gpu_trees.py).  The training data carries a +-1 feature (a split threshold at exactly 0), a feature of
float32 subnormals (thresholds between subnormals) and float32-valued features everywhere else."""
import numpy as np
from sklearn.ensemble import ExtraTreesClassifier, GradientBoostingClassifier, RandomForestClassifier

F = 12


def dataset(n=600, n_classes=4, seed=0, nan=False):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, n_classes, size=n)
    X = rng.normal(size=(n, F)) + 0.6 * y[:, None] * rng.normal(size=F)[None, :]
    X[:, 0] = np.where((y % 2 == 1) ^ (rng.random(n) < 0.2), 1.0, -1.0)                    # threshold exactly 0
    X[:, 1] = (rng.integers(1, 200, size=n) + 40 * (y == 2)) * np.float32(1e-45)             # subnormal thresholds
    X = X.astype(np.float32).astype(np.float64)
    if nan:
        X[rng.random(X.shape) < 0.08] = np.nan
    return X, y


def models():
    """name -> fitted estimator: forests and boosting, binary, 4-class and 40-class, and the model corners of the
    contract."""
    X4, y4 = dataset()
    X2, y2 = dataset(n_classes=2, seed=1)
    Xn, yn = dataset(seed=2, nan=True)
    X40, y40 = dataset(n=1200, n_classes=40, seed=3)
    n = 30
    out = {
        "rf4": RandomForestClassifier(n, random_state=0).fit(X4, y4),
        "et4": ExtraTreesClassifier(n, random_state=1).fit(X4, y4),
        "gb4": GradientBoostingClassifier(n_estimators=n, random_state=2).fit(X4, y4),
        "rf2": RandomForestClassifier(n, random_state=3).fit(X2, y2),
        "et2": ExtraTreesClassifier(n, random_state=4).fit(X2, y2),
        "gb2": GradientBoostingClassifier(n_estimators=n, random_state=5).fit(X2, y2),
        "gb2_zero": GradientBoostingClassifier(n_estimators=n, init="zero", random_state=6).fit(X2, y2),
        "rf_nan": RandomForestClassifier(n, random_state=7).fit(Xn, yn),
        "et_nan": ExtraTreesClassifier(n, random_state=8).fit(Xn, yn),
        "rf1": RandomForestClassifier(1, random_state=9).fit(X4, y4),
        "rf500": RandomForestClassifier(500, max_depth=3, random_state=10).fit(X4, y4),
        "labels_257": RandomForestClassifier(n, random_state=11).fit(X4[:, :], np.array([2, 5, 7, 7])[y4]),
        "labels_str": GradientBoostingClassifier(n_estimators=n, random_state=12).fit(X4, np.array(["a", "bb", "c", "d"])[y4]),
        "labels_str_et": ExtraTreesClassifier(n, random_state=13).fit(X2, np.array(["no", "yes"])[y2]),
        # bootstraps of four rows: many trees see one class only and are a single leaf
        "one_leaf": RandomForestClassifier(40, random_state=14).fit(X4[:4], np.array([0, 0, 0, 1])),
        "stump_leaf": RandomForestClassifier(5, min_samples_split=10 ** 6, random_state=15).fit(X4, y4),
        # two fully grown trees on disjoint views: they disagree, P = [0.5, 0.5] ties
        "tie": ExtraTreesClassifier(2, bootstrap=False, random_state=16).fit(X2, y2),
        # more classes than a warp has lanes: each lane sums and compares several classes.  Three unbootstrapped trees
        # give P in thirds, so maxima tie across lanes; class 35 repeats class 3's rows, so 3 and 35 (one lane) tie too
        "rf40": RandomForestClassifier(n, random_state=17).fit(X40, y40),
        "gb40": GradientBoostingClassifier(n_estimators=4, random_state=18).fit(X40, y40),
        "tie40": ExtraTreesClassifier(3, bootstrap=False, random_state=19).fit(
            np.concatenate([X40, X40[y40 == 3]]), np.concatenate([y40, np.full((y40 == 3).sum(), 35)])),
    }
    return out


def threshold_rows(model, rng, base):
    """Per internal node: rows of `base` with the split feature at the threshold t itself (float64), the float32 values
    just below and above t (t itself and the next one up when t is a float32), and the float64 neighbours of t (which
    round onto or across the float32 ones)."""
    trees = [e.tree_ for e in np.ravel(model.estimators_)]
    # (a forest trained with NaN may split NaN from everything else at threshold +inf: no finite row sits on that one)
    pairs = [(int(tr.feature[i]), float(tr.threshold[i])) for tr in trees for i in range(tr.node_count)
             if tr.children_left[i] >= 0 and np.isfinite(tr.threshold[i])]
    rows = []
    for f, t in pairs:
        lo = np.float32(t)
        if float(lo) > t:
            lo = np.nextafter(lo, np.float32(-np.inf))
        hi = np.nextafter(lo, np.float32(np.inf))
        for v in (t, float(lo), float(hi), float(np.nextafter(lo, np.float32(-np.inf))), np.nextafter(t, -np.inf),
                  np.nextafter(t, np.inf)):
            r = base[rng.integers(base.shape[0])].copy()
            r[f] = v
            rows.append(r)
    return np.array(rows).reshape(-1, base.shape[1])


def query_bank(model, seed=0, nan=False):
    """float64 rows: training-like rows, every threshold case, +-0 against the 0 threshold, subnormals, values at the edge of
    the float32 range (finite after the cast), and NaN in the split features when `nan`."""
    rng = np.random.default_rng(seed)
    base, _ = dataset(n=300, n_classes=max(len(model.classes_), 2), seed=100 + seed)
    base = np.nan_to_num(base)
    rows = [base, threshold_rows(model, rng, base)]
    z = base[:40].copy()
    z[:20, 0], z[20:, 0] = 0.0, -0.0
    rows.append(z)
    s = base[:60].copy()
    s[:, 1] = rng.integers(-300, 300, size=60) * 1e-45 * rng.choice([0.5, 1.0, 1.3], size=60)
    s[:20, 2] = 1e-42
    s[20:40, 3] = -2e-45                                  # rounds to the smallest float32 subnormal's negative or -0
    rows.append(s)
    e = base[:10].copy()
    e[:5, 4] = float(np.finfo(np.float32).max) * (1 + 2.0 ** -25)         # just above FLT_MAX: rounds back to it
    e[5:, 5] = -float(np.finfo(np.float32).max)
    rows.append(e)
    if nan:
        m = base[:80].copy()
        m[rng.random(m.shape) < 0.25] = np.nan
        m[:5] = np.nan
        rows.append(m)
    return np.concatenate(rows)


def refused_rows(F_=F):
    """float64 rows scikit-learn refuses for every model: +-inf, and a value beyond float32's range."""
    r = np.zeros((4, F_))
    r[0, 3] = np.inf
    r[1, 0] = -np.inf
    r[2, 7] = 1e39
    r[3, 5] = -float(np.finfo(np.float32).max) * (1 + 2.0 ** -23)
    return r

"""Host side of forest training (kernel 13, csrc/forest.cuh): what scikit-learn 1.9's RandomForestClassifier /
ExtraTreesClassifier ``fit`` draws from NumPy, drawn with NumPy itself in ``fit``'s order, and the fitted estimator built
from the trees the kernel returns.

The device builds each tree node for node as scikit-learn does; everything NumPy draws stays on the host:
  1. ``_make_estimator`` (scikit-learn's own) draws one ``randint(np.iinfo(np.int32).max)`` per tree from the global
     state: the tree's seed;
  2. a random forest bootstraps with ``RandomState(seed).randint(0, n, n)``; ``np.bincount`` of those indices are the
     tree's sample weights (extra trees: every weight 1);
  3. the tree's splitter takes ``rand_r_state = RandomState(seed).randint(0, RAND_R_MAX)``.
Only the weights and the rand_r seeds go to the device.  The global state afterwards is the one ``fit`` leaves.

The result is a real scikit-learn estimator: its trees come from ``Tree.__setstate__``, so predict, predict_proba,
feature_importances_, pickling and kernel 8 (``consumers.TreeEnsembleModel``) take it as they take a fitted one.
"""
import numpy as np

RAND_R_MAX = 2147483647
MAX_FEATS = 512           # forest::kMaxFeats
MAX_CLASSES = 32          # forest::kMaxClasses
KINDS = {"randomforest": 0, "extratrees": 1}
REGRESSOR = "randomforest_regressor"      # RandomForestRegressor, in draw / derive / tree_seeds

NODE_DTYPE = np.dtype([("left", "<i4"), ("right", "<i4"), ("feature", "<i4"), ("n_samples", "<i4"), ("threshold", "<f8"),
                       ("impurity", "<f8"), ("weighted", "<f8"), ("missing_left", "<i4"), ("pad", "<i4")])
assert NODE_DTYPE.itemsize == 48


class Unsupported(ValueError):
    """The GPU trainer refused the call (a tree's scratch over the bound); NumPy's global state is as before the call."""


def _estimator_class(kind):
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier, RandomForestRegressor
    return {"randomforest": RandomForestClassifier, "extratrees": ExtraTreesClassifier, REGRESSOR: RandomForestRegressor}[kind]


def unsupported(X, y, n_estimators, kind, sample_weight=None, **params):
    """None when the GPU trainer reproduces ``fit`` for these arguments, else the reason it does not (such calls go to
    scikit-learn unchanged).  ``params``: estimator arguments besides n_estimators; only the library's (none) run here."""
    import sklearn
    if not sklearn.__version__.startswith("1.9."):
        return "scikit-learn %s: the trainer restates 1.9.x" % sklearn.__version__
    if kind not in KINDS:
        return "classifier %r: only 'randomforest' and 'extratrees' train on the GPU" % (kind,)
    if params:
        return "hyper-parameters other than the library's: %s" % ", ".join(sorted(params))
    if sample_weight is not None:
        return "sample weights"
    if not (isinstance(n_estimators, (int, np.integer)) and not isinstance(n_estimators, bool) and n_estimators >= 1):
        return "n_estimators must be an integer >= 1, got %r" % (n_estimators,)
    if not isinstance(X, np.ndarray) or X.ndim != 2 or X.shape[0] < 1 or X.shape[1] < 1:
        return "X must be a non-empty 2-d NumPy array"
    if X.dtype.kind not in "fiub":
        return "X must be numeric"
    if X.shape[0] > (1 << 29):
        return "more rows than the trainer's 32-bit node arrays take"
    if X.shape[1] > MAX_FEATS:
        return "%d features: the trainer's shared-memory layout takes at most %d" % (X.shape[1], MAX_FEATS)
    with np.errstate(over="ignore", invalid="ignore"):
        if not np.isfinite(X.astype(np.float32)).all():
            return "NaN or inf in X (as float32): missing-value splits"
    y = np.asarray(y)
    if y.ndim != 1 or y.shape[0] != X.shape[0]:
        return "y must be 1-d with one label per row of X"
    from sklearn.utils.multiclass import type_of_target
    if type_of_target(y) not in ("binary", "multiclass"):
        return "y is not a classification target"
    if np.unique(y).size > MAX_CLASSES:
        return "%d classes: the trainer's shared-memory layout takes at most %d" % (np.unique(y).size, MAX_CLASSES)
    return None


def draw(n_estimators, kind, n):
    """(estimator, trees, weights, seeds): the unfitted estimator with its trees made by scikit-learn's own
    ``_make_estimator`` from the global RNG, every tree's sample weights (int32 [n_trees, n], or None for extra trees)
    and its splitter's rand_r seed (uint32 [n_trees]).  kind: "randomforest", "extratrees" or REGRESSOR."""
    est = _estimator_class(kind)(n_estimators=n_estimators)
    est._validate_estimator()
    rs = np.random.mtrand._rand
    trees = [est._make_estimator(append=False, random_state=rs) for _ in range(n_estimators)]
    weights, seeds = derive([t.random_state for t in trees], kind, n)
    return est, trees, weights, seeds


def derive(tree_seeds, kind, n):
    """(weights, rand_r seeds) of trees with these seeds on n training rows: np.bincount of RandomState(seed).randint(0,
    n, n) (int32 [n_trees, n], a random forest's bootstrap; None for extra trees) and RandomState(seed).randint(0,
    RAND_R_MAX) (uint32 [n_trees])."""
    weights = None
    if kind in ("randomforest", REGRESSOR):
        weights = np.empty((len(tree_seeds), n), dtype=np.int32)
        for i, s in enumerate(tree_seeds):
            weights[i] = np.bincount(np.random.RandomState(s).randint(0, n, n), minlength=n)
    seeds = np.array([np.random.RandomState(s).randint(0, RAND_R_MAX) for s in tree_seeds], dtype=np.uint32)
    return weights, seeds


def tree_seeds(n_estimators, kind):
    """The seeds fit draws for its trees from the global state (scikit-learn's own _make_estimator, one randint each)."""
    est = _estimator_class(kind)(n_estimators=n_estimators)
    est._validate_estimator()
    rs = np.random.mtrand._rand
    return [est._make_estimator(append=False, random_state=rs).random_state for _ in range(n_estimators)]


def tree_state(nodes, values, max_depth, n_classes):
    """Tree.__getstate__ of one tree from the kernel's nodes (NODE_DTYPE) and values [node_count, n_classes]."""
    from sklearn.tree._tree import NODE_DTYPE as SK_NODE
    out = np.zeros(nodes.shape[0], dtype=SK_NODE)
    out["left_child"] = nodes["left"]
    out["right_child"] = nodes["right"]
    out["feature"] = nodes["feature"]
    out["threshold"] = nodes["threshold"]
    out["impurity"] = nodes["impurity"]
    out["n_node_samples"] = nodes["n_samples"]
    out["weighted_n_node_samples"] = nodes["weighted"]
    out["missing_go_to_left"] = nodes["missing_left"]
    vals = np.ascontiguousarray(values, dtype=np.float64).reshape(nodes.shape[0], 1, n_classes)
    return {"max_depth": int(max_depth), "node_count": int(nodes.shape[0]), "nodes": out, "values": vals}


def assemble(est, trees, n_feats, n_samples, classes, states):
    """The fitted estimator: ``fit``'s attributes on `est` and every tree, each tree_ from Tree.__setstate__(state)."""
    from sklearn.tree._tree import Tree
    C = len(classes)
    tree_classes = np.arange(C, dtype=np.float64)
    for t, state in zip(trees, states):
        t.n_features_in_ = n_feats
        t.n_outputs_ = 1
        t.classes_ = tree_classes.copy()
        t.n_classes_ = np.intp(C)
        t.max_features_ = max(1, int(np.sqrt(n_feats)))
        t.tree_ = Tree(n_feats, np.array([C], dtype=np.intp), 1)
        t.tree_.__setstate__(state)
    est.n_features_in_ = n_feats
    est._n_samples = n_samples
    est.n_outputs_ = 1
    est.classes_ = classes
    est.n_classes_ = C
    est._sample_weight = None
    est._n_samples_bootstrap = n_samples if est.bootstrap else None
    est.estimators_ = list(trees)
    return est


# ---- RandomForestRegressor (criterion="squared_error", max_features=1.0, bootstrap; kernel 13's regression builder) ----

def unsupported_regressor(X, y, n_estimators, sample_weight=None, **params):
    """None when the GPU trainer reproduces ``RandomForestRegressor(n_estimators).fit(X, y)`` for these arguments, else
    the reason it does not (such calls go to scikit-learn unchanged).  Only the library's arguments (none besides
    n_estimators) run here."""
    import sklearn
    if not sklearn.__version__.startswith("1.9."):
        return "scikit-learn %s: the trainer restates 1.9.x" % sklearn.__version__
    if params:
        return "hyper-parameters other than the library's: %s" % ", ".join(sorted(params))
    if sample_weight is not None:
        return "sample weights"
    if not (isinstance(n_estimators, (int, np.integer)) and not isinstance(n_estimators, bool) and n_estimators >= 1):
        return "n_estimators must be an integer >= 1, got %r" % (n_estimators,)
    if not isinstance(X, np.ndarray) or X.ndim != 2 or X.shape[0] < 1 or X.shape[1] < 1:
        return "X must be a non-empty 2-d NumPy array"
    if X.dtype.kind not in "fiub":
        return "X must be numeric"
    if X.shape[0] > (1 << 29):
        return "more rows than the trainer's 32-bit node arrays take"
    if X.shape[1] > MAX_FEATS:
        return "%d features: the trainer's shared-memory layout takes at most %d" % (X.shape[1], MAX_FEATS)
    with np.errstate(over="ignore", invalid="ignore"):
        if not np.isfinite(X.astype(np.float32)).all():
            return "NaN or inf in X (as float32): missing-value splits"
    try:
        yv = np.asarray(y, dtype=np.float64)
    except (TypeError, ValueError):
        return "y is not numeric"
    if yv.ndim != 1 or yv.shape[0] != X.shape[0]:
        return "y must be 1-d with one target per row of X"
    if not np.isfinite(yv).all():
        return "NaN or inf in y"
    return None


def assemble_regressor(est, trees, n_feats, n_samples, states):
    """The fitted regressor: ``fit``'s attributes on `est` and every tree, each tree_ a Tree(F, [1], 1) from
    Tree.__setstate__(state) (values [node_count, 1, 1])."""
    from sklearn.tree._tree import Tree
    for t, state in zip(trees, states):
        t.n_features_in_ = n_feats
        t.n_outputs_ = 1
        t.max_features_ = n_feats
        t.tree_ = Tree(n_feats, np.array([1], dtype=np.intp), 1)
        t.tree_.__setstate__(state)
    est.n_features_in_ = n_feats
    est._n_samples = n_samples
    est.n_outputs_ = 1
    est._sample_weight = None
    est._n_samples_bootstrap = n_samples
    est.estimators_ = list(trees)
    return est

"""Host side of gradient boosting training (kernel 13, csrc/forest.cuh boost_leaves): the boosting counterpart of
``forests.py``.

scikit-learn 1.9's ``GradientBoostingClassifier(n_estimators).fit`` splits into steps that need libm and steps that do not:
  - on the host, with scikit-learn's own objects, so that they carry its bits on any CPU: the initial raw prediction
    (``DummyClassifier(strategy="prior")`` through ``_init_raw_predictions``), every stage's negative gradient
    (``-loss.gradient``) and ``train_score_`` (``factor * loss(...)``);
  - on the device, one call per stage (``b200aa_boosting_stage``): the stage's K regression trees, their Newton leaf
    values and the raw-prediction update, all ordered float64 arithmetic.
Each tree's splitter draws one ``randint(0, RAND_R_MAX)`` from the global RandomState at fit time, stage by stage, k
inside the stage, and nothing else in ``fit`` draws from it, so every seed is drawn up front (``draw_seeds``).

The result is a real scikit-learn estimator: its trees come from ``Tree.__setstate__``, so predict, predict_proba,
decision_function, pickling and kernel 8 (``consumers.TreeEnsembleModel``) take it as they take a fitted one.
"""
import numpy as np

from .forests import MAX_CLASSES, MAX_FEATS, RAND_R_MAX


class SingleClass(ValueError):
    """A model-selection training split holds one class, where the reference's fit raises; NumPy's global state is as
    before the call."""


def unsupported(X, y, n_estimators, sample_weight=None, **params):
    """None when the GPU trainer reproduces ``GradientBoostingClassifier(n_estimators).fit(X, y)`` for these arguments,
    else the reason it does not (such calls go to scikit-learn unchanged).  Only the library's arguments (none besides
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
            return "NaN or inf in X (as float32)"
    y = np.asarray(y)
    if y.ndim != 1 or y.shape[0] != X.shape[0]:
        return "y must be 1-d with one label per row of X"
    from sklearn.utils.multiclass import type_of_target
    if type_of_target(y) not in ("binary", "multiclass"):
        return "y is not a classification target"
    n_classes = np.unique(y).size
    if n_classes < 2:
        return "y has one class: fit raises"
    if n_classes > MAX_CLASSES:
        return "%d classes: the trainer takes at most %d trees per stage" % (n_classes, MAX_CLASSES)
    return None


def draw_seeds(count):
    """The splitter seeds of `count` trees, drawn from the global RandomState as each tree's fit draws its own."""
    rs = np.random.mtrand._rand
    return np.array([rs.randint(0, RAND_R_MAX) for _ in range(count)], dtype=np.uint32)


def trees_per_stage(n_classes):
    """n_trees_per_iteration_: 1 for two classes (binomial loss), else the class count."""
    return 1 if n_classes <= 2 else int(n_classes)


def begin(X, y, n_estimators):
    """(est, X32, y_enc, raw0): an unfitted GradientBoostingClassifier(n_estimators) taken through ``fit``'s preamble
    with scikit-learn's own methods (validate_data, _encode_y, _set_max_features, _get_loss, _init_state, init_.fit, the
    global RandomState as _rng), X as fit casts it (float32), the encoded labels (float64) and the initial raw prediction
    of one row [1, K] (the prior's link, the same for every row).  Draws nothing."""
    from sklearn.ensemble import GradientBoostingClassifier
    from sklearn.ensemble._gb import _init_raw_predictions
    from sklearn.utils import check_random_state, column_or_1d
    from sklearn.utils.validation import _check_sample_weight, validate_data
    est = GradientBoostingClassifier(n_estimators=int(n_estimators))
    X32, yv = validate_data(est, X, y, accept_sparse=["csr", "csc", "coo"], dtype=np.float32, multi_output=True)
    sw = _check_sample_weight(None, X32)
    y_enc = column_or_1d(est._encode_y(y=yv, sample_weight=None), warn=True)
    est._set_max_features()
    est._loss = est._get_loss(sample_weight=sw)
    est._init_state()
    est.init_.fit(X32, y_enc)
    raw0 = _init_raw_predictions(X32[:1], est.init_, est._loss, True)
    est._rng = check_random_state(est.random_state)
    return est, X32, y_enc, raw0


def loss_factor(loss):
    """_fit_stages' factor of train_score_: 2 for the binomial loss, 1 for the multinomial one."""
    from sklearn._loss.loss import HalfBinomialLoss
    return 2 if isinstance(loss, HalfBinomialLoss) else 1


def neg_gradient(loss, y_enc, raw):
    """-loss.gradient as _fit_stage computes it, as [n, K] float64."""
    g = -loss.gradient(y_true=y_enc, raw_prediction=raw, sample_weight=None)
    return np.ascontiguousarray(g.reshape(raw.shape[0], -1), dtype=np.float64)


def make_tree(est, n_feats, state):
    """One fitted stage tree: the DecisionTreeRegressor _fit_stage makes (random_state the global RandomState), with
    ``fit``'s attributes and tree_ from Tree.__setstate__(state)."""
    from sklearn.tree import DecisionTreeRegressor
    from sklearn.tree._tree import Tree
    t = DecisionTreeRegressor(criterion="squared_error", splitter="best", max_depth=est.max_depth,
                              min_samples_split=est.min_samples_split, min_samples_leaf=est.min_samples_leaf,
                              min_weight_fraction_leaf=est.min_weight_fraction_leaf,
                              min_impurity_decrease=est.min_impurity_decrease, max_features=est.max_features,
                              max_leaf_nodes=est.max_leaf_nodes, random_state=est._rng, ccp_alpha=est.ccp_alpha)
    t.n_features_in_ = n_feats
    t.n_outputs_ = 1
    t.max_features_ = n_feats
    t.tree_ = Tree(n_feats, np.array([1], dtype=np.intp), 1)
    t.tree_.__setstate__(state)
    return t


def problem_init(y_train):
    """(classes, K, loss, y_enc, raw0 [1, K]) of one model-selection problem's training labels, as fit makes them: the
    present classes (LabelEncoder), the loss fit builds, and the prior's initial raw prediction."""
    est, _, y_enc, raw0 = begin(np.zeros((len(y_train), 1)), y_train, 1)
    return est.classes_, est.n_trees_per_iteration_, est._loss, y_enc, raw0

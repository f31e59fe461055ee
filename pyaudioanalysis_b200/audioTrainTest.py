"""The kNN and forest model selection of the reference's audioTrainTest.evaluate_classifier (audioTrainTest.py:576-771)
on the GPU.

For every neighbour count in `params` and each of `n_exp` experiments the reference draws a train / test split, fits a
StandardScaler on the training rows, classifies every test row with its Knn and scores the experiment with scikit-learn.
Here the splits are drawn up front from NumPy's global RNG in the reference's order, all (param, experiment) problems go
to the GPU in one call (``consumers.knn_cross_validate``, kernel 6), and the per-experiment confusion counts come back.
The reference's scores follow from those counts: its confusion_matrix is the count block restricted to the classes in
y_test or y_pred, and its macro f1_score is the mean over those classes of 2 tp / (n_true + n_pred).  The printed table
and the returned parameter are the reference's, text for text.

The forests ("randomforest", "extratrees") go the same way: each problem's split and then its forest's tree seeds are
drawn in the reference's order, and ``consumers.forest_cross_validate`` (kernel 13) scales, trains and classifies every
problem on the device, bit for bit scikit-learn 1.9's fit and predict.  So does "gradientboosting": each problem's split,
then the n_estimators * K splitter seeds its fit draws, and ``consumers.boosting_cross_validate`` runs every problem's
stages together, the gradients on the host with scikit-learn's loss and the trees on the device.

Only "knn", "randomforest", "extratrees" and "gradientboosting" without SMOTE on finite float64 features run here
(``unsupported`` says why not otherwise); ``install.install_training`` sends everything else to the reference's own
function.
"""
import math

import numpy as np
from sklearn.model_selection import GroupShuffleSplit


_FORESTS = ("randomforest", "extratrees")
_TREES = _FORESTS + ("gradientboosting",)


def features_to_matrix(features):
    """(X [n, F], y [n] float64 class indices): the class matrices stacked in order (audioTrainTest.py:887-911)."""
    X = np.vstack([np.asarray(f) for f in features])
    y = np.concatenate([i * np.ones(len(f)) for i, f in enumerate(features)])
    return X, y


def unsupported(features, classifier_name, params, train_percentage=0.90, smote=False):
    """None when evaluate_classifier runs on the GPU for these arguments, else the reason it does not."""
    if classifier_name not in ("knn",) + _TREES:
        return "classifier %r: only 'knn', 'randomforest', 'extratrees' and 'gradientboosting' run on the GPU" % (
            classifier_name,)
    if classifier_name in _TREES:
        import sklearn
        if not sklearn.__version__.startswith("1.9."):
            return "scikit-learn %s: the forest trainer restates 1.9.x" % sklearn.__version__
    if smote:
        return "SMOTE resamples the training rows"
    if len(features) < 2:
        return "fewer than two classes"
    shapes = set()
    for f in features:
        a = np.asarray(f)
        if a.ndim != 2 or a.shape[0] < 1 or a.dtype != np.float64:
            return "every class needs a non-empty float64 [n, F] matrix"
        if not np.isfinite(a).all():
            return "non-finite features"
        shapes.add(a.shape[1])
    # StandardScaler's column sums add the rows in sequence only when a row holds more than one value (numpy sums a
    # single contiguous column pairwise)
    if len(shapes) != 1 or shapes.pop() < 2:
        return "the classes need the same number (>= 2) of features"
    if classifier_name in _TREES:
        if features[0].shape[1] > 512 or len(features) > 32:
            return "more than 512 features or 32 classes: the forest trainer's shared-memory layout"
        with np.errstate(over="ignore"):
            if not all(np.isfinite(np.asarray(f).astype(np.float32)).all() for f in features):
                return "features that become inf as float32"
    for k in params:
        if not (isinstance(k, (int, np.integer)) and not isinstance(k, bool) and k >= 1):
            return "every parameter (kNN neighbours, forest trees) must be an integer >= 1, got %r" % (k,)
    if not 0 < 1 - train_percentage < 1:
        return "train_percentage must leave a test fraction in (0, 1)"
    return None


def split_sizes(n, train_percentage):
    """(n_train, n_test) of train_test_split(X, y, test_size=1 - train_percentage) on n rows."""
    n_test = math.ceil((1 - train_percentage) * n)
    return n - n_test, n_test


def draw_splits(X, y, n_params, n_exp, train_percentage, list_of_ids=None):
    """The (train, test) row indices of every (param, experiment), params outer, drawn as the reference draws them:
    GroupShuffleSplit(n_splits=n_exp, train_size=.8) once for all params (:624-629), else one
    train_test_split(X, y, test_size=1 - train_percentage) per (param, experiment) from NumPy's global RNG (:648-649),
    whose ShuffleSplit takes one permutation: test = perm[:n_test], train = perm[n_test:n_test + n_train]."""
    if list_of_ids:
        gss = GroupShuffleSplit(n_splits=n_exp, train_size=.8)
        fixed = [(train, test) for train, test in gss.split(X, y, list_of_ids)]
        return fixed * n_params
    n = X.shape[0]
    n_train, n_test = split_sizes(n, train_percentage)
    if n_train < 1:
        raise ValueError("train_percentage %r leaves no training row of %d" % (train_percentage, n))
    splits = []
    for _ in range(n_params * n_exp):
        perm = np.random.permutation(n)
        splits.append((perm[n_test:n_test + n_train], perm[:n_test]))
    return splits


def draw_forest_problems(X, params, n_exp, train_percentage, kind, list_of_ids=None):
    """(splits, seeds) of every (param, experiment) of the forest branch, params outer, drawn from NumPy's global RNG in
    the reference's order: GroupShuffleSplit's splits once up front (list_of_ids), then per problem its
    train_test_split permutation (without list_of_ids) followed by the seeds its forest's fit draws, one per tree."""
    fixed = draw_splits(X, None, 1, n_exp, train_percentage, list_of_ids) if list_of_ids else None
    from .forests import tree_seeds
    splits, seeds = [], []
    for C in params:
        for e in range(n_exp):
            splits.append(fixed[e] if fixed else draw_splits(X, None, 1, 1, train_percentage)[0])
            seeds.append(tree_seeds(int(C), kind))
    return splits, seeds


def draw_boosting_problems(X, y, params, n_exp, train_percentage, list_of_ids=None):
    """(splits, seeds) of every (param, experiment) of the "gradientboosting" branch, params outer, drawn from NumPy's
    global RNG in the reference's order: GroupShuffleSplit's splits once up front (list_of_ids), then per problem its
    train_test_split permutation (without list_of_ids) followed by the n_estimators * K seeds its fit draws, K from the
    classes in its training rows.  None when a training set holds a single class (the reference's fit raises there)."""
    from .boosting import draw_seeds, trees_per_stage
    fixed = draw_splits(X, None, 1, n_exp, train_percentage, list_of_ids) if list_of_ids else None
    splits, seeds = [], []
    for C in params:
        for e in range(n_exp):
            split = fixed[e] if fixed else draw_splits(X, None, 1, 1, train_percentage)[0]
            present = np.unique(y[split[0]]).size
            if present < 2:
                return None
            splits.append(split)
            seeds.append(draw_seeds(int(C) * trees_per_stage(present)))
    return splits, seeds


def experiment_scores(counts, all_classes):
    """(cmt, f1t) of one experiment from its [C, C] counts, as the reference has them: confusion_matrix(y_test, y_pred)
    over the classes present, widened back to C x C by the reference's own insertion (:690-699), and the macro F1."""
    true, pred = counts.sum(axis=1), counts.sum(axis=0)
    present = np.flatnonzero(true + pred)
    cmt = counts[np.ix_(present, present)]
    f1t = np.mean(2.0 * np.diagonal(cmt) / (1.0 * true[present] + pred[present]))
    if cmt.size != counts.size:
        # the reference's set iteration order decides the insertion order; keep it
        missing = [int(c) for c in all_classes.difference(set(present.tolist()))]
        for m in missing:
            cmt = np.insert(cmt, m, 0, axis=0)
        for m in missing:
            cmt = np.insert(cmt, m, 0, axis=1)
    return cmt, f1t


def _print_confusion_matrix(cm, class_names):
    if cm.shape[0] != len(class_names):
        print("printConfusionMatrix: Wrong argument sizes\n")
        return
    short = [c[0:3] if len(c) > 4 else c for c in class_names]
    print("".join("\t" + c for c in short))
    total = np.sum(cm)
    for i, c in enumerate(short):
        print(c + "".join("\t{0:.2f}".format(100.0 * cm[i][j] / total) for j in range(len(class_names))))


def report(y, class_names, params, parameter_mode, n_exp, counts):
    """Everything evaluate_classifier prints, and its return value, from the confusion counts [len(params) * n_exp, C, C]
    of its (param, experiment) problems (params outer)."""
    all_classes = set(y)
    n_classes = counts.shape[1]
    pre_all, rec_all, f1_cls_all, ac_all, f1_all, f1_std_all, cms_all = [], [], [], [], [], [], []
    for ci, C in enumerate(params):
        cm = np.zeros((n_classes, n_classes))
        f1_per_exp = []
        for e in range(n_exp):
            print("Param = {0:.5f} - classifier Evaluation Experiment {1:d} of {2:d}".format(C, e + 1, n_exp))
            cmt, f1t = experiment_scores(counts[ci * n_exp + e], all_classes)
            f1_per_exp.append(f1t)
            cm = cm + cmt
        cm = cm + 0.0000000010
        rec = np.array([cm[i, i] / np.sum(cm[i, :]) for i in range(n_classes)])
        pre = np.array([cm[i, i] / np.sum(cm[:, i]) for i in range(n_classes)])
        f1 = 2 * rec * pre / (rec + pre)
        pre_all.append(pre)
        rec_all.append(rec)
        f1_cls_all.append(f1)
        ac_all.append(np.sum(np.diagonal(cm)) / np.sum(cm))
        cms_all.append(cm)
        f1_all.append(np.mean(f1))
        f1_std_all.append(np.std(f1_per_exp))

    names = ["{0:s}\t\t\t".format(c) for c in class_names[:-1]] + ["{0:s}\t\t".format(c) for c in class_names[-1:]]
    print("\t\t" + "".join(names) + "OVERALL")
    print("\tC" + "\tPRE\tREC\tf1" * len(class_names) + "\t{0:s}\t{1:s}".format("ACC", "f1"))
    best_ac, best_f1 = np.argmax(ac_all), np.argmax(f1_all)
    for i in range(len(pre_all)):
        line = "\t{0:.3f}".format(params[i])
        for c in range(len(pre_all[i])):
            line += "\t{0:.1f}\t{1:.1f}\t{2:.1f}".format(100.0 * pre_all[i][c], 100.0 * rec_all[i][c], 100.0 * f1_cls_all[i][c])
        line += "\t{0:.1f}\t{1:.1f}".format(100.0 * ac_all[i], 100.0 * f1_all[i])
        line += "\t best f1" if i == best_f1 else ""
        line += "\t best Acc" if i == best_ac else ""
        print(line)
    if parameter_mode == 0:
        print("Confusion Matrix:")
        _print_confusion_matrix(cms_all[best_ac], class_names)
        return params[best_ac]
    if parameter_mode == 1:
        print("Confusion Matrix:")
        _print_confusion_matrix(cms_all[best_f1], class_names)
        print(f"Best macro f1 {100 * f1_all[best_f1]:.1f}")
        print(f"Best macro f1 std {100 * f1_std_all[best_f1]:.1f}")
        return params[best_f1]
    return None


def evaluate_classifier(features, class_names, classifier_name, params, parameter_mode, list_of_ids=None, n_exp=-1,
                        train_percentage=0.90, smote=False):
    """audioTrainTest.evaluate_classifier (:576-771) for classifier_name "knn", "randomforest", "extratrees" and
    "gradientboosting": the same prints and return value, every (param, experiment) problem trained (trees) and
    classified on the GPU in one call.  Raises ValueError for arguments it does not cover (``unsupported``), and
    ``boosting.SingleClass`` (a ValueError), with NumPy's global state as before the call, when a boosting training set
    holds one class; there is no CPU path."""
    from .consumers import boosting_cross_validate, forest_cross_validate, knn_cross_validate
    why = unsupported(features, classifier_name, params, train_percentage, smote)
    if why is not None:
        raise ValueError("evaluate_classifier on the GPU: " + why)
    X, y = features_to_matrix(features)
    if n_exp == -1:
        n_exp = int(50000 / X.shape[0]) + 1
    if classifier_name == "gradientboosting":
        from .boosting import SingleClass
        state = np.random.get_state()
        drawn = draw_boosting_problems(X, y, params, n_exp, train_percentage, list_of_ids)
        if drawn is None:
            np.random.set_state(state)
            raise SingleClass("evaluate_classifier on the GPU: a training split holds a single class")
        stages = [int(C) for C in params for _ in range(n_exp)]
        try:
            _, counts = boosting_cross_validate(X, y, drawn[0], drawn[1], stages, n_classes=len(features))
        except ValueError:
            np.random.set_state(state)
            raise
        return report(y, class_names, params, parameter_mode, n_exp, counts.cpu().numpy())
    if classifier_name in _FORESTS:
        splits, seeds = draw_forest_problems(X, params, n_exp, train_percentage, classifier_name, list_of_ids)
        trees = [int(C) for C in params for _ in range(n_exp)]
        _, counts = forest_cross_validate(X, y, splits, seeds, trees, classifier_name, n_classes=len(features))
        return report(y, class_names, params, parameter_mode, n_exp, counts.cpu().numpy())
    splits = draw_splits(X, y, len(params), n_exp, train_percentage, list_of_ids)
    ks = [int(C) for C in params for _ in range(n_exp)]
    _, counts = knn_cross_validate(X, y, splits, ks, n_classes=len(features))
    return report(y, class_names, params, parameter_mode, n_exp, counts.cpu().numpy())


def dispatcher(original):
    """An evaluate_classifier that runs the arguments the GPU covers here and hands the rest to `original`."""
    from .boosting import SingleClass
    from .forests import Unsupported

    def evaluate_classifier_dispatch(features, class_names, classifier_name, params, parameter_mode, list_of_ids=None,
                                     n_exp=-1, train_percentage=0.90, smote=False):
        kw = dict(list_of_ids=list_of_ids, n_exp=n_exp, train_percentage=train_percentage, smote=smote)
        if unsupported(features, classifier_name, params, train_percentage, smote) is None:
            try:
                return evaluate_classifier(features, class_names, classifier_name, params, parameter_mode, **kw)
            except (SingleClass, Unsupported):
                pass                    # NumPy's state is as before the call: the original draws the same problems
        return original(features, class_names, classifier_name, params, parameter_mode, **kw)
    evaluate_classifier_dispatch.original = original
    return evaluate_classifier_dispatch


def _train_forest(kind, features, labels, n_estimators):
    from . import forests
    from .consumers import forest_fit
    X = np.asarray(features) if not isinstance(features, np.ndarray) else features
    if forests.unsupported(X, labels, n_estimators, kind) is None:
        return forest_fit(X, labels, n_estimators, kind)
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    cls = RandomForestClassifier if kind == "randomforest" else ExtraTreesClassifier
    return cls(n_estimators=n_estimators).fit(features, labels)


def train_random_forest(features, labels, n_estimators):
    """audioTrainTest.train_random_forest (:158-178): RandomForestClassifier(n_estimators).fit(features, labels), trained
    on the GPU (``consumers.forest_fit``) tree for tree as scikit-learn trains it; arguments the trainer does not
    reproduce (``forests.unsupported``) go to scikit-learn."""
    return _train_forest("randomforest", features, labels, n_estimators)


def train_extra_trees(features, labels, n_estimators):
    """audioTrainTest.train_extra_trees (:202-219), as ``train_random_forest`` with ExtraTreesClassifier."""
    return _train_forest("extratrees", features, labels, n_estimators)


def train_gradient_boosting(features, labels, n_estimators):
    """audioTrainTest.train_gradient_boosting (:181-199): GradientBoostingClassifier(n_estimators).fit(features,
    labels), trained on the GPU (``consumers.boosting_fit``) stage for stage as scikit-learn trains it; arguments the
    trainer does not reproduce (``boosting.unsupported``) or whose trees would exceed its scratch bound
    (``forests.Unsupported``) go to scikit-learn."""
    from . import boosting, forests
    from .consumers import boosting_fit
    X = np.asarray(features) if not isinstance(features, np.ndarray) else features
    if boosting.unsupported(X, labels, n_estimators) is None:
        try:
            return boosting_fit(X, labels, n_estimators)
        except forests.Unsupported:
            pass                        # one tree over the scratch bound; NumPy's state is untouched
    from sklearn.ensemble import GradientBoostingClassifier
    return GradientBoostingClassifier(n_estimators=n_estimators).fit(features, labels)


# ---- regression: evaluate_regression's "randomforest" branch and train_random_forest_regression ----

def train_random_forest_regression(features, labels, n_estimators):
    """audioTrainTest.train_random_forest_regression: ``(rf, train_err)`` with rf =
    RandomForestRegressor(n_estimators).fit(features, labels) trained on the GPU (``consumers.forest_regressor_fit``) tree
    for tree as scikit-learn trains it, and train_err = np.mean(np.abs(rf.predict(features) - labels)); arguments the
    trainer does not reproduce (``forests.unsupported_regressor``) or whose trees would exceed its scratch bound
    (``forests.Unsupported``) go to scikit-learn."""
    from . import forests
    from .consumers import forest_regressor_fit
    X = np.asarray(features) if not isinstance(features, np.ndarray) else features
    rf = None
    if forests.unsupported_regressor(X, labels, n_estimators) is None:
        try:
            rf = forest_regressor_fit(X, labels, n_estimators)
        except forests.Unsupported:
            pass                        # one tree over the scratch bound; NumPy's state is untouched
    if rf is None:
        from sklearn.ensemble import RandomForestRegressor
        rf = RandomForestRegressor(n_estimators=n_estimators).fit(features, labels)
    train_err = np.mean(np.abs(rf.predict(features) - labels))
    return rf, train_err


def unsupported_regression(features, labels, n_exp, method_name, params):
    """None when evaluate_regression here reproduces the reference's for these arguments, else the reason it does not."""
    import sklearn
    if method_name != "randomforest":
        return "method %r: only 'randomforest' runs on the GPU" % (method_name,)
    if not sklearn.__version__.startswith("1.9."):
        return "scikit-learn %s: the forest trainer restates 1.9.x" % sklearn.__version__
    if not (isinstance(features, np.ndarray) and features.dtype == np.float64 and features.ndim == 2 and
            features.flags.c_contiguous and features.shape[0] >= 1 and features.shape[1] >= 1):
        return "features must be a non-empty C-contiguous float64 matrix (the scaler's column sums follow the layout)"
    if features.shape[1] > 512:
        return "more than 512 features: the forest trainer's shared-memory layout"
    if not np.isfinite(features).all():
        return "NaN or inf in the features"
    if not isinstance(labels, np.ndarray) or labels.ndim != 1 or labels.shape[0] != features.shape[0]:
        return "labels must be a 1-d array with one target per row"
    if labels.dtype.kind not in "fiub" or not np.isfinite(labels.astype(np.float64)).all():
        return "labels must be finite numbers"
    n = labels.shape[0]
    if int(round(0.9 * n)) == n:
        return "no test rows (n_train == n): the reference's errors are NaN"
    if not (isinstance(n_exp, (int, np.integer)) and n_exp >= 1):
        return "n_exp must be an integer >= 1"
    for C in params:
        if not (isinstance(C, (int, np.integer)) and not isinstance(C, bool) and C >= 1):
            return "every parameter (forest trees) must be an integer >= 1, got %r" % (C,)
    return None


def draw_regression_problems(n, params, n_exp):
    """(splits, seeds) of every (param, experiment) of evaluate_regression's forest branch, params outer, drawn from
    NumPy's global RNG in the reference's order: per problem np.random.permutation(range(n)), then the seeds its forest's
    fit draws.  The first int(round(0.9 n)) rows of the permutation train, the rest test."""
    from .forests import REGRESSOR, tree_seeds
    n_train = int(round(0.9 * n))
    splits, seeds = [], []
    for C in params:
        for _ in range(n_exp):
            randperm = np.random.permutation(range(n))
            splits.append((randperm[:n_train], randperm[n_train:]))
            seeds.append(tree_seeds(int(C), REGRESSOR))
    return splits, seeds


def evaluate_regression(features, labels, n_exp, method_name, params):
    """audioTrainTest.evaluate_regression for method_name "randomforest": the same prints and return value, every
    (param, experiment) problem's forest trained and its test and training rows predicted on the GPU in one call
    (``consumers.forest_regression_cross_validate``); the errors and means are the reference's NumPy expressions on the
    host.  Raises ValueError for arguments it does not cover (``unsupported_regression``), and ``forests.Unsupported``
    (a ValueError), with NumPy's global state as before the call, when one tree would exceed the trainer's scratch
    bound."""
    from .consumers import forest_regression_cross_validate
    from .forests import Unsupported
    why = unsupported_regression(features, labels, n_exp, method_name, params)
    if why is not None:
        raise ValueError("evaluate_regression on the GPU: " + why)
    n_samples = labels.shape[0]
    state = np.random.get_state()
    splits, seeds = draw_regression_problems(n_samples, params, n_exp)
    trees = [int(C) for C in params for _ in range(n_exp)]
    try:
        pred_test, pred_train = forest_regression_cross_validate(features, labels, splits, seeds, trees)
    except Unsupported:
        np.random.set_state(state)
        raise
    pred_test, pred_train = pred_test.cpu().numpy(), pred_train.cpu().numpy()
    errors_all, er_train_all, er_base_all = [], [], []
    k, o_te, o_tr = 0, 0, 0
    for C in params:
        errors, errors_train, errors_baseline = [], [], []
        for _ in range(n_exp):
            tr, te = splits[k]
            k += 1
            l_train = [labels[i] for i in tr]
            l_test = [labels[i] for i in te]
            p_tr, p_te = pred_train[o_tr:o_tr + tr.size], pred_test[o_te:o_te + te.size]
            o_tr += tr.size
            o_te += te.size
            train_err = np.mean(np.abs(p_tr - l_train))
            error_test, error_test_baseline = [], []
            for itest in range(te.size):
                R = p_te[itest]
                Rbaseline = np.mean(l_train)
                error_test.append((R - l_test[itest]) * (R - l_test[itest]))
                error_test_baseline.append((Rbaseline - l_test[itest]) * (Rbaseline - l_test[itest]))
            errors.append(np.array(error_test).mean())
            errors_train.append(train_err)
            errors_baseline.append(np.array(error_test_baseline).mean())
        errors_all.append(np.array(errors).mean())
        er_train_all.append(np.array(errors_train).mean())
        er_base_all.append(np.array(errors_baseline).mean())
    best_ind = np.argmin(errors_all)
    print("{0:s}\t\t{1:s}\t\t{2:s}\t\t{3:s}".format("Param", "MSE", "T-MSE", "R-MSE"))
    for i in range(len(errors_all)):
        print("{0:.4f}\t\t{1:.2f}\t\t{2:.2f}\t\t{3:.2f}".format(params[i], errors_all[i], er_train_all[i], er_base_all[i]),
              end="")
        if i == best_ind:
            print("\t\t best", end="")
        print("")
    return params[best_ind], errors_all[best_ind], er_base_all[best_ind]


def regression_dispatcher(original):
    """An evaluate_regression that runs the arguments the GPU covers here ("randomforest") and hands the rest ("svm",
    "svm_rbf", anything ``unsupported_regression`` names, and trees over the scratch bound) to `original`."""
    from .forests import Unsupported

    def evaluate_regression_dispatch(features, labels, n_exp, method_name, params):
        if unsupported_regression(features, labels, n_exp, method_name, params) is None:
            try:
                return evaluate_regression(features, labels, n_exp, method_name, params)
            except Unsupported:
                pass                    # NumPy's state is as before the call: the original draws the same problems
        return original(features, labels, n_exp, method_name, params)
    evaluate_regression_dispatch.original = original
    return evaluate_regression_dispatch

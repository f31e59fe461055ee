"""GPU: kernel 13 (b200aa_forest_fit, consumers.forest_fit) against scikit-learn 1.9's RandomForestClassifier /
ExtraTreesClassifier fit under the same NumPy global state: every tree's state in bits, the fitted attributes and the
global state afterwards, on the CPU harness's problems, a 500-tree forest and a forest spanning several scratch slices;
at 512 features and 32 classes, at root sizes on the team and padding edges, on proxy ties across thread chunks and on
duplicated columns; GPU-built models through kernel 8 and pickle; concurrent streams and threads; the drop-ins and install_training."""
import pickle
import threading
import types

import numpy as np
import pytest
import torch

from tests import forest_cases as FC

pytestmark = pytest.mark.gpu


def _sklearn(kind):
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    return RandomForestClassifier if kind == "randomforest" else ExtraTreesClassifier


def _check(X, y, kind, n_estimators, seed=11):
    from pyaudioanalysis_b200.consumers import forest_fit
    np.random.seed(seed)
    ref = _sklearn(kind)(n_estimators=n_estimators).fit(X, y)
    ref_state = np.random.get_state()
    np.random.seed(seed)
    got = forest_fit(X, y, n_estimators, kind)
    assert FC.same_state(np.random.get_state(), ref_state)
    FC.compare(got, ref)
    return got, ref


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
@pytest.mark.parametrize("case", FC.problems(), ids=lambda c: c[0])
def test_forest_equals_sklearn(kind, case):
    _, X, y = case
    got, ref = _check(X, y, kind, 6)
    assert np.array_equal(got.predict_proba(X), ref.predict_proba(X))


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
def test_500_trees(kind):
    r = np.random.RandomState(21)
    X, y = r.randn(1000, 136), r.randint(0, 4, 1000)
    _check(X, y, kind, 500, seed=4)


def test_several_scratch_slices():
    # 20 000 rows: about 4.3 MB of scratch per tree, so 150 trees take three 256 MB slices
    r = np.random.RandomState(8)
    X, y = r.randn(20000, 11), r.randint(0, 4, 20000)
    _check(X, y, "randomforest", 150, seed=2)


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
def test_512_features_32_classes(kind):
    """The launchers' limits: forest_build_kernel asks for 49 832 B of dynamic shared memory, past the 48 KB default, and
    every class-count array runs full."""
    X, y = FC.limits()
    got, ref = _check(X, y, kind, 4)
    assert np.array_equal(got.predict_proba(X), ref.predict_proba(X))


def _draw_unweighted(n_estimators, kind, n):
    """FO.draw for RandomForestClassifier(bootstrap=False): the best splitter on every sample with weight 1, as
    b200aa_forest_fit builds it when given no weights."""
    from sklearn.ensemble import RandomForestClassifier
    from pyaudioanalysis_b200 import forests as FO
    assert kind == "randomforest"
    est = RandomForestClassifier(n_estimators=n_estimators, bootstrap=False)
    est._validate_estimator()
    rs = np.random.mtrand._rand
    trees = [est._make_estimator(append=False, random_state=rs) for _ in range(n_estimators)]
    return est, trees, None, FO.derive([t.random_state for t in trees], "extratrees", n)[1]


@pytest.mark.parametrize("n", FC.ROOT_SIZES)
def test_root_sizes_at_team_and_padding_edges(n, monkeypatch):
    """Roots of exactly n rows (unweighted: extra trees, and the best splitter with h_weights = NULL against
    RandomForestClassifier(bootstrap=False)): one row per thread and one over, and the bitonic sort's padding."""
    from sklearn.ensemble import RandomForestClassifier
    from pyaudioanalysis_b200 import forests as FO
    from pyaudioanalysis_b200.consumers import forest_fit
    r = np.random.RandomState(n)
    X, y = np.round(r.randn(n, 7), 1), r.randint(0, 5, n)
    _check(X, y, "extratrees", 3)
    np.random.seed(12)
    ref = RandomForestClassifier(n_estimators=3, bootstrap=False).fit(X, y)
    monkeypatch.setattr(FO, "draw", _draw_unweighted)
    np.random.seed(12)
    got = forest_fit(X, y, 3, "randomforest")
    FC.compare(got, ref)
    assert got.estimators_[0].tree_.n_node_samples[0] == n


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
@pytest.mark.parametrize("n", [300, 1000])
def test_proxy_ties_across_thread_chunks(kind, n):
    """Palindrome labels: splits at p and n - p tie, and at these n the tied positions lie in different threads' chunks,
    so the cross-thread reduction must keep the first."""
    X, y = FC.palindrome(39, n)
    _check(X, y, kind, 4)


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
def test_duplicated_columns_first_visit_wins(kind):
    X, y = FC.duplicated_columns(3)
    _check(X, y, kind, 6)


def test_device_input_and_float32():
    from pyaudioanalysis_b200.consumers import forest_fit
    r = np.random.RandomState(5)
    X, y = r.randn(400, 11), r.randint(0, 3, 400)
    np.random.seed(1)
    ref = _sklearn("extratrees")(n_estimators=8).fit(X, y)
    for d in (torch.from_numpy(X).cuda(), torch.from_numpy(X.astype(np.float32)).cuda()):
        np.random.seed(1)
        FC.compare(forest_fit(d, y, 8, "extratrees"), ref)


def test_models_through_kernel8_and_pickle():
    from pyaudioanalysis_b200.consumers import TreeEnsembleModel, forest_fit, tree_classify_batch
    r = np.random.RandomState(9)
    X, y = r.randn(600, 136), r.randint(0, 4, 600)
    Q = r.randn(300, 136)
    for kind in ("randomforest", "extratrees"):
        np.random.seed(3)
        m = forest_fit(X, y, 50, kind)
        m2 = pickle.loads(pickle.dumps(m))
        np.random.seed(3)
        FC.compare(m2, _sklearn(kind)(n_estimators=50).fit(X, y))
        ids, P = tree_classify_batch(TreeEnsembleModel(m2), torch.from_numpy(Q).cuda())
        assert np.array_equal(P.cpu().numpy(), m.predict_proba(Q))
        assert np.array_equal(ids.cpu().numpy(), np.argmax(m.predict_proba(Q), axis=1))


def test_streams_and_threads():
    from pyaudioanalysis_b200.consumers import forest_fit
    r = np.random.RandomState(13)
    probs = [(r.randn(700, 11), r.randint(0, 3, 700), k) for k in ("randomforest", "extratrees", "randomforest")]
    # every thread fits on a stream of its own; the fits draw from NumPy's one global state, so each seeds and fits under
    # a lock, and its forest is the sequential fit from the same seed
    expected = []
    for i, (X, y, k) in enumerate(probs):
        np.random.seed(100 + i)
        expected.append(_sklearn(k)(n_estimators=20).fit(X, y))
    lock, got, errors = threading.Lock(), [None] * len(probs), []

    def work(i):
        try:
            X, y, k = probs[i]
            s = torch.cuda.Stream()
            with torch.cuda.stream(s), lock:
                np.random.seed(100 + i)
                got[i] = forest_fit(X, y, 20, k)
        except Exception as e:                      # noqa: BLE001 - reported below
            errors.append(e)
    ts = [threading.Thread(target=work, args=(i,)) for i in range(len(probs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for g, e in zip(got, expected):
        FC.compare(g, e)


def test_drop_ins_and_install_training():
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    r = np.random.RandomState(17)
    X, y = r.randn(300, 11), np.array(["a", "b", "c"])[r.randint(0, 3, 300)]
    calls = []

    def rf(features, labels, n):
        calls.append("rf")

    def et(features, labels, n):
        calls.append("et")
    mod = types.ModuleType("standin_training")
    mod.evaluate_classifier = lambda *a, **k: None
    mod.train_random_forest, mod.train_extra_trees = rf, et
    names = install_training(mod)
    try:
        assert names == ["standin_training.evaluate_classifier", "standin_training.train_random_forest",
                         "standin_training.train_extra_trees"]
        for name, kind in (("train_random_forest", "randomforest"), ("train_extra_trees", "extratrees")):
            np.random.seed(6)
            got = getattr(mod, name)(X, y, 10)
            np.random.seed(6)
            FC.compare(got, _sklearn(kind)(n_estimators=10).fit(X, y))
        # what the GPU trainer refuses goes to scikit-learn unchanged
        bad = X.copy()
        bad[0, 0] = np.nan
        np.random.seed(6)
        m = at.train_random_forest(bad, y, 5)
        np.random.seed(6)
        FC.compare(m, _sklearn("randomforest")(n_estimators=5).fit(bad, y))
        assert calls == []
    finally:
        uninstall()
    assert mod.train_random_forest is rf and mod.train_extra_trees is et


def _golden_case(g, c):
    from tests.knn_cv_oracle import seeded_features
    seed, F = (int(v) for v in g[c + "_gen"])
    feats = seeded_features(seed, tuple(int(s) for s in g[c + "_sizes"]), F)
    assert np.float64(np.vstack(feats).sum()) == g[c + "_X_sum"]
    ids = [int(i) for i in g[c + "_ids"]] or None
    return feats, dict(class_names=[str(s) for s in g[c + "_class_names"]], classifier_name=str(g[c + "_classifier"]),
                       params=g[c + "_params"], parameter_mode=int(g[c + "_mode"]), list_of_ids=ids,
                       n_exp=int(g[c + "_n_exp"]), train_percentage=float(g[c + "_train_percentage"]))


def test_evaluate_classifier_goldens_directly_and_through_install_training():
    """The unmodified reference's evaluate_classifier for both forests (tests/golden/forest_cv.npz): printed text and
    return value, from our evaluate_classifier and from a module whose evaluate_classifier install_training rebound."""
    import contextlib
    import io
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    from tests.conftest import load_golden
    g = load_golden("forest_cv.npz")
    mod = types.ModuleType("standin_forest_training")
    mod.evaluate_classifier = lambda *a, **k: "original"
    install_training(mod)
    try:
        for c in [str(x) for x in g["cases"]]:
            feats, kw = _golden_case(g, c)
            for fn in (at.evaluate_classifier, mod.evaluate_classifier):
                np.random.seed(int(g[c + "_seed"]))
                out = io.StringIO()
                with contextlib.redirect_stdout(out):
                    ret = fn(feats, kw["class_names"], kw["classifier_name"], kw["params"], kw["parameter_mode"],
                             list_of_ids=kw["list_of_ids"], n_exp=kw["n_exp"], train_percentage=kw["train_percentage"])
                assert out.getvalue() == str(g[c + "_stdout"]), c
                assert ret == int(g[c + "_ret"]), c
    finally:
        uninstall()


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
def test_cross_validate_512_features_32_classes_with_splits_missing_classes(kind):
    """forest_cross_validate at 512 features and 32 classes: one training set holds every class, the others miss some (the local class
    map runs short of kMaxClasses and the missing classes' test rows are counted against the present ones); problem by
    problem against scikit-learn."""
    from sklearn.preprocessing import StandardScaler
    from pyaudioanalysis_b200 import forests as FO
    from pyaudioanalysis_b200.consumers import forest_cross_validate
    r = np.random.RandomState(33)
    n = 384
    y = (np.arange(n) % 32).astype(np.float64)
    X = r.randn(n, 512) + 0.3 * (y[:, None] % 5 == np.arange(512) % 5)
    perm = r.permutation(n)
    splits = [(perm[:320], perm[320:])]
    for missing in ([0, 5, 31], list(range(16, 32))):
        keep = ~np.isin(y, missing)
        rows = r.permutation(np.flatnonzero(keep))
        splits.append((rows[:200], np.concatenate([rows[200:], np.flatnonzero(~keep)[:30]])))
    trees = [5, 4, 3]
    seeds = []
    for p, T in enumerate(trees):
        np.random.seed(60 + p)
        seeds.append(FO.tree_seeds(T, kind))
    pred, counts = forest_cross_validate(X, y, splits, seeds, trees, kind, n_classes=32)
    pred, counts = pred.cpu().numpy(), counts.cpu().numpy()
    off = 0
    for p, ((tr, te), T) in enumerate(zip(splits, trees)):
        sc = StandardScaler().fit(X[tr])
        np.random.seed(60 + p)
        m = _sklearn(kind)(n_estimators=T).fit(sc.transform(X[tr]), y[tr])
        want = m.predict(sc.transform(X[te])).astype(int)
        assert np.array_equal(pred[off:off + te.size], want), p
        c = np.zeros((32, 32), dtype=np.int64)
        np.add.at(c, (y[te].astype(int), want), 1)
        assert np.array_equal(counts[p], c), p
        off += te.size


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
def test_cross_validate_counts_against_sklearn_problem_by_problem(kind):
    """forest_cross_validate's predictions and counts equal scikit-learn run problem by problem: StandardScaler on the
    training rows, the forest's fit (drawing its seeds after the split's permutation) and predict on the test rows; the
    problems include training sets that miss a class and a problem whose trees take more than one scratch slice."""
    from sklearn.preprocessing import StandardScaler
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.consumers import forest_cross_validate
    r = np.random.RandomState(31)
    sizes = (60, 3, 50)
    X = np.vstack([r.randn(m, 9) + i * 0.4 for i, m in enumerate(sizes)])
    y = np.concatenate([np.full(m, i) for i, m in enumerate(sizes)]).astype(np.float64)
    params, n_exp = [3, 12], 4
    np.random.seed(77)
    splits, seeds = at.draw_forest_problems(X, params, n_exp, 0.9, kind)
    trees = [p for p in params for _ in range(n_exp)]
    pred, counts = forest_cross_validate(X, y, splits, seeds, trees, kind, n_classes=3)
    pred, counts = pred.cpu().numpy(), counts.cpu().numpy()
    np.random.seed(77)
    off = 0
    for p, (tr, te) in enumerate(splits):
        perm = np.random.permutation(X.shape[0])
        n_test = te.size
        assert np.array_equal(perm[:n_test], te) and np.array_equal(perm[n_test:], tr)
        sc = StandardScaler().fit(X[tr])
        m = _sklearn(kind)(n_estimators=trees[p]).fit(sc.transform(X[tr]), y[tr])
        want = m.predict(sc.transform(X[te])).astype(int)
        assert np.array_equal(pred[off:off + n_test], want), p
        c = np.zeros((3, 3), dtype=np.int64)
        np.add.at(c, (y[te].astype(int), want), 1)
        assert np.array_equal(counts[p], c), p
        off += n_test
    # one problem of 20 000 training rows and 130 trees: its forest is built and summed over several scratch slices
    rb = np.random.RandomState(32)
    Xb, yb = rb.randn(22000, 4), rb.randint(0, 3, 22000).astype(np.float64)
    tr, te = np.arange(20000), np.arange(20000, 22000)
    np.random.seed(5)
    s = __import__("pyaudioanalysis_b200.forests", fromlist=["tree_seeds"]).tree_seeds(130, kind)
    pb, _ = forest_cross_validate(Xb, yb, [(tr, te)], [s], [130], kind, n_classes=3)
    np.random.seed(5)
    sc = StandardScaler().fit(Xb[tr])
    m = _sklearn(kind)(n_estimators=130).fit(sc.transform(Xb[tr]), yb[tr])
    assert np.array_equal(pb.cpu().numpy(), m.predict(sc.transform(Xb[te])).astype(int))

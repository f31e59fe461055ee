"""CPU: the host pieces of the kNN cross-validation (kernel 6, pyaudioanalysis_b200/audioTrainTest.py) -- the scaler chain
and standardise step of csrc/knn_cv.cuh (run by tests/knn_cv_host.cu) against scikit-learn's StandardScaler bit for bit,
the up-front split draw against the reference's interleaved train_test_split calls, the confusion / macro-F1
restatements against scikit-learn, the printed report against the reference's own runs (tests/golden/knn_cv.npz), and
the C ABI's argument checks."""
import contextlib
import ctypes
import io

import numpy as np
import pytest
from sklearn.preprocessing import StandardScaler

from pyaudioanalysis_b200 import audioTrainTest as at
from tests import host_exe
from tests.host_exe import floats, hexes, run
from tests.conftest import load_golden
from tests.knn_cv_oracle import golden_args, golden_features, reference_splits, scores, seeded_features

INVALID = -1


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "knn_cv_host.cu", "-O1")


def _fit(exe, train, test):
    n, F = train.shape
    lines = run(exe, "fit %d %d %d %s %s\n" % (n, test.shape[0], F, hexes(train), hexes(test)))
    out = {t[0]: floats(t[1:]) for t in lines}
    return out["mean"], out["scale"], out["train"].reshape(n, F), out["test"].reshape(test.shape)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _scaler_cases():
    rng = np.random.default_rng(11)
    yield rng.normal(size=(108, 136)) * rng.choice([1e-3, 1.0, 1e4], size=136), rng.normal(size=(12, 136))
    const = rng.normal(size=(50, 7))
    const[:, 2] = 3.7                                               # constant columns
    const[:, 5] = 0.0
    yield const, rng.normal(size=(5, 7))
    near = 1e8 + rng.normal(size=(40, 4)) * np.array([1e-9, 1e-8, 1e-7, 1.0])    # near constant on a 1e8 offset
    yield near, 1e8 + rng.normal(size=(6, 4))
    neg0 = rng.normal(size=(9, 3))
    neg0[:, 0] = -0.0
    neg0[::2, 1] = -0.0
    yield neg0, np.array([[-0.0, -0.0, 0.0], [0.0, 1.0, -0.0]])
    yield rng.normal(size=(1, 5)), rng.normal(size=(3, 5))           # n = 1
    yield rng.normal(size=(2, 5)), rng.normal(size=(3, 5))           # n = 2
    yield np.array([[1.0, 2.0], [1.0, 2.0]]), np.array([[0.5, 2.5]])
    yield rng.normal(size=(4499, 6)) + 50.0, rng.normal(size=(4, 6))  # a long chain


def test_scaler_chain_matches_standard_scaler(exe):
    for train, test in _scaler_cases():
        mean, scale, tr, te = _fit(exe, train, test)
        sc = StandardScaler().fit(train)
        assert np.array_equal(_bits(mean), _bits(sc.mean_)), train.shape
        assert np.array_equal(_bits(scale), _bits(sc.scale_)), train.shape
        assert np.array_equal(_bits(tr), _bits(sc.transform(train))), train.shape
        assert np.array_equal(_bits(te), _bits(sc.transform(test))), train.shape


def test_split_draw_matches_interleaved_train_test_split():
    for n, tp, n_exp in ((120, 0.90, 5), (57, 0.90, 7), (120, 0.7, 3), (999, 0.9, 2), (33, 0.55, 4), (2, 0.5, 3)):
        np.random.seed(n)
        ref = reference_splits(n, 3, n_exp, tp)
        ref_state = np.random.get_state()
        np.random.seed(n)
        X = np.zeros((n, 2))
        got = at.draw_splits(X, np.zeros(n), 3, n_exp, tp)
        state = np.random.get_state()
        assert len(got) == len(ref) == 3 * n_exp
        for (a, b), (c, d) in zip(got, ref):
            assert np.array_equal(a, c) and np.array_equal(b, d), (n, tp)
        assert ref_state[0] == state[0] and np.array_equal(ref_state[1], state[1]) and ref_state[2:] == state[2:]


def test_group_split_draw_matches_group_shuffle_split():
    ids = [i // 5 for i in range(60)]
    np.random.seed(7)
    ref = reference_splits(60, 4, 6, list_of_ids=ids)
    np.random.seed(7)
    got = at.draw_splits(np.zeros((60, 3)), np.zeros(60), 4, 6, 0.9, ids)
    for (a, b), (c, d) in zip(got, ref):
        assert np.array_equal(a, c) and np.array_equal(b, d)


def test_scores_match_sklearn():
    """The confusion and macro-F1 restatements, with classes missing from y_test, y_pred or both."""
    rng = np.random.default_rng(5)
    for trial in range(400):
        C = int(rng.integers(2, 7))
        m = int(rng.integers(1, 15))
        present = rng.choice(C, size=int(rng.integers(1, C + 1)), replace=False)
        y_test = rng.choice(present, size=m).astype(np.float64)
        y_pred = [np.int64(v) for v in rng.choice(rng.choice(C, size=int(rng.integers(1, C + 1)), replace=False), size=m)]
        counts = np.zeros((C, C), dtype=np.int64)
        np.add.at(counts, (y_test.astype(np.int64), np.asarray(y_pred)), 1)
        cmt, f1t = at.experiment_scores(counts, set(np.arange(C, dtype=np.float64)))
        ref_cmt, ref_f1 = scores(y_test, y_pred)
        assert np.float64(f1t).view(np.uint64) == np.float64(ref_f1).view(np.uint64), trial
        labels = np.unique(np.concatenate([y_test, np.asarray(y_pred, dtype=np.float64)])).astype(np.int64)
        assert np.array_equal(cmt[np.ix_(labels, labels)], ref_cmt), trial
        if labels.size == C:
            assert np.array_equal(cmt, counts), trial


def test_report_reproduces_reference_output():
    """The host half of evaluate_classifier, fed each golden's own predictions, prints the reference's text and returns
    its choice."""
    g = load_golden("knn_cv.npz")
    for c in g["cases"]:
        feats = golden_features(g, c)
        class_names, params, mode, _, n_exp, _ = golden_args(g, c)
        X, y = at.features_to_matrix(feats)
        if n_exp == -1:
            n_exp = int(50000 / X.shape[0]) + 1
        ends = np.cumsum(g[c + "_exp_len"])
        C = len(feats)
        counts = np.zeros((len(ends), C, C), dtype=np.int64)
        for p, (a, b) in enumerate(zip(np.concatenate([[0], ends[:-1]]), ends)):
            np.add.at(counts[p], (g[c + "_y_test"][a:b].astype(np.int64), g[c + "_y_pred"][a:b].astype(np.int64)), 1)
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            ret = at.report(y, class_names, params, mode, n_exp, counts)
        assert out.getvalue() == str(g[c + "_stdout"]), c
        assert ret == g[c + "_ret"], c


def test_golden_scalers_match_standard_scaler():
    """The goldens' first scalers are StandardScaler fits of the rows the split draw gives (the draw and the fit the GPU
    path uses, tied to the reference's runs)."""
    g = load_golden("knn_cv.npz")
    for c in g["cases"]:
        feats = golden_features(g, c)
        class_names, params, mode, ids, n_exp, tp = golden_args(g, c)
        X, y = at.features_to_matrix(feats)
        if n_exp == -1:
            n_exp = int(50000 / X.shape[0]) + 1
        np.random.seed(int(g[c + "_seed"]))
        splits = at.draw_splits(X, y, len(params), n_exp, tp, ids)
        for e in range(g[c + "_mean"].shape[0]):
            sc = StandardScaler().fit(X[splits[e][0]])
            assert np.array_equal(sc.mean_, g[c + "_mean"][e]) and np.array_equal(sc.scale_, g[c + "_scale"][e]), (c, e)
        ends = np.cumsum(g[c + "_exp_len"])
        starts = np.concatenate([[0], ends[:-1]])
        for p, (tr, te) in enumerate(splits):
            assert np.array_equal(y[te], g[c + "_y_test"][starts[p]:ends[p]]), (c, p)


def test_unsupported_arguments():
    f = seeded_features(1, (5, 6), 3)
    params = np.array([1, 3])
    assert at.unsupported(f, "knn", params) is None
    assert at.unsupported(f, "svm", params)
    assert at.unsupported(f, "knn", params, smote=True)
    assert at.unsupported([f[0]], "knn", params)
    assert at.unsupported([f[0], f[1][:, :2]], "knn", params)
    assert at.unsupported([x[:, :1] for x in f], "knn", params)
    bad = [f[0].copy(), f[1]]
    bad[0][1, 1] = np.nan
    assert at.unsupported(bad, "knn", params)
    assert at.unsupported([f[0].astype(np.float32), f[1]], "knn", params)
    assert at.unsupported(f, "knn", np.array([0, 3]))
    assert at.unsupported(f, "knn", [1.5])
    assert at.unsupported(f, "knn", params, train_percentage=1.0)
    with pytest.raises(ValueError):
        at.evaluate_classifier(f, ["a", "b"], "svm", params, 1)


@pytest.fixture(scope="module")
def lib():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib.lib()


def test_cross_validate_rejects_bad_arguments(lib):
    p = 256                                    # never dereferenced: every call below fails its argument check first

    def arr(v, t):
        a = np.ascontiguousarray(v, dtype=t)
        keep.append(a)
        return ctypes.c_void_p(a.ctypes.data)

    keep = []

    def call(n=10, F=3, C=2, tr_off=(0, 3, 5), tr=(0, 1, 2, 3, 4), te_off=(0, 2, 4), te=(5, 6, 7, 8), k=(1, 3), cls=(2, 1),
             X=p, y=p, pred=p, counts=p, null=None):
        args = [X, y, n, F, C, len(k), arr(tr_off, np.int64), arr(tr, np.int32), arr(te_off, np.int64), arr(te, np.int32),
                arr(k, np.int64), arr(cls, np.int32), pred, counts, None]
        if null is not None:
            args[null] = None
        return lib.b200aa_knn_cross_validate(*args)

    for null in (0, 1, 6, 7, 8, 9, 10, 11, 12, 13):
        assert call(null=null) == INVALID, null
    assert call(n=0) == INVALID
    assert call(n=1 << 31) == INVALID
    assert call(F=0) == INVALID
    assert call(C=0) == INVALID
    assert call(tr_off=(1, 3, 5)) == INVALID                           # offsets not from 0
    assert call(te_off=(0, 0, 4)) == INVALID                           # an empty test list
    assert call(tr_off=(0, 3, 3)) == INVALID                           # an empty training list
    assert call(tr=(0, 1, 2, 3, 10)) == INVALID                        # index n
    assert call(te=(5, -1, 7, 8)) == INVALID
    assert call(k=(1, 0)) == INVALID
    assert call(cls=(2, 0)) == INVALID
    assert call(cls=(3, 1)) == INVALID                                 # more classes than n_classes
    assert lib.b200aa_knn_cross_validate(p, p, 10, 3, 2, -1, arr((0,), np.int64), arr((0,), np.int32), arr((0,), np.int64),
                                         arr((0,), np.int32), arr((1,), np.int64), arr((1,), np.int32), p, p, None) == INVALID
    # no problems: nothing to do, no CUDA call
    assert lib.b200aa_knn_cross_validate(p, p, 10, 3, 2, 0, arr((0,), np.int64), arr((0,), np.int32), arr((0,), np.int64),
                                         arr((0,), np.int32), arr((1,), np.int64), arr((1,), np.int32), p, p, None) == 0

"""GPU: the kNN cross-validation (b200aa_knn_cross_validate, consumers.knn_cross_validate, audioTrainTest.evaluate_classifier)
against the reference's own evaluate_classifier runs (tests/golden/knn_cv.npz: printed text, return value and every
experiment's predictions), kernel 5 on scikit-learn-standardised rows and the stable-sort oracle: mixed problem sizes in
one launch, a problem cut across scratch slices, k > n_train, duplicated rows under different labels, a non-default
stream, the install_training dispatcher and folders of generated WAV files."""
import contextlib
import io
import types

import numpy as np
import pytest
from sklearn.preprocessing import StandardScaler

from tests import knn_cv_oracle as oracle
from tests.conftest import load_golden
from tests.knn_cv_oracle import golden_args, golden_features

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import consumers
    return consumers


def _cv(C, X, y, splits, ks, n_classes=None):
    import torch
    pred, counts = C.knn_cross_validate(X, y, splits, ks, n_classes)
    torch.cuda.synchronize()
    assert pred.dtype == torch.int32 and counts.dtype == torch.int64 and pred.is_cuda and counts.is_cuda
    pred = pred.cpu().numpy()
    ends = np.cumsum([len(te) for _, te in splits])
    return np.split(pred, ends[:-1]), counts.cpu().numpy()


def _check(C, X, y, splits, ks, n_classes=None):
    """Predictions equal the stable-sort oracle per problem, and the counts are theirs."""
    got, counts = _cv(C, X, y, splits, ks, n_classes)
    ref = oracle.predict(X, y, splits, ks)
    for p, (a, b) in enumerate(zip(got, ref)):
        assert np.array_equal(a, b), p
    assert np.array_equal(counts, oracle.counts(y, splits, ref, counts.shape[1]))
    return got


def test_goldens_text_return_and_predictions(C):
    from pyaudioanalysis_b200 import audioTrainTest as at
    g = load_golden("knn_cv.npz")
    for c in g["cases"]:
        feats = golden_features(g, c)
        class_names, params, mode, ids, n_exp, tp = golden_args(g, c)
        np.random.seed(int(g[c + "_seed"]))
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            ret = at.evaluate_classifier(feats, class_names, "knn", params, mode, list_of_ids=ids, n_exp=n_exp,
                                         train_percentage=tp)
        assert out.getvalue() == str(g[c + "_stdout"]), c
        assert ret == g[c + "_ret"], c
        X, y = at.features_to_matrix(feats)
        n_exp = int(50000 / X.shape[0]) + 1 if n_exp == -1 else n_exp
        np.random.seed(int(g[c + "_seed"]))
        splits = at.draw_splits(X, y, len(params), n_exp, tp, ids)
        got, _ = _cv(C, X, y, splits, [int(k) for k in params for _ in range(n_exp)], len(feats))
        assert np.array_equal(np.concatenate(got), g[c + "_y_pred"]), c


def test_equals_kernel5_on_sklearn_standardised_rows(C):
    """Mixed problem sizes in one launch: each problem's predictions are knn_classify_batch's on StandardScaler rows."""
    import torch
    rng = np.random.default_rng(21)
    X = np.concatenate([rng.standard_normal((400, 24)) + 0.4 * i for i in range(4)])
    y = np.repeat(np.arange(4.0), 400)
    splits, ks = [], []
    for p in range(40):
        perm = rng.permutation(X.shape[0])
        n_tr = int(rng.integers(5, 1300))
        n_te = int(rng.integers(1, 300))
        splits.append((perm[:n_tr], perm[n_tr:n_tr + n_te]))
        ks.append(int(rng.choice([1, 2, 7, 15, 64])))
    got = _check(C, X, y, splits, ks)
    for (tr, te), k, pr in zip(splits, ks, got):
        sc = StandardScaler().fit(X[tr])
        model = types.SimpleNamespace(features=sc.transform(X[tr]), labels=y[tr], neighbors=k)
        ids, _ = C.knn_classify_batch(model, torch.from_numpy(sc.transform(X[te])).cuda())
        assert np.array_equal(ids.cpu().numpy(), pr)


def test_problem_larger_than_a_slice(C):
    """20 000 training rows x 2 000 test rows: 320 MB of keys, so the problem is cut by its test rows; small problems
    share the launches."""
    rng = np.random.default_rng(22)
    X = np.concatenate([rng.standard_normal((11000, 12)) + 0.3 * i for i in range(2)])
    y = np.repeat([0.0, 1.0], 11000)
    perm = rng.permutation(X.shape[0])
    splits = [(perm[:20000], perm[20000:]), (perm[:50], perm[50:60]), (perm[100:20100], perm[:3])]
    _check(C, X, y, splits, [13, 3, 1])


def test_k_above_n_train_and_missing_classes(C):
    rng = np.random.default_rng(23)
    X = rng.standard_normal((60, 5))
    y = np.repeat([0.0, 1.0, 2.0], 20)
    splits = [(np.arange(0, 8), np.arange(30, 40)),                   # class 0 only: C_p = 1
              (np.arange(20, 45), np.arange(0, 5)),                   # classes 1, 2: class 2 never votes (C_p = 2)
              (np.array([3, 41, 25]), np.arange(50, 60))]
    _check(C, X, y, splits, [50, 40, 3], 3)
    _check(C, X, y, splits, [1, 4, 2], 3)


def test_duplicate_rows_lower_split_position_wins(C):
    rng = np.random.default_rng(24)
    base = rng.standard_normal((30, 4))
    X = np.concatenate([base, base, base[:10]])
    y = np.concatenate([np.zeros(30), np.ones(30), np.full(10, 2.0)])
    splits, ks = [], []
    for p in range(12):
        perm = rng.permutation(70)
        splits.append((perm[:60], perm[60:]))
        ks.append(int(rng.choice([1, 2, 4])))
    splits.append((np.array([40, 10, 62, 2]), np.array([10, 40, 2])))
    ks.append(1)
    got = _check(C, X, y, splits, ks)
    assert got[-1].tolist() == [1, 1, 2]          # exact ties: the row earlier in the split's order votes


def test_non_default_stream(C):
    import torch
    rng = np.random.default_rng(25)
    X = rng.standard_normal((200, 10))
    y = rng.integers(0, 3, size=200).astype(np.float64)
    splits = [(rng.permutation(200)[:150], rng.permutation(200)[:30]) for _ in range(6)]
    ks = [1, 3, 5, 7, 9, 11]
    ref, ref_counts = _cv(C, X, y, splits, ks)
    s = torch.cuda.Stream()
    Xd = torch.from_numpy(X).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        pred, counts = C.knn_cross_validate(Xd, y, splits, ks)
        pred, counts = pred.cpu().numpy(), counts.cpu().numpy()
    assert np.array_equal(np.concatenate(ref), pred) and np.array_equal(ref_counts, counts)


def test_install_training_dispatcher(C):
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    calls = []

    def original(*a, **kw):
        calls.append((a[2], kw.get("smote")))
        return "original"

    mod = types.ModuleType("standin_audioTrainTest")
    mod.evaluate_classifier = original
    assert install_training(mod) == ["standin_audioTrainTest.evaluate_classifier"]
    try:
        feats = oracle.seeded_features(7, (20, 25, 15), 8)
        params = np.array([1, 3, 5])
        np.random.seed(3)
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            got = mod.evaluate_classifier(feats, ["a", "b", "c"], "knn", params, 1, n_exp=4)
        np.random.seed(3)
        ref_out = io.StringIO()
        with contextlib.redirect_stdout(ref_out):
            ref = at.evaluate_classifier(feats, ["a", "b", "c"], "knn", params, 1, n_exp=4)
        assert got == ref and out.getvalue() == ref_out.getvalue() and calls == []
        assert mod.evaluate_classifier(feats, ["a", "b", "c"], "svm", params, 1) == "original"
        assert mod.evaluate_classifier(feats, ["a", "b", "c"], "knn", params, 1, smote=True) == "original"
        bad = [feats[0].copy(), feats[1], feats[2]]
        bad[0][0, 0] = np.inf
        assert mod.evaluate_classifier(bad, ["a", "b", "c"], "knn", params, 1) == "original"
        assert calls == [("svm", False), ("knn", True), ("knn", False)]
    finally:
        uninstall()
    assert mod.evaluate_classifier is original


def test_generated_folders_through_feature_extraction(C, tmp_path):
    """WAV folders -> multiple_directory_feature_extraction -> evaluate_classifier, against the oracle loop on the same
    features and the same draws."""
    from tests import wavgen
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.MidTermFeatures import multiple_directory_feature_extraction
    dirs = []
    for c in range(3):
        d = tmp_path / ("class%d" % c)
        d.mkdir()
        for i in range(14):
            wavgen.write(str(d / ("f%02d.wav" % i)), 16000, wavgen.signal("s16", 1, 16000 + 977 * i, 300 * c + i), "s16")
        dirs.append(str(d))
    with contextlib.redirect_stdout(io.StringIO()):
        feats, names, _ = multiple_directory_feature_extraction(dirs, 0.5, 0.5, 0.05, 0.05)
    feats = [np.asarray(f, dtype=np.float64) for f in feats]
    params = np.array([1, 3, 5, 7, 9, 11, 13, 15])
    np.random.seed(9)
    with contextlib.redirect_stdout(io.StringIO()):
        ret = at.evaluate_classifier(feats, names, "knn", params, 1, n_exp=6)
    X, y = at.features_to_matrix(feats)
    np.random.seed(9)
    splits = oracle.reference_splits(X.shape[0], len(params), 6)
    ks = [int(k) for k in params for _ in range(6)]
    preds = oracle.predict(X, y, splits, ks)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        ref = at.report(y, names, params, 1, 6, oracle.counts(y, splits, preds, 3))
    assert ret == ref
    _check(C, X, y, splits, ks)

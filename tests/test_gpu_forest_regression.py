"""GPU: kernel 13's regression builder (b200aa_forest_regressor_fit, consumers.forest_regressor_fit) against
scikit-learn 1.9's RandomForestRegressor fit under the same NumPy global state: every tree's state in bits, the fitted
attributes and the global state afterwards, on the CPU harness's case bank, 100- and 500-tree forests, a forest
spanning several scratch slices, 512 features, bootstrapped roots near the team and padding edges and tied duplicated
columns; float32 / float64 device input; pickling and predict; concurrent streams and threads;
b200aa_forest_regression_cross_validate against scikit-learn problem by problem, in one launch, across launches and at
512 features; the scratch bound's refusal going to scikit-learn; evaluate_regression directly and through
install_training against the unmodified reference's output (tests/golden/forest_regression_cv.npz)."""
import contextlib
import io
import pickle
import threading
import types

import numpy as np
import pytest
import torch

from tests import forest_regression_cases as RC

pytestmark = pytest.mark.gpu


def _check(X, y, n_estimators, seed=5, X_in=None):
    from sklearn.ensemble import RandomForestRegressor
    from pyaudioanalysis_b200.consumers import forest_regressor_fit
    np.random.seed(seed)
    ref = RandomForestRegressor(n_estimators=n_estimators).fit(X, y)
    ref_state = np.random.get_state()
    np.random.seed(seed)
    got = forest_regressor_fit(X if X_in is None else X_in, y, n_estimators)
    assert RC.same_state(np.random.get_state(), ref_state)
    RC.compare(got, ref)
    return got, ref


@pytest.mark.parametrize("case", [c[0] for c in RC.problems()])
def test_case_bank_in_bits(case):
    _, X, y = next(c for c in RC.problems() if c[0] == case)
    _check(X, y, 4)


def test_512_features():
    """kMaxFeats: every per-feature array of forest_reg_build_kernel's shared memory runs full, and the batched sort
    holds 512 visits."""
    r = np.random.RandomState(61)
    X = r.randn(300, 512)
    _check(X, X[:, 7] - 0.5 * X[:, 300] + 0.1 * r.randn(300), 3)


@pytest.mark.parametrize("n", (127, 128, 129, 255, 256, 257, 1025))
def test_bootstrapped_roots_near_team_and_padding_edges(n):
    """n rows before the bootstrap's zero weights drop some (the root holds the positively weighted ones, about 0.63 n,
    so not exactly n: the regressor always bootstraps), on tied values, so that the introsort replay and the bitonic
    padding meet sizes around the team's edges."""
    r = np.random.RandomState(n)
    X = np.round(r.randn(n, 5), 1)
    _check(X, X[:, 0] + r.randint(0, 3, n), 3)


def test_tied_duplicated_columns():
    """Columns 6 .. 11 repeat 0 .. 5 with ties inside each: every visit's introsort replay starts from the order the
    previous visit left, and the first of two tied copies wins."""
    r = np.random.RandomState(62)
    X = np.round(r.randn(400, 6), 1)
    X = np.hstack([X, X])
    _check(X, X[:, 0] + 2 * X[:, 1] + r.randint(0, 2, 400), 4)


def test_100_and_500_trees():
    r = np.random.RandomState(41)
    X = r.randn(300, 11)
    y = 50.0 + X[:, 0] + r.randn(300) * 0.1
    _check(X, y, 100)
    _check(np.round(X, 1), np.round(y), 500, seed=6)


def test_several_scratch_slices():
    """2000 x 136 rows: each tree's sort keys take 136 x 2048 x 8 bytes, so 150 trees need two launches."""
    r = np.random.RandomState(43)
    X = r.randn(2000, 136)
    _check(X, X[:, 5] + r.randn(2000), 150)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_device_input(dtype):
    r = np.random.RandomState(44)
    X = r.randn(400, 9)
    y = r.randint(0, 5, 400).astype(np.float64)
    Xd = torch.from_numpy(X).to(dtype).cuda()
    _check(X.astype(np.float32).astype(np.float64) if dtype == torch.float32 else X, y, 6, X_in=Xd)


def test_pickle_and_predict():
    r = np.random.RandomState(45)
    X = r.randn(500, 12)
    y = X[:, 0] * 3 + r.randn(500)
    got, ref = _check(X, y, 20)
    back = pickle.loads(pickle.dumps(got))
    Q = r.randn(300, 12)
    for m in (got, back):
        assert np.array_equal(m.predict(Q).view(np.uint64), ref.predict(Q).view(np.uint64))


def test_streams_and_threads():
    """Fits on two threads, each on its own stream, equal the fits made one after another."""
    from pyaudioanalysis_b200.consumers import forest_regressor_fit
    r = np.random.RandomState(46)
    probs = [(r.randn(300, 7), r.randn(300)) for _ in range(4)]
    expected = []
    for i, (X, y) in enumerate(probs):
        np.random.seed(100 + i)
        expected.append(forest_regressor_fit(X, y, 8))
    # the NumPy global state is process-wide: draw under a lock, as the trainer draws before its launch
    got, errors, lock = [None] * 4, [], threading.Lock()

    def work(ids):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for i in ids:
                try:
                    with lock:
                        np.random.seed(100 + i)
                        got[i] = forest_regressor_fit(*probs[i], 8)
                except Exception as e:          # noqa: BLE001
                    errors.append(e)
    ts = [threading.Thread(target=work, args=(ids,)) for ids in ((0, 2), (1, 3))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for g, e in zip(got, expected):
        RC.compare(g, e)


def _cv_against_sklearn(X, y, params, n_exp, seed=9):
    """forest_regression_cross_validate's test and training predictions equal scikit-learn run problem by problem:
    StandardScaler on the whole matrix, the forest's fit on the training rows (its seeds drawn after the split's
    permutation) and predict, in bits."""
    from sklearn.ensemble import RandomForestRegressor
    from sklearn.preprocessing import StandardScaler
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.consumers import forest_regression_cross_validate
    np.random.seed(seed)
    splits, seeds = at.draw_regression_problems(X.shape[0], params, n_exp)
    trees = [C for C in params for _ in range(n_exp)]
    pte, ptr = forest_regression_cross_validate(X, y, splits, seeds, trees)
    pte, ptr = pte.cpu().numpy(), ptr.cpu().numpy()
    Xn = StandardScaler().fit_transform(X)
    np.random.seed(seed)
    o_te = o_tr = 0
    for p, ((tr, te), C) in enumerate(zip(splits, trees)):
        np.random.permutation(range(X.shape[0]))
        rf = RandomForestRegressor(n_estimators=C).fit(Xn[tr], y[tr])
        assert np.array_equal(pte[o_te:o_te + te.size].view(np.uint64), rf.predict(Xn[te]).view(np.uint64)), p
        assert np.array_equal(ptr[o_tr:o_tr + tr.size].view(np.uint64), rf.predict(Xn[tr]).view(np.uint64)), p
        o_te += te.size
        o_tr += tr.size


def test_cross_validate_one_launch_against_sklearn():
    """Small problems whose trees all go into one launch."""
    r = np.random.RandomState(47)
    _cv_against_sklearn(r.randn(120, 9), r.randn(120) + 10.0, [3, 11], 3)


def test_cross_validate_512_features():
    r = np.random.RandomState(63)
    X = r.randn(150, 512)
    _cv_against_sklearn(X, X[:, 3] + 0.2 * r.randn(150), [2, 3], 2)


def test_cross_validate_across_launches_against_sklearn():
    """Problems whose trees take several launches, one problem split across a launch boundary, on tie-heavy rows.

    900 x 136 rows train on 810: one tree's sort keys alone take 136 x pow2(810) x 8 = 1 114 112 bytes, so one 256 MB
    launch holds at most 240 trees, and [5, 150] x 2 = 310 trees take at least two.  A tree's whole scratch (keys,
    samples, replay arrays, stack, 1 619 nodes and values, weights) stays under 1.3 MB, so a launch holds more than 160
    trees: the fourth problem (trees 160-309) is split by the boundary.  That covers the sums carried from one launch to
    the next, the per-launch tree offsets, the walk that starts in the middle of a problem, the weight offsets of a
    problem's later trees and the division by T after the problem's last launch."""
    launch = 256 << 20
    keys = 136 * 1024 * 8
    assert 310 > launch // keys and launch // (13 * 10 ** 5) > 160
    r = np.random.RandomState(48)
    _cv_against_sklearn(np.round(r.randn(900, 136), 0), r.randint(1, 6, 900).astype(np.float64), [5, 150], 2)


def test_scratch_bound_goes_to_sklearn():
    """A regressor whose single tree would pass the 256 MB scratch bound (131 073 x 136 rows: 285 MB of sort keys) is
    refused by the GPU trainer before any draw it keeps: train_random_forest_regression gives scikit-learn's fit and
    leaves NumPy's global state as fit leaves it."""
    from sklearn.ensemble import RandomForestRegressor
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200 import forests as FO
    from pyaudioanalysis_b200.consumers import forest_regressor_fit
    r = np.random.RandomState(49)
    X = np.round(r.randn(131073, 136), 1).astype(np.float32)
    y = np.round(X[:, 0] * 2)
    np.random.seed(12)
    before = np.random.get_state()
    with pytest.raises(FO.Unsupported):
        forest_regressor_fit(X, y, 1)
    assert RC.same_state(np.random.get_state(), before)
    np.random.seed(12)
    ref = RandomForestRegressor(n_estimators=1).fit(X, y)
    ref_state = np.random.get_state()
    np.random.seed(12)
    rf, _ = at.train_random_forest_regression(X, y, 1)
    assert RC.same_state(np.random.get_state(), ref_state)
    RC.compare(rf, ref)


def test_train_random_forest_regression_drop_in():
    from sklearn.ensemble import RandomForestRegressor
    from pyaudioanalysis_b200 import audioTrainTest as at
    r = np.random.RandomState(48)
    X, y = r.randn(200, 6), r.randn(200)
    for Xi in (X, np.where(r.rand(200, 6) < 0.01, np.nan, X)):      # the second goes to scikit-learn (NaN)
        np.random.seed(3)
        rf, err = at.train_random_forest_regression(Xi, y, 12)
        np.random.seed(3)
        ref = RandomForestRegressor(n_estimators=12).fit(Xi, y)
        RC.compare(rf, ref)
        assert err == np.mean(np.abs(ref.predict(Xi) - y))


def test_evaluate_regression_goldens_directly_and_through_install_training():
    """The unmodified reference's evaluate_regression with its random forest (tests/golden/forest_regression_cv.npz):
    printed text and return value, from our evaluate_regression and from a module whose evaluate_regression
    install_training rebound (its svm methods still reach the original)."""
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    from tests.conftest import load_golden
    g = load_golden("forest_regression_cv.npz")
    mod = types.ModuleType("standin_regression_training")
    mod.evaluate_classifier = lambda *a, **k: None
    mod.evaluate_regression = lambda *a, **k: "original"
    install_training(mod)
    try:
        assert mod.evaluate_regression(g["a_X"], g["a_y"], 1, "svm_rbf", [1.0]) == "original"
        for c in [str(x) for x in g["cases"]]:
            params = [int(p) for p in g[c + "_params"]]
            for fn in (at.evaluate_regression, mod.evaluate_regression):
                np.random.seed(int(g[c + "_seed"]))
                out = io.StringIO()
                with contextlib.redirect_stdout(out):
                    ret = fn(g[c + "_X"], g[c + "_y"], int(g[c + "_n_exp"]), "randomforest", params)
                assert out.getvalue() == str(g[c + "_stdout"]), c
                assert np.array_equal(np.asarray(ret, dtype=np.float64).view(np.uint64), g[c + "_ret"].view(np.uint64)), c
    finally:
        uninstall()

"""GPU: kernel 13's gradient boosting (b200aa_boosting_stage, consumers.boosting_fit and boosting_cross_validate) against
scikit-learn 1.9's GradientBoostingClassifier fit under the same NumPy global state: every tree in bits, train_score_,
init_, classes_, the predictions and the global state afterwards, on the CPU harness's case bank, 100 and 500 stages,
stages spanning several scratch slices, 32 classes at 512 features and root sizes on the team and padding edges; float32 / float64 device input; pickling; kernel 8 on the GPU-trained model;
concurrent streams and threads; the batched model selection against scikit-learn problem by problem, in one launch,
across launches and at 32 classes; the scratch bound's refusal going to scikit-learn; evaluate_classifier directly and through
install_training against the unmodified reference's output (tests/golden/boosting_cv.npz); the final fit of
extract_features_and_train through the rebound train_gradient_boosting."""
import contextlib
import io
import pickle
import threading
import types

import numpy as np
import pytest
import torch

from tests import boosting_cases as BC

pytestmark = pytest.mark.gpu


def _check(X, y, T, seed=7, X_in=None):
    from sklearn.ensemble import GradientBoostingClassifier
    from pyaudioanalysis_b200.consumers import boosting_fit
    np.random.seed(seed)
    ref = GradientBoostingClassifier(n_estimators=T).fit(X, y)
    ref_state = np.random.get_state()
    np.random.seed(seed)
    got = boosting_fit(X if X_in is None else X_in, y, T)
    assert BC.same_state(np.random.get_state(), ref_state)
    BC.compare(got, ref, BC.held_out(X))
    return got, ref


@pytest.mark.parametrize("case", [c[0] for c in BC.problems()])
def test_case_bank_in_bits(case):
    _, X, y, T = next(c for c in BC.problems() if c[0] == case)
    _check(X, y, T)


def _limits(seed, n):
    """n rows of 512 features and 32 classes (kMaxFeats, kMaxClasses: 32 trees per stage), each class present at least
    twice"""
    r = np.random.RandomState(seed)
    y = r.permutation(np.arange(n) % 32)
    X = r.randn(n, 512)
    X[:, :32] += 1.5 * (y[:, None] == np.arange(32))
    return X, y


def test_32_classes_512_features():
    X, y = _limits(71, 160)
    got, _ = _check(X, y, 3)
    assert got.n_trees_per_iteration_ == 32


@pytest.mark.parametrize("n", (127, 128, 129, 255, 256, 257, 1025))
def test_root_sizes_at_team_and_padding_edges(n):
    """Unit-weight roots of exactly n rows: one row per thread and one over, and the bitonic sort's padding."""
    r = np.random.RandomState(n)
    X = np.round(r.randn(n, 4), 1)
    _check(X, (X[:, 0] + 0.5 * r.randn(n) > 0).astype(int) + (X[:, 1] > 0.8), 3)


def test_100_and_500_stages():
    r = np.random.RandomState(41)
    X = r.randn(200, 8)
    _check(X, np.argmax(X[:, :3] + r.randn(200, 3), 1), 100)
    X = np.round(r.randn(150, 5), 1)
    _check(X, (X[:, 0] + r.randn(150) > 0).astype(int), 500, seed=6)


def test_stage_over_several_scratch_slices():
    """17 000 x 136 rows, 10 classes: each tree's sort keys take 136 x 32 768 x 8 bytes (35.7 MB), so a 256 MB launch
    holds at most 7 trees and each stage's 10 trees take two launches."""
    assert 256 * 2 ** 20 // (136 * 32768 * 8) == 7
    r = np.random.RandomState(43)
    X = r.randn(17000, 136)
    _check(X, r.randint(0, 10, 17000), 2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_device_input(dtype):
    r = np.random.RandomState(44)
    X = r.randn(300, 9)
    y = r.randint(0, 4, 300)
    Xd = torch.from_numpy(X).to(dtype).cuda()
    _check(X.astype(np.float32).astype(np.float64) if dtype == torch.float32 else X, y, 8, X_in=Xd)


def test_pickle_and_kernel8():
    """A pickle round trip keeps the predictions; kernel 8's TreeEnsembleModel on the GPU-trained model equals it on
    scikit-learn's."""
    from pyaudioanalysis_b200.consumers import tree_classify_batch
    r = np.random.RandomState(45)
    X = r.randn(400, 12)
    got, ref = _check(X, np.argmax(X[:, :4] + r.randn(400, 4), 1), 20)
    back = pickle.loads(pickle.dumps(got))
    Q = r.randn(300, 12)
    assert np.array_equal(back.predict_proba(Q).view(np.uint64), ref.predict_proba(Q).view(np.uint64))
    Qd = torch.from_numpy(Q).cuda()
    ids_g, P_g = tree_classify_batch(got, Qd)
    ids_r, P_r = tree_classify_batch(ref, Qd)
    assert torch.equal(ids_g, ids_r) and torch.equal(P_g.view(torch.int64), P_r.view(torch.int64))


def test_streams_and_threads():
    """Fits on two threads, each on its own stream, equal the fits made one after another."""
    from pyaudioanalysis_b200.consumers import boosting_fit
    r = np.random.RandomState(46)
    probs = [(r.randn(200, 7), r.randint(0, 3, 200)) for _ in range(4)]
    expected = []
    for i, (X, y) in enumerate(probs):
        np.random.seed(100 + i)
        expected.append(boosting_fit(X, y, 6))
    got, errors, lock = [None] * 4, [], threading.Lock()

    def work(ids):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for i in ids:
                try:
                    with lock:                      # the NumPy global state is process-wide
                        np.random.seed(100 + i)
                        got[i] = boosting_fit(*probs[i], 6)
                except Exception as e:          # noqa: BLE001
                    errors.append(e)
    ts = [threading.Thread(target=work, args=(ids,)) for ids in ((0, 2), (1, 3))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for g, e, (X, _) in zip(got, expected, probs):
        BC.compare(g, e, BC.held_out(X))


def _cv_against_sklearn(X, y, params, n_exp, seed=9, tp=0.9):
    """boosting_cross_validate's predictions and counts equal scikit-learn run problem by problem: StandardScaler fit on
    the training rows, GradientBoostingClassifier's fit on them (its seeds drawn after the split's permutation) and
    predict of the test rows."""
    from sklearn.ensemble import GradientBoostingClassifier
    from sklearn.preprocessing import StandardScaler
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.consumers import boosting_cross_validate
    np.random.seed(seed)
    splits, seeds = at.draw_boosting_problems(X, y, params, n_exp, tp)
    stages = [C for C in params for _ in range(n_exp)]
    pred, counts = boosting_cross_validate(X, y, splits, seeds, stages)
    pred, counts = pred.cpu().numpy(), counts.cpu().numpy()
    np.random.seed(seed)
    o = 0
    C = int(y.max()) + 1
    for p, ((tr, te), T) in enumerate(zip(splits, stages)):
        np.random.permutation(X.shape[0])          # the split's draw, then the fit's
        sc = StandardScaler().fit(X[tr])
        m = GradientBoostingClassifier(n_estimators=T).fit(sc.transform(X[tr]), y[tr])
        ref = m.predict(sc.transform(X[te]))
        assert np.array_equal(pred[o:o + te.size], ref.astype(np.int32)), p
        want = np.zeros((C, C), np.int64)
        np.add.at(want, (y[te].astype(int), ref.astype(int)), 1)
        assert np.array_equal(counts[p], want), p
        o += te.size


def test_cross_validate_one_launch_against_sklearn():
    """Small problems, binary and 3-class ones, every stage's trees in one launch; some training sets miss a class."""
    r = np.random.RandomState(47)
    X = r.randn(90, 6)
    y = np.concatenate([np.zeros(50), np.ones(38), 2 * np.ones(2)])
    _cv_against_sklearn(X, y, [3, 7], 4, tp=0.7)


def test_cross_validate_32_classes_512_features():
    """Every training set holds all 32 classes: 32 trees per stage and the count kernel's full class table."""
    X, y = _limits(72, 192)
    _cv_against_sklearn(X, y.astype(np.float64), [2], 2, tp=0.85)


def test_cross_validate_across_launches_against_sklearn():
    """2 000 x 136 rows training on 1 800: one tree's sort keys take 136 x 2 048 x 8 bytes (2.2 MB), so a 256 MB launch
    holds at most 120 trees, and [2, 3] x 20 = 40 problems of 4 classes grow 160 trees a stage: two launches per stage,
    and in the third stage only the 20 three-stage problems remain."""
    assert 256 * 2 ** 20 // (136 * 2048 * 8) == 120
    r = np.random.RandomState(48)
    X = np.round(r.randn(2000, 136), 1)
    y = np.argmax(X[:, :4] + r.randn(2000, 4), 1).astype(np.float64)
    _cv_against_sklearn(X, y, [2, 3], 20)


def test_scratch_bound_goes_to_sklearn():
    """A fit whose single tree would pass the 256 MB scratch bound (131 073 x 136 rows) is refused before any draw it
    keeps: train_gradient_boosting gives scikit-learn's fit from the same state."""
    from sklearn.ensemble import GradientBoostingClassifier
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200 import forests as FO
    from pyaudioanalysis_b200.consumers import boosting_fit
    r = np.random.RandomState(49)
    X = np.round(r.randn(131073, 136), 1).astype(np.float32)
    y = (X[:, 0] > 0).astype(int)
    np.random.seed(12)
    before = np.random.get_state()
    with pytest.raises(FO.Unsupported):
        boosting_fit(X, y, 1)
    assert BC.same_state(np.random.get_state(), before)
    np.random.seed(12)
    ref = GradientBoostingClassifier(n_estimators=1).fit(X, y)
    np.random.seed(12)
    got = at.train_gradient_boosting(X, y, 1)
    BC.compare(got, ref, X[:50])


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
    """The unmodified reference's evaluate_classifier with gradient boosting (tests/golden/boosting_cv.npz): printed
    text and return value, from our evaluate_classifier and from a module whose evaluate_classifier install_training
    rebound."""
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    from tests.conftest import load_golden
    g = load_golden("boosting_cv.npz")
    mod = types.ModuleType("standin_boosting_training")
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


def test_final_fit_through_rebound_train_gradient_boosting():
    """extract_features_and_train's last step: the selected stage count fitted on the scaled features of every class
    through the module's train_gradient_boosting, which install_training rebound; equal to scikit-learn's fit."""
    from sklearn.ensemble import GradientBoostingClassifier
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    mod = types.ModuleType("standin_final_fit")
    mod.evaluate_classifier = lambda *a, **k: None
    mod.train_gradient_boosting = lambda *a: "original"
    r = np.random.RandomState(50)
    feats = [r.randn(60, 10) + i for i in range(3)]
    X, y = at.features_to_matrix(feats)
    Xn = (X - X.mean(0)) / X.std(0)
    install_training(mod)
    try:
        np.random.seed(13)
        got = mod.train_gradient_boosting(Xn, y, 10)
    finally:
        uninstall()
    np.random.seed(13)
    ref = GradientBoostingClassifier(n_estimators=10).fit(Xn, y)
    BC.compare(got, ref, BC.held_out(Xn))


def test_scale_accepts_a_training_split_longer_than_X():
    """b200aa_boosting_scale accepts a training split of more rows than X has (repeated rows), as the stage does, and
    standardises both splits with the training rows' StandardScaler fit."""
    import ctypes
    from sklearn.preprocessing import StandardScaler
    from pyaudioanalysis_b200 import _lib as L
    r = np.random.RandomState(4)
    X = r.randn(6, 3)
    tr, te = np.array([0, 1, 2, 3, 4, 5, 0, 1], np.int32), np.array([4, 5], np.int32)
    tro, teo = np.array([0, tr.size], np.int64), np.array([0, te.size], np.int64)
    d_X = torch.from_numpy(X).cuda()
    out = torch.empty((tr.size + te.size, 3), dtype=torch.float32, device="cuda")

    def p(a):
        return ctypes.c_void_p(a.ctypes.data)
    assert L.lib().b200aa_boosting_scale(ctypes.c_void_p(d_X.data_ptr()), 6, 3, 1, p(tro), p(tr), p(teo), p(te),
                                         ctypes.c_void_p(out.data_ptr()), None) == L.OK
    torch.cuda.synchronize()
    sc = StandardScaler().fit(X[tr])
    want = np.concatenate([sc.transform(X[tr]), sc.transform(X[te])]).astype(np.float32)
    np.testing.assert_allclose(out.cpu().numpy(), want, rtol=1e-6, atol=1e-6)

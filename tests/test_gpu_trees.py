"""GPU: the tree-ensemble kernel (b200aa_trees_classify, consumers.tree_classify_batch) bit for bit scikit-learn's predict /
predict_proba on the rows the kernel read: float32, float64 and strided views, n = 0, 1, 65 536 and 600 000, a 500-tree
forest and deep extra trees; refused rows; classify_vectors / mid_term_classification against the host path and the
reference's per-window loop; unsupported models on the host path; streams and threads sharing one model."""
import threading

import numpy as np
import pytest

from tests import tree_models as TM

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import consumers
    return consumers


@pytest.fixture(scope="module")
def models():
    return TM.models()


def _ref(model, X):
    return model.predict(X), model.predict_proba(X)


def _gpu(C, model, t):
    import torch
    m = model if isinstance(model, C.TreeEnsembleModel) else C.TreeEnsembleModel(model)
    ids, P = C.tree_classify_batch(m, t)
    torch.cuda.synchronize()
    assert ids.dtype == torch.int64 and P.dtype == torch.float64 and ids.is_cuda and P.is_cuda
    return m.classes[ids.cpu().numpy()], P.cpu().numpy()


def _same(got, ref, what):
    assert np.array_equal(got[0], ref[0]), what
    assert np.array_equal(got[1], ref[1]), what


@pytest.mark.parametrize("name", ["rf4", "et4", "gb4", "rf2", "gb2", "gb2_zero", "rf1", "rf500", "labels_257", "labels_str",
                                  "labels_str_et", "one_leaf", "stump_leaf", "tie", "rf_nan", "et_nan", "rf40",
                                  "gb40", "tie40"])
def test_query_bank_float64_float32_strided(C, models, name):
    import torch
    model = models[name]
    X = TM.query_bank(model, seed=5, nan=name in ("rf_nan", "et_nan"))
    t = torch.from_numpy(X).cuda()
    _same(_gpu(C, model, t), _ref(model, X), name)
    _same(_gpu(C, model, t.float()), _ref(model, X.astype(np.float32)), name + " float32")
    wide = torch.zeros((X.shape[0], X.shape[1] + 7), dtype=torch.float64, device="cuda")
    wide[:, 3:3 + X.shape[1]] = t
    _same(_gpu(C, model, wide[:, 3:3 + X.shape[1]]), _ref(model, X), name + " row stride")
    _same(_gpu(C, model, t[::3]), _ref(model, X[::3]), name + " every third row")
    _same(_gpu(C, model, t.t().contiguous().t()), _ref(model, X), name + " column-major")


def test_sizes_0_1_65536_600000(C, models):
    import torch
    model = C.TreeEnsembleModel(models["et4"])
    ids, P = C.tree_classify_batch(model, torch.zeros((0, TM.F), dtype=torch.float64, device="cuda"))
    assert ids.shape == (0,) and P.shape == (0, 4)
    rng = np.random.default_rng(7)
    for n in (1, 65536, 600000):
        X = (rng.normal(size=(n, TM.F)) * 1.5).astype(np.float32)
        _same(_gpu(C, model, torch.from_numpy(X).cuda()), _ref(models["et4"], X), n)


def test_large_models(C):
    """A 500-tree forest and fully grown extra trees on 4 000 x 136 rows, as the library trains them."""
    import torch
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    rng = np.random.default_rng(8)
    y = rng.integers(0, 4, size=4000)
    X = rng.normal(size=(4000, 136)) + 0.3 * y[:, None] * rng.normal(size=136)[None, :]
    Q = rng.normal(size=(20000, 136)) + 0.3 * rng.integers(0, 4, size=20000)[:, None] * rng.normal(size=136)[None, :]
    for m in (RandomForestClassifier(500, random_state=0).fit(X, y), ExtraTreesClassifier(100, random_state=1).fit(X, y)):
        _same(_gpu(C, m, torch.from_numpy(Q).cuda()), _ref(m, Q), type(m).__name__)


def test_refused_rows_raise_sklearns_error(C, models):
    import torch
    for name in ("rf4", "gb4", "gb2"):
        model = models[name]
        base = TM.query_bank(model, seed=6)[:100]
        for r in TM.refused_rows():
            X = base.copy()
            X[57] = r
            with pytest.raises(ValueError) as got:
                C.tree_classify_batch(C.TreeEnsembleModel(model), torch.from_numpy(X).cuda())
            with pytest.raises(ValueError) as ref:
                model.predict(X)
            assert str(got.value) == str(ref.value), name
    X = TM.query_bank(models["gb4"], seed=6)[:100]
    X[9, 4] = np.nan
    with pytest.raises(ValueError) as got:
        C.tree_classify_batch(C.TreeEnsembleModel(models["gb4"]), torch.from_numpy(X).cuda())
    with pytest.raises(ValueError) as ref:
        models["gb4"].predict(X)
    assert str(got.value) == str(ref.value)


def test_classify_vectors_equals_host_path(C, models):
    import torch
    rng = np.random.default_rng(9)
    v = torch.from_numpy(rng.normal(size=(3000, TM.F)).astype(np.float32)).cuda()
    for mtype, name in (("randomforest", "rf4"), ("extratrees", "et4"), ("gradientboosting", "gb4"),
                        ("gradientboosting", "labels_str"), ("randomforest", "labels_257")):
        model = models[name]
        host = C.classify_vectors(model, mtype, v.cpu().numpy())
        for clf in (model, C.TreeEnsembleModel(model)):
            got = C.classify_vectors(clf, mtype, v)
            assert np.array_equal(got[0], host[0]) and np.array_equal(got[1], host[1]), (mtype, name)


def test_unsupported_models_take_the_host_path(C):
    import torch
    from sklearn.dummy import DummyClassifier
    from sklearn.ensemble import GradientBoostingClassifier, RandomForestClassifier
    from sklearn.svm import SVC
    X, y = TM.dataset(n=200)
    v = torch.from_numpy(TM.dataset(n=50, seed=3)[0]).cuda()
    cases = [("svm", SVC(probability=True, random_state=0).fit(X, y)),
             ("gradientboosting", GradientBoostingClassifier(n_estimators=5, init=DummyClassifier(strategy="most_frequent")).fit(X, y)),
             ("randomforest", RandomForestClassifier(5, random_state=0).fit(X, np.stack([y, 3 - y], axis=1)))]
    for mtype, model in cases:
        with pytest.raises(ValueError):
            C.TreeEnsembleModel(model)
        host = C.classify_vectors(model, mtype, v.cpu().numpy())
        got = C.classify_vectors(model, mtype, v)
        for a, b in zip(got, host):
            assert np.array_equal(np.asarray(a), np.asarray(b)), mtype


def test_errors(C, models):
    import torch
    model = C.TreeEnsembleModel(models["rf4"])
    with pytest.raises(TypeError):
        C.tree_classify_batch(model, torch.zeros((2, TM.F), dtype=torch.float64))
    with pytest.raises(ValueError):
        C.tree_classify_batch(model, torch.zeros((2, TM.F + 1), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        C.tree_classify_batch(model, torch.zeros((2, TM.F), dtype=torch.int32, device="cuda"))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            C.tree_classify_batch(model, torch.zeros((2, TM.F), dtype=torch.float64, device="cuda:1"))
    from pyaudioanalysis_b200._lib import ERR_INVALID, lib
    q = torch.zeros((2, TM.F), dtype=torch.float64, device="cuda")
    ids = torch.empty(2, dtype=torch.int64, device="cuda")
    P = torch.empty((2, 4), dtype=torch.float64, device="cuda")
    bad = torch.empty(2, dtype=torch.int32, device="cuda")
    good = [model.handle, q.data_ptr(), 2, 2, TM.F, TM.F, ids.data_ptr(), P.data_ptr(), bad.data_ptr(), None]
    assert lib().b200aa_trees_classify(*good) == 0
    for i, v in ((0, None), (1, None), (6, None), (7, None), (8, None), (2, 0), (2, 3), (3, -1), (4, TM.F + 1), (5, TM.F - 1)):
        args = list(good)
        args[i] = v
        assert lib().b200aa_trees_classify(*args) == ERR_INVALID, (i, v)
    args = list(good)
    args[3] = 0
    assert lib().b200aa_trees_classify(*args) == 0


def test_streams_and_threads_share_one_model(C, models):
    import torch
    rng = np.random.default_rng(10)
    model = C.TreeEnsembleModel(models["rf500"])
    qs = [torch.from_numpy(rng.normal(size=(5000, TM.F))).cuda() for _ in range(4)]
    alone = []
    for q in qs:
        ids, P = C.tree_classify_batch(model, q)
        alone.append((ids.cpu().numpy(), P.cpu().numpy()))
    streams = [torch.cuda.Stream() for _ in range(2)]
    out = [None] * 4
    for i, q in enumerate(qs):
        with torch.cuda.stream(streams[i % 2]):
            out[i] = C.tree_classify_batch(model, q)
    torch.cuda.synchronize()
    for i in range(4):
        _same((out[i][0].cpu().numpy(), out[i][1].cpu().numpy()), alone[i], "stream %d" % i)
    res, errs = [None] * 4, []

    def work(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                ids, P = C.tree_classify_batch(model, qs[i])
                torch.cuda.current_stream().synchronize()
                res[i] = (ids.cpu().numpy(), P.cpu().numpy())
        except Exception as e:                                  # pragma: no cover - reported below
            errs.append(e)

    for rnd in range(2):
        th = [threading.Thread(target=work, args=(2 * rnd + j,)) for j in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
    assert not errs, errs
    for i in range(4):
        _same(res[i], alone[i], "thread %d" % i)


def test_model_built_and_used_on_a_side_stream(C, models):
    """The upload is complete when the model is made: a model built under a fresh stream and used there at once (as
    classify_vectors does with a plain estimator) gives the default stream's results."""
    import torch
    rng = np.random.default_rng(11)
    v = torch.from_numpy(rng.normal(size=(20000, TM.F))).cuda()
    for mtype, name in (("randomforest", "rf500"), ("extratrees", "et4"), ("gradientboosting", "gb40")):
        model = models[name]
        ref = _ref(model, v.cpu().numpy())
        for _ in range(3):
            with torch.cuda.stream(torch.cuda.Stream()):
                got = C.classify_vectors(model, mtype, v)
                m = C.TreeEnsembleModel(model)
                ids, P = C.tree_classify_batch(m, v)
                torch.cuda.current_stream().synchronize()
            _same(got, ref, name)
            _same((m.classes[ids.cpu().numpy()], P.cpu().numpy()), ref, name)


def _signal(fs):
    rng = np.random.default_rng(21)
    t = np.arange(8 * fs)
    x = np.concatenate([rng.normal(0, 3000, 8 * fs), 9000 * np.sin(2 * np.pi * 440 * t / fs) + rng.normal(0, 300, 8 * fs),
                        4000 * np.sign(np.sin(2 * np.pi * 3 * t / fs)) * rng.normal(1, 0.2, 8 * fs)])
    return np.round(np.clip(x, -32768, 32767)).astype(np.int16)


def test_mid_term_classification_matches_host_and_reference_loop(C):
    """Models trained on this signal's own mid-term windows: mid_term_classification on the device equals the host path on
    the same normalised vectors, and a sample of windows equals classifier_wrapper's one-row predict / predict_proba."""
    import torch
    from sklearn.ensemble import ExtraTreesClassifier, GradientBoostingClassifier, RandomForestClassifier
    from pyaudioanalysis_b200.batch import mid_feature_extraction_batch
    fs, mt, step, st = 16000, 1.0, 0.1, 0.05
    x = _signal(fs)
    mid, _ = mid_feature_extraction_batch(torch.from_numpy(x).cuda().reshape(1, -1), fs, mt * fs, step * fs, round(fs * st),
                                          round(fs * st))
    feats = mid[0].double().cpu().numpy().T
    mean, std = feats.mean(axis=0), feats.std(axis=0) + 1e-8
    y = np.arange(feats.shape[0]) * 3 // feats.shape[0]
    Xn = (feats - mean) / std
    for mtype, model in (("randomforest", RandomForestClassifier(50, random_state=0).fit(Xn, y)),
                         ("extratrees", ExtraTreesClassifier(50, random_state=1).fit(Xn, y)),
                         ("gradientboosting", GradientBoostingClassifier(n_estimators=30, random_state=2).fit(Xn, y))):
        vec = C.normalize_windows_batch(mid[0:1].contiguous(), mean, std)[0]
        host_ids, host_P = C.classify_vectors(model, mtype, vec.cpu().numpy())
        ids, post = C.mid_term_classification(x, fs, model, mtype, mean, std, mt, step, st, st)
        assert np.array_equal(ids, host_ids), mtype
        assert np.array_equal(post, np.max(host_P, axis=1)), mtype
        v = vec.double().cpu().numpy()
        for j in range(0, v.shape[0], 17):                     # audioTrainTest.classifier_wrapper, one row at a time
            assert ids[j] == model.predict(v[j].reshape(1, -1))[0], (mtype, j)
            assert post[j] == np.max(model.predict_proba(v[j].reshape(1, -1))[0]), (mtype, j)

"""GPU: the kNN kernel (b200aa_knn_classify, consumers.knn_classify_batch) bit for bit against the reference's Knn.classify
(tests/golden/knn.npz) and the stable-sort oracle, across scratch slices, ties, NaN / inf, strides, concurrency, and through
mid_term_classification."""
import threading
import types

import numpy as np
import pytest

from tests.conftest import load_golden
from tests.knn_oracle import knn_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import consumers
    return consumers


def _model(feats, labels, k):
    return types.SimpleNamespace(features=feats, labels=labels, neighbors=k)


def _run(C, model, x, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    if dtype is not None:
        t = t.to(dtype)
    ids, P = C.knn_classify_batch(model, t)
    torch.cuda.synchronize()
    assert ids.dtype == torch.int64 and P.dtype == torch.float64 and ids.is_cuda and P.is_cuda
    return ids.cpu().numpy(), P.cpu().numpy()


def _same(got, ref, what):
    assert np.array_equal(got[0], ref[0]), what
    assert np.array_equal(got[1], ref[1]), what


def test_golden_float64_and_float32(C):
    g = load_golden("knn.npz")
    for c in g["cases"]:
        feats, labels, k, q = g[c + "_features"], g[c + "_labels"], int(g[c + "_k"]), g[c + "_queries"]
        model = C.KnnModel(_model(feats, labels, k))
        _same(_run(C, model, q), (g[c + "_ids"], g[c + "_P"]), c)
        q32 = q.astype(np.float32)
        _same(_run(C, model, q32), knn_oracle(feats, labels, k, q32.astype(np.float64)), c + " float32")


def test_many_slices_against_stable_oracle(C):
    """N = 20 000: 1 677 queries fill the 256 MiB of keys, so 4 000 queries take three slices."""
    from scipy.spatial.distance import cdist
    rng = np.random.default_rng(17)
    N, F, n = 20000, 136, 4000
    feats = rng.normal(size=(N, F))
    labels = rng.integers(0, 5, size=N).astype(np.float64)
    feats += labels[:, None] * 0.05
    q = rng.normal(size=(n, F))
    order = np.concatenate([np.argsort(cdist(q[a:a + 250], feats), axis=1, kind="stable") for a in range(0, n, 250)])
    for k in (1, 13, 64, N, N + 7):
        near = labels[order[:, :k]]
        P = np.stack([(near == i).sum(axis=1) / float(k) for i in range(5)], axis=1)
        _same(_run(C, C.KnnModel(_model(feats, labels, k)), q), (np.argmax(P, axis=1), P), k)


def test_ties_nan_inf_and_empty(C):
    import torch
    rng = np.random.default_rng(18)
    grid = rng.integers(0, 3, size=(60, 3)).astype(np.float64)               # exact ties across labels everywhere
    labels = rng.integers(0, 3, size=60).astype(np.float64)
    q = rng.integers(0, 3, size=(30, 3)).astype(np.float64)
    q[0, 0], q[1, 1], q[2, 2] = np.nan, np.inf, -np.inf
    tr = grid.copy()
    tr[[4, 9], 1] = np.nan
    tr[5, 0] = np.inf
    for feats in (grid, tr):
        for k in (1, 2, 7, 59, 60, 67):
            _same(_run(C, C.KnnModel(_model(feats, labels, k)), q), knn_oracle(feats, labels, k, q), k)
    ids, P = C.knn_classify_batch(C.KnnModel(_model(grid, labels, 3)), torch.zeros((0, 3), dtype=torch.float64, device="cuda"))
    assert ids.shape == (0,) and P.shape == (0, 3)


def test_strided_rows(C):
    import torch
    rng = np.random.default_rng(19)
    feats, labels = rng.normal(size=(300, 20)), rng.integers(0, 4, size=300).astype(np.float64)
    model = C.KnnModel(_model(feats, labels, 9))
    wide = torch.from_numpy(rng.normal(size=(50, 33))).cuda()
    for t in (wide[:, 5:25], wide[::2, :20], wide[:, :20].float(), wide[:, 5:25].t().contiguous().t()):
        ids, P = C.knn_classify_batch(model, t)
        _same((ids.cpu().numpy(), P.cpu().numpy()), knn_oracle(feats, labels, 9, t.double().cpu().numpy()), tuple(t.stride()))


def test_errors(C):
    import torch
    from pyaudioanalysis_b200._lib import ERR_INVALID, lib
    feats, labels = np.zeros((4, 3)), np.zeros(4)
    model = C.KnnModel(_model(feats, labels, 1))
    with pytest.raises(TypeError):
        C.knn_classify_batch(model, torch.zeros((2, 3), dtype=torch.float64))
    with pytest.raises(ValueError):
        C.knn_classify_batch(model, torch.zeros((2, 4), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        C.knn_classify_batch(model, torch.zeros((2, 3), dtype=torch.int32, device="cuda"))
    for bad in (_model(feats, labels, 0), _model(feats, labels, -2), _model(np.zeros((0, 3)), np.zeros(0), 1),
                _model(feats, np.zeros(3), 1)):
        with pytest.raises(ValueError):
            C.KnnModel(bad)
    q = torch.zeros((2, 3), dtype=torch.float64, device="cuda")
    ids = torch.empty(2, dtype=torch.int64, device="cuda")
    P = torch.empty((2, 1), dtype=torch.float64, device="cuda")
    f, s = model.features.data_ptr(), model.slots.data_ptr()
    good = [f, s, 4, 3, 1, 1, q.data_ptr(), 2, 2, 3, ids.data_ptr(), P.data_ptr(), None]
    assert lib().b200aa_knn_classify(*good) == 0
    for i, v in ((0, None), (1, None), (6, None), (10, None), (11, None), (2, 0), (3, 0), (4, 0), (5, 0), (8, -1), (9, 2),
                 (7, 0), (7, 3)):
        args = list(good)
        args[i] = v
        assert lib().b200aa_knn_classify(*args) == ERR_INVALID, (i, v)
    args = list(good)
    args[8] = 0
    assert lib().b200aa_knn_classify(*args) == 0                             # n = 0: nothing to do


def test_streams_and_threads_share_one_model(C):
    import torch
    rng = np.random.default_rng(20)
    feats, labels = rng.normal(size=(5000, 136)), rng.integers(0, 4, size=5000).astype(np.float64)
    model = C.KnnModel(_model(feats, labels, 13))
    qs = [torch.from_numpy(rng.normal(size=(700, 136))).cuda() for _ in range(4)]
    alone = []
    for q in qs:
        ids, P = C.knn_classify_batch(model, q)
        alone.append((ids.cpu().numpy(), P.cpu().numpy()))
    streams = [torch.cuda.Stream() for _ in range(2)]
    out = [None] * 4
    for i, q in enumerate(qs):
        with torch.cuda.stream(streams[i % 2]):
            out[i] = C.knn_classify_batch(model, q)
    torch.cuda.synchronize()
    for i in range(4):
        _same((out[i][0].cpu().numpy(), out[i][1].cpu().numpy()), alone[i], "stream %d" % i)
    res, errs = [None] * 4, []

    def work(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                ids, P = C.knn_classify_batch(model, qs[i])
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


def _signal(fs):
    rng = np.random.default_rng(21)
    t = np.arange(8 * fs)
    x = np.concatenate([rng.normal(0, 3000, 8 * fs), 9000 * np.sin(2 * np.pi * 440 * t / fs) + rng.normal(0, 300, 8 * fs),
                        4000 * np.sign(np.sin(2 * np.pi * 3 * t / fs)) * rng.normal(1, 0.2, 8 * fs)])
    return np.round(np.clip(x, -32768, 32767)).astype(np.int16)


def test_mid_term_classification_with_golden_models(C):
    """knn_4class (row subset, k = 13) and knn_speaker_male_female (k = 1) through mid_term_classification: ids and maximum
    posteriors equal the per-window Knn.classify loop over the same GPU-normalised vectors, which stay on the device."""
    import torch
    from pyaudioanalysis_b200.batch import mid_feature_extraction_batch
    g = load_golden("knn.npz")
    fs, mt, st = 16000, 1.0, 0.05
    x = _signal(fs)
    mid, _ = mid_feature_extraction_batch(torch.from_numpy(x).cuda().reshape(1, -1), fs, mt * fs, mt * fs, round(fs * st),
                                          round(fs * st))
    for c in ("knn_4class", "knn_speaker_male_female"):
        feats, labels, k = g[c + "_features"], g[c + "_labels"], int(g[c + "_k"])
        mean, std = g[c + "_mean"], g[c + "_std"]
        vec = C.normalize_windows_batch(mid[0:1].contiguous(), mean, std)[0].double().cpu().numpy()
        ref_ids, ref_post = [], []
        for v in vec:                                           # audioSegmentation.py:579-590, one window at a time
            i, p = knn_oracle(feats, labels, k, v.reshape(1, -1))
            ref_ids.append(i[0])
            ref_post.append(np.max(p[0]))
        for clf in (_model(feats, labels, k), C.KnnModel(_model(feats, labels, k))):
            ids, post = C.mid_term_classification(x, fs, clf, "knn", mean, std, mt, mt, st, st)
            assert isinstance(ids, np.ndarray) and isinstance(post, np.ndarray)
            assert np.array_equal(ids, ref_ids), c
            assert np.array_equal(post, ref_post), c

"""CPU: the pieces of kernel 7 (csrc/hmm.cuh, __host__ __device__) run on the host by tests/hmm_host.cu -- the class
statistics against NumPy's mean / std of features[:, idx], the emissions against hmmlearn's diagonal density evaluated by
NumPy on features.T, the Viterbi pass against tests/hmm_oracle.py and an exhaustive search over every path -- bit for bit;
the host helpers of audioSegmentation; and the C ABI's argument checks, which return before any CUDA call."""
import ctypes
import itertools

import numpy as np
import pytest

from tests import hmm_oracle as H
from tests import host_exe
from tests.host_exe import bits, floats, hexes, run


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "hmm_host.cu", "-O1")


def _features(rng, F, M):
    """A C-contiguous float64 matrix of float32 values (the drop-in's layout), rows of very different scales."""
    x = rng.normal(size=(F, M)) * rng.choice([1e-4, 1.0, 1e3], size=(F, 1)) + rng.normal(size=(F, 1))
    return np.ascontiguousarray(x.astype(np.float32).astype(np.float64))


@pytest.mark.parametrize("F,M", [(136, 50), (136, 4097), (3, 300), (1, 700), (1, 5), (2, 1)])
def test_class_stats_match_numpy(exe, F, M):
    rng = np.random.default_rng(F * 1000 + M)
    feats = _features(rng, F, M)
    labels = rng.integers(0, 3, size=M)
    for u in np.unique(labels):
        idx = np.nonzero(labels == u)[0]
        mean = feats[:, idx].mean(axis=1)
        std = np.std(feats[:, idx], axis=1)
        script = "".join("stats %d %d %s\n" % (idx.size, F == 1, hexes(feats[f, idx])) for f in range(F))
        got = np.array([floats(ln[1:]) for ln in run(exe, script)])
        assert np.array_equal(bits(got[:, 1]), bits(mean)), (F, M, u)
        assert np.array_equal(bits(got[:, 3]), bits(std)), (F, M, u)


def test_class_stats_edges(exe):
    """A constant feature (std 0), one window, -0.0 values, an empty class (NaN)."""
    feats = np.array([[2.5, 2.5, 2.5, 2.5], [-0.0, -0.0, -0.0, -0.0], [1.0, -1.0, 3.0, 1e300]])
    for idx in (np.arange(4), np.array([2]), np.array([0, 1])):
        script = "".join("stats %d 0 %s\n" % (idx.size, hexes(feats[f, idx])) for f in range(3))
        got = np.array([floats(ln[1:]) for ln in run(exe, script)])
        assert np.array_equal(bits(got[:, 1]), bits(feats[:, idx].mean(axis=1)))
        assert np.array_equal(bits(got[:, 3]), bits(np.std(feats[:, idx], axis=1)))
    got = floats(run(exe, "stats 0 0\n")[0][1:])
    assert np.isnan(got[1]) and np.isnan(got[3])


def _emissions(exe, feats, means, var):
    F, M = feats.shape
    konst = F * np.log(2 * np.pi) + np.log(var).sum(axis=-1)
    out = []
    for j in range(means.shape[0]):
        ln = run(exe, "emission %d %d %d %s %s %s %s\n" % (F, M, M == 1, float(konst[j]).hex(), hexes(means[j]), hexes(var[j]),
                                                            hexes(feats.T)))[0]
        out.append(floats(ln[1:]))
    return np.stack(out, axis=1)


@pytest.mark.parametrize("F,M,C", [(136, 40, 3), (136, 1, 4), (5, 30, 2), (1, 9, 3), (136, 2, 1)])
def test_emission_matches_numpy_density(exe, F, M, C):
    rng = np.random.default_rng(F + 7 * M + C)
    feats = _features(rng, F, M)
    means = feats[:, rng.integers(0, M, size=C)].T + rng.normal(scale=0.1, size=(C, F))
    var = rng.random((C, F)) * rng.choice([1e-6, 1.0, 1e4], size=(C, 1)) + 1e-9
    got = _emissions(exe, feats, means, var)
    ref = H.log_density(feats.T, means, var)
    assert np.array_equal(bits(got), bits(ref)), (F, M, C)


def _viterbi(exe, log_start, log_trans, frame):
    n, C = frame.shape
    ln = run(exe, "viterbi %d %d %s %s %s\n" % (C, n, hexes(log_start), hexes(log_trans), hexes(frame)))[0]
    return np.array([int(t) for t in ln[1:]], dtype=np.int64)


def _model(rng, C, zeros=False):
    start = rng.random(C) + 0.05
    trans = rng.random((C, C)) + 0.05
    if zeros and C > 1:
        start[rng.integers(0, C)] = 0.0
        trans[rng.random((C, C)) < 0.3] = 0.0
        trans[np.arange(C), np.arange(C)] = 0.5
    return H.model_logs(start / start.sum(), trans / trans.sum(axis=1, keepdims=True), np.ones((C, 1)))[:2]


def test_viterbi_step_matches_oracle(exe):
    rng = np.random.default_rng(11)
    for C, n in ((1, 1), (1, 20), (2, 1), (3, 50), (10, 200), (33, 60)):
        for zeros in (False, True):
            ls, la = _model(rng, C, zeros)
            frame = rng.normal(scale=30.0, size=(n, C)) - 200.0
            assert np.array_equal(_viterbi(exe, ls, la, frame), H.viterbi(ls, la, frame)), (C, n, zeros)


def test_viterbi_tie_rule(exe):
    """Equal emissions and transitions: every path ties.  The last state is the first maximum (0); each backtrack step
    takes the last maximal predecessor (C - 1)."""
    C, n = 3, 5
    ls, la = np.log(np.full(C, 1.0 / 2 ** 2)), np.log(np.full((C, C), 1.0 / 2 ** 2))
    frame = np.zeros((n, C))
    want = np.array([C - 1] * (n - 1) + [0])
    assert np.array_equal(_viterbi(exe, ls, la, frame), want)
    assert np.array_equal(H.viterbi(ls, la, frame), want)


def test_brute_force_paths(exe):
    """For C <= 3 and n <= 7 every one of the C^n paths is scored in the recursion's order: the decoded path has the
    maximal score, equal in bits; draws with an exact tie between distinct best paths are skipped."""
    rng = np.random.default_rng(12)
    checked = 0
    for _ in range(60):
        C, n = int(rng.integers(1, 4)), int(rng.integers(1, 8))
        ls, la = _model(rng, C, zeros=bool(rng.integers(0, 2)))
        frame = rng.normal(scale=5.0, size=(n, C))
        scores = {p: H.path_score(ls, la, frame, p) for p in itertools.product(range(C), repeat=n)}
        best = max(scores.values())
        if sum(1 for s in scores.values() if s == best) > 1:
            continue
        path = _viterbi(exe, ls, la, frame)
        assert np.array_equal(path, H.viterbi(ls, la, frame))
        assert H.path_score(ls, la, frame, tuple(path)).view(np.uint64) == np.float64(best).view(np.uint64)
        checked += 1
    assert checked > 40


def test_oracle_against_hmmlearn():
    hmmlearn = pytest.importorskip("hmmlearn.hmm")
    rng = np.random.default_rng(13)
    for C, F, n in ((2, 5, 40), (4, 136, 120)):
        feats = _features(rng, F, n)
        hmm = hmmlearn.GaussianHMM(C, "diag")
        start, trans = rng.random(C) + 0.1, rng.random((C, C)) + 0.1
        hmm.startprob_, hmm.transmat_ = start / start.sum(), trans / trans.sum(axis=1, keepdims=True)
        hmm.means_ = feats[:, rng.integers(0, n, size=C)].T
        hmm.covars_ = rng.random((C, F)) + 0.5
        want = hmm.predict(feats.T)
        assert np.array_equal(H.predict(feats, hmm.startprob_, hmm.transmat_, hmm.means_, hmm._covars_), want)


# ------------------------------------------------------------------ host helpers
def test_segments_to_labels_quirks(tmp_path):
    from pyaudioanalysis_b200 import audioSegmentation as S
    gt = tmp_path / "a.segments"
    gt.write_text("0.0\t2.0\tspeech\n2.5\t4.0\tmusic\nbad row\n3.5\t6.0\tspeech\n")
    start, end, labels = S.read_segmentation_gt(str(gt))
    assert list(start) == [0.0, 2.5, 3.5] and list(end) == [2.0, 4.0, 6.0] and labels == ["speech", "music", "speech"]
    flags, names = S.segments_to_labels(start, end, labels, 1.0)
    assert names == list(set(labels))
    # centres 0.5 1.5 | 2.5 (gap: the last segment's label) | 3.5 (music) | 4.5 5.5 (overlap ends: speech)
    want = [names.index(c) for c in ("speech", "speech", "speech", "music", "speech", "speech")]
    assert list(flags) == want


def test_statistics_priors_and_transitions():
    from pyaudioanalysis_b200 import audioSegmentation as S
    labels = np.array([0, 0, 1, 1, 1, 0, 2, 2, 0.0])
    T = S._transitions(labels, 3)
    ref = np.zeros((3, 3))
    for i in range(len(labels) - 1):
        ref[int(labels[i]), int(labels[i + 1])] += 1
    ref = ref / ref.sum(axis=1, keepdims=True)
    assert np.array_equal(T, ref)
    with np.errstate(invalid="ignore"):
        T = S._transitions(np.array([0.0, 1.0, 1.0, 0.0, 3.0]), 4)         # class 2 has no outgoing transition: NaN row
    assert np.isnan(T[2]).all() and np.isnan(T[3]).all()
    with pytest.raises(IndexError):
        S._transitions(np.array([0.0, 2.0, 1.0]), 2)                      # a label >= C


def test_confusion_and_metrics():
    from pyaudioanalysis_b200 import audioSegmentation as S
    pred, gt = np.array([0, 1, -1, 1, 0]), np.array([0, 1, 1, 0])
    cm = S.calculate_confusion_matrix(pred, gt, ["a", "b"])
    assert np.array_equal(cm, np.array([[1.0, 1.0], [0.0, 2.0]]))         # -1 counts in the last column
    assert S.segmentation_accuracy(pred, gt) == 0.5
    assert S.segmentation_accuracy(pred[:0], gt) == -1
    rec, pre, f1 = S.compute_metrics(cm, ["a", "b"])
    assert rec == [0.5, 1.0] and pre == [1.0, 2 / 3.0]


# ------------------------------------------------------------------ C ABI argument checks (no CUDA call is made)
@pytest.fixture(scope="module")
def L():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib


def test_statistics_rejects_bad_arguments(L):
    lib = L.lib()
    dummy = ctypes.c_void_p(16)
    n = np.array([3, 2], dtype=np.int64)
    off = np.array([0, 2, 5], dtype=np.int64)
    idx = np.array([0, 4, 1, 2, 3], dtype=np.int64)

    def call(mid=dummy, dtype=L.DTYPE_F32, B=2, F=4, M=3, n=n, C=2, off=off, idx=idx, out=dummy):
        p = (lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data))
        return lib.b200aa_hmm_statistics(mid, dtype, B, F, M, p(n), C, p(off), p(idx), out, None)

    assert call(mid=None) == L.ERR_INVALID
    assert call(out=None) == L.ERR_INVALID
    assert call(n=None) == L.ERR_INVALID
    assert call(dtype=0) == L.ERR_INVALID
    assert call(B=0) == L.ERR_INVALID
    assert call(F=0) == L.ERR_INVALID
    assert call(C=0) == L.ERR_INVALID
    assert call(n=np.array([4, 2], dtype=np.int64)) == L.ERR_INVALID                  # a count above m_stride
    assert call(n=np.array([-1, 2], dtype=np.int64)) == L.ERR_INVALID
    assert call(idx=np.array([0, 5, 1, 2, 3], dtype=np.int64)) == L.ERR_INVALID       # outside [0, 5)
    assert call(idx=np.array([0, -1, 1, 2, 3], dtype=np.int64)) == L.ERR_INVALID
    assert call(off=np.array([1, 2, 5], dtype=np.int64)) == L.ERR_INVALID
    assert call(off=np.array([0, 3, 2], dtype=np.int64)) == L.ERR_INVALID


def test_decode_rejects_bad_arguments(L):
    lib = L.lib()
    d = ctypes.c_void_p(16)
    n = np.array([3, 1], dtype=np.int64)

    def call(mid=d, B=2, F=4, M=3, n=n, C=2, ptrs=(d,) * 5, ids=d, bad=d):
        return lib.b200aa_hmm_decode(mid, B, F, M, None if n is None else ctypes.c_void_p(n.ctypes.data), C, *ptrs, ids, bad,
                                     None)

    assert call(mid=None) == L.ERR_INVALID
    assert call(ids=None) == L.ERR_INVALID
    assert call(bad=None) == L.ERR_INVALID
    assert call(n=None) == L.ERR_INVALID
    for k in range(5):
        assert call(ptrs=tuple(None if i == k else d for i in range(5))) == L.ERR_INVALID
    assert call(B=0) == L.ERR_INVALID
    assert call(F=0) == L.ERR_INVALID
    assert call(M=0) == L.ERR_INVALID
    assert call(C=0) == L.ERR_INVALID
    assert call(C=2049) == L.ERR_INVALID
    assert call(n=np.array([3, 0], dtype=np.int64)) == L.ERR_INVALID                  # a count below 1
    assert call(n=np.array([4, 1], dtype=np.int64)) == L.ERR_INVALID                  # a count above m_stride

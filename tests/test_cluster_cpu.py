"""CPU: kernel 9 (csrc/cluster.cuh) run on the host by tests/cluster_host.cu -- its plan, distances, leaves and combines --
against np.mean of scipy's pdist / cdist, compared as float64 bit patterns; NumPy's reduction order that the kernel
relies on; and the C ABI's argument checks, which return before any CUDA call."""
import ctypes

import numpy as np
import pytest
from scipy.spatial import distance

from tests import host_exe
from tests.cluster_cases import PLAN_CASES, Plan, adversarial
from tests.diarization_oracle import reference
from tests.host_exe import bits, floats, hexes, run


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "cluster_host.cu", "-O2")


def host_means(exe, X, labels, K, want=None, seg_terms=1 << 22, pass_terms=1 << 24):
    n, D = X.shape
    want = np.ones(K, dtype=np.int64) if want is None else np.asarray(want, dtype=np.int64)
    script = "means %d %d %d %d %d %s %s %s\n" % (K, D, n, seg_terms, pass_terms, " ".join(map(str, labels)),
                                                 " ".join(map(str, want)), hexes(X))
    out = floats(run(exe, script)[0][1:])
    return out[:K], out[K:].reshape(K, K)


def _check(exe, X, labels, K, want=None, **plan):
    A, B = host_means(exe, X, labels, K, want, **plan)
    rA, rB = reference(X, labels, K, want)
    assert np.array_equal(bits(A), bits(rA)), (A, rA)
    assert np.array_equal(bits(B), bits(rB)), (B, rB)


@pytest.mark.parametrize("kind", [0, 1])
def test_pdist_adds_like_cdist(exe, kind):
    """Both kinds of distance run the same chain and equal scipy's, element by element, on adversarial values (the
    chain's order shows at huge and tiny scales)."""
    rng = np.random.default_rng(3 + kind)
    for n, D in ((1, 1), (1, 5), (7, 1), (9, 13), (40, 24), (3, 150)):
        X = adversarial(rng, n, D)
        if n * D > 4:
            X.flat[rng.integers(0, n * D, size=2)] = [np.nan, np.inf]
        got = floats(run(exe, "dist %d %d %d %s\n" % (kind, n, D, hexes(X)))[0][1:])
        want = (distance.cdist(X, X) if kind == 0 else distance.pdist(X.T)).ravel()
        assert np.array_equal(bits(got), bits(want)), (kind, n, D)
    # the two scipy functions agree with each other on the same pairs
    X = adversarial(rng, 30, 6)
    assert np.array_equal(bits(distance.pdist(X.T)), bits(distance.cdist(X.T, X.T)[np.triu_indices(6, 1)]))


@pytest.mark.parametrize("sizes", [(1, 1), (1, 7), (8, 16), (13, 10), (128, 1), (64, 3), (129, 2), (100, 83), (91, 91)])
def test_block_sizes(exe, sizes):
    """Blocks of n_c x n_c2 terms below, at and past multiples of 8 and 128 (and past 8192), one feature to many."""
    rng = np.random.default_rng(sum(sizes))
    n1, n2 = sizes
    for D in (1, 5, 37):
        X = rng.normal(size=(n1 + n2, D)) * rng.choice([1e-3, 1.0, 1e3], size=(1, D))
        labels = np.array([0] * n1 + [1] * n2)
        rng.shuffle(labels)
        _check(exe, X, labels, 2)


def test_adversarial_values(exe):
    """+-0, subnormals, huge and tiny scales, NaN and inf in the rows; a one-row cluster; one feature (A is NaN)."""
    rng = np.random.default_rng(5)
    X = adversarial(rng, 60, 9)
    labels = rng.integers(0, 4, size=60)
    labels[17] = 4                                                  # cluster 4 has one row
    _check(exe, X, labels, 5)
    X[3, 2], X[40, 7] = np.nan, np.inf
    _check(exe, X, labels, 5)
    _check(exe, X[:, :1].copy(), labels, 5)


def test_empty_and_unwanted_clusters(exe):
    """An empty cluster gives NaN means against it (NumPy's mean of an empty array); clusters not wanted stay NaN."""
    rng = np.random.default_rng(6)
    X = rng.normal(size=(50, 4))
    labels = rng.integers(0, 3, size=50)
    labels[labels == 1] = 2                                         # cluster 1 empty
    _check(exe, X, labels, 3)
    _check(exe, X, labels, 3, want=[1, 0, 1])


@pytest.mark.parametrize("seg_terms,pass_terms", [(128, 200), (300, 5000), (1000, 1000), (1 << 22, 1 << 24)])
def test_segments_and_passes(exe, seg_terms, pass_terms):
    """The same means when every mean is cut into many segments and the segments into many passes: the split follows
    the pairwise tree, so the result cannot change."""
    rng = np.random.default_rng(seg_terms)
    X = rng.normal(size=(260, 11)) * np.exp(rng.uniform(-5, 5, size=(260, 11)))
    labels = rng.choice(4, size=260, p=[0.5, 0.3, 0.15, 0.05])
    _check(exe, X, labels, 4, seg_terms=seg_terms, pass_terms=pass_terms)


def test_block_past_numpy_buffer(exe):
    """A block of 120 x 90 = 10 800 terms (past NumPy's 8192-element buffer) and a condensed vector of 8 385 terms
    (D = 130)."""
    rng = np.random.default_rng(7)
    X = rng.normal(size=(210, 130)) * np.exp(rng.uniform(-3, 3, size=(1, 130)))
    labels = np.array([0] * 120 + [1] * 90)
    _check(exe, X, labels, 2, seg_terms=4096)


def test_numpy_mean_is_one_pairwise_sum():
    """np.mean of a C-contiguous 2-D array (and of a 1-D one) is np.add.reduce over all its elements in one pairwise
    tree, divided by the count: the order kernel 9 reproduces, below and past NumPy's 8192-element buffer."""
    rng = np.random.default_rng(8)

    def pairwise(a):
        n = a.size
        if n < 8:
            r = 0.0
            for x in a:
                r += x
            return r
        if n <= 128:
            r = [a[j] for j in range(8)]
            i = 8
            while i < n - n % 8:
                for j in range(8):
                    r[j] += a[i + j]
                i += 8
            res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            for k in range(i, n):
                res += a[k]
            return res
        n2 = n // 2
        n2 -= n2 % 8
        return pairwise(a[:n2]) + pairwise(a[n2:])

    for shape in ((5,), (127, 1), (64, 128), (8192,), (8193,), (91, 91), (300, 701), (20000,)):
        a = np.abs(rng.normal(size=shape)) * np.exp(rng.uniform(-30, 30, size=shape))
        want = pairwise(a.ravel()) / a.size
        assert np.float64(np.mean(a)).view(np.uint64) == np.float64(want).view(np.uint64), shape


def test_sum_past_2_31_terms(exe):
    """A pairwise sum of more than 2^31 terms (64-bit offsets), cut into segments and leaves, equals the direct
    pairwise sum; the segments tile the terms and no leaf exceeds 128 (the harness checks both)."""
    got = floats(run(exe, "bigsum %d %d\n" % ((1 << 31) + 1000, 1 << 22))[0][1:])
    assert got[0].view(np.uint64) == got[1].view(np.uint64)


@pytest.mark.parametrize("case", PLAN_CASES, ids=lambda c: c.name)
def test_plan_cases_take_their_path(exe, case):
    """Each clustering that tests/test_gpu_cluster.py runs to reach a path of make_plan still takes it at the library's
    kSegTerms and kPassTerms, so a change of either limit cannot quietly turn the case into an easy one."""
    plan = Plan.parse(run(exe, "plan %d %d %s\n" % (len(case.sizes), case.D, " ".join(map(str, case.sizes))))[0])
    assert case.check(plan, case.D), (case.hits, plan.passes, plan.kind, plan.len, plan.pass_of)


# ------------------------------------------------------------------ C ABI argument checks (no CUDA call is made)
@pytest.fixture(scope="module")
def L():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib


def test_cluster_rejects_bad_arguments(L):
    lib = L.lib()
    d = ctypes.c_void_p(16)
    labels = np.array([0, 1, 1, 0], dtype=np.int32)

    def call(X=d, n=4, D=3, stride=3, labels=labels, K=2, want=None, A=d, B=d):
        lab = None if labels is None else ctypes.c_void_p(labels.ctypes.data)
        w = None if want is None else ctypes.c_void_p(np.asarray(want, dtype=np.uint8).ctypes.data)
        return lib.b200aa_cluster_distance_means(X, n, D, stride, lab, K, w, A, B, None)

    assert call(X=None) == L.ERR_INVALID
    assert call(A=None) == L.ERR_INVALID
    assert call(B=None) == L.ERR_INVALID
    assert call(labels=None) == L.ERR_INVALID
    assert call(n=0) == L.ERR_INVALID
    assert call(D=0) == L.ERR_INVALID
    assert call(D=4097, stride=4097) == L.ERR_INVALID
    assert call(stride=2) == L.ERR_INVALID
    assert call(K=0) == L.ERR_INVALID
    assert call(K=1025) == L.ERR_INVALID
    assert call(labels=np.array([0, 2, 1, 0], dtype=np.int32)) == L.ERR_INVALID      # a label >= K
    assert call(labels=np.array([0, -1, 1, 0], dtype=np.int32)) == L.ERR_INVALID


def test_decode_f64_rejects_bad_arguments(L):
    lib = L.lib()
    d = ctypes.c_void_p(16)
    n = np.array([3, 1], dtype=np.int64)

    def call(mid=d, B=2, F=4, M=3, major=1, n=n, C=2, ptrs=(d,) * 5, ids=d, bad=d):
        return lib.b200aa_hmm_decode_f64(mid, B, F, M, major, None if n is None else ctypes.c_void_p(n.ctypes.data), C, *ptrs,
                                         ids, bad, None)

    assert call(major=2) == L.ERR_INVALID
    assert call(major=-1) == L.ERR_INVALID
    assert call(mid=None) == L.ERR_INVALID
    assert call(ids=None) == L.ERR_INVALID
    assert call(bad=None) == L.ERR_INVALID
    assert call(n=None) == L.ERR_INVALID
    for k in range(5):
        assert call(ptrs=tuple(None if i == k else d for i in range(5))) == L.ERR_INVALID
    assert call(B=0) == L.ERR_INVALID
    assert call(C=2049) == L.ERR_INVALID
    assert call(n=np.array([3, 0], dtype=np.int64)) == L.ERR_INVALID
    assert call(n=np.array([4, 1], dtype=np.int64)) == L.ERR_INVALID

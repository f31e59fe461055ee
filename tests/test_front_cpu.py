"""CPU: kernel 11 (csrc/front.cuh) run on the host by tests/front_host.cu -- the scaler in both summation orders, the
outlier rule and the per-frame pooling -- against scikit-learn 1.9, scipy and NumPy, compared as float64 bit patterns;
the layouts each call site hands the scaler, read from NumPy's flags; the C ABI's argument checks, which return before
any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.spatial import distance

from tests import host_exe
from tests.front_cases import NS, column_major, outlier_rule, pool_bank, pool_loop, sk_scale, value_bank, with_nans
from tests.host_exe import bits, floats, hexes, run
from pyaudioanalysis_b200 import audioSegmentation as A


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "front_host.cu", "-O2")


def host_scale(exe, X, pairwise):
    n, D = X.shape
    out = run(exe, "scale %d %d %d %s\n" % (n, D, int(pairwise), hexes(X)))[0]
    v = floats(out[1:])
    return v[2 * D + 1:].reshape(n, D), v[:D], v[D:2 * D], bool(v[2 * D])


def check_scale(exe, X):
    """Both layouts of X against scikit-learn, each in the order NumPy sums it; the other order is a mutant."""
    results = {}
    for layout, Xl in (("C", np.ascontiguousarray(X)), ("F", column_major(X))):
        Y, mean, scale = sk_scale(Xl)
        assert Y.flags.f_contiguous == (layout == "F") or X.shape[1] == 1 or X.shape[0] == 1
        pairwise = layout == "F" or X.shape[1] == 1
        hY, hmean, hscale, inf = host_scale(exe, X, pairwise)
        assert not inf
        np.testing.assert_array_equal(bits(hmean), bits(mean))
        np.testing.assert_array_equal(bits(hscale), bits(scale))
        np.testing.assert_array_equal(bits(hY), bits(Y))
        results[layout] = (mean, scale)
    return results


@pytest.mark.parametrize("n", NS)
def test_scaler_matches_sklearn_both_layouts(exe, n):
    rng = np.random.default_rng(n)
    check_scale(exe, value_bank(rng, n, 11))
    check_scale(exe, rng.normal(size=(n, 3)) * 1e3 + 7)


@pytest.mark.parametrize("n", (1, 9, 129, 8193))
def test_scaler_nan_rows_and_all_nan_column(exe, n):
    rng = np.random.default_rng(100 + n)
    check_scale(exe, with_nans(rng, value_bank(rng, n, 7), all_nan_col=3))
    X = np.full((n, 2), np.nan)
    check_scale(exe, X)


def test_scaler_single_column_and_row_strides(exe):
    """A strided view sums in the order of its smaller stride: NumPy's rule the library applies to strides."""
    rng = np.random.default_rng(5)
    base = rng.normal(size=(300, 40)) * 3 + 1
    for X in (base[::3, 5:6], base.T[::2, ::5].T, base[10:200:2, ::7], base.T[:, 10:250].T):
        pairwise = X.shape[1] == 1 or abs(X.strides[0]) < abs(X.strides[1])
        Y, mean, scale = sk_scale(X)
        hY, hmean, hscale, _ = host_scale(exe, np.ascontiguousarray(X), pairwise)
        np.testing.assert_array_equal(bits(hmean), bits(mean))
        np.testing.assert_array_equal(bits(hY), bits(Y))


def test_summation_order_matters(exe):
    """The wrong order changes some bit on the value bank: the two layouts are not interchangeable."""
    rng = np.random.default_rng(11)
    X = rng.normal(size=(8193, 8)) * 1e3 + 1e7
    _, mean, _ = sk_scale(column_major(X))
    _, wrong, _, _ = host_scale(exe, X, False)
    assert (bits(wrong) != bits(mean)).any()


def test_inf_is_flagged_and_sklearn_refuses(exe):
    X = np.random.default_rng(3).normal(size=(20, 4))
    for v in (np.inf, -np.inf):
        Xi = X.copy()
        Xi[7, 2] = v
        assert host_scale(exe, Xi, True)[3] and host_scale(exe, Xi, False)[3]
        with pytest.raises(ValueError):
            sk_scale(column_major(Xi))
    assert not host_scale(exe, with_nans(np.random.default_rng(4), X), True)[3]


def host_outlier(exe, Xn):
    M, D = Xn.shape
    v = floats(run(exe, "outlier %d %d %s\n" % (M, D, hexes(Xn)))[0][1:])
    return np.flatnonzero(v[D + 1:]), v[:D], v[D]


@pytest.mark.parametrize("M,D", [(1, 1), (5, 2), (9, 17), (300, 64), (129, 146)])
def test_outlier_rule_matches_scipy(exe, M, D):
    rng = np.random.default_rng(M * D)
    Xn = sk_scale(column_major(value_bank(rng, M, D)))[0]
    keep, dist_all = outlier_rule(Xn)
    hkeep, hdist, hmean = host_outlier(exe, Xn)
    np.testing.assert_array_equal(bits(hdist), bits(dist_all))
    assert bits(hmean) == bits(np.mean(dist_all))
    np.testing.assert_array_equal(hkeep, keep)


def test_outlier_rule_with_nan_column(exe):
    rng = np.random.default_rng(9)
    Xn = sk_scale(column_major(rng.normal(size=(40, 6))))[0]
    Xn[3, 2] = np.nan
    keep, dist_all = outlier_rule(Xn)
    hkeep, hdist, _ = host_outlier(exe, Xn)
    np.testing.assert_array_equal(bits(hdist), bits(dist_all))
    np.testing.assert_array_equal(hkeep, keep)


def test_outlier_column_sums_are_sequential(exe):
    """np.sum(axis=0) of the C-contiguous squareform adds its rows in sequence: a pairwise sum differs somewhere."""
    rng = np.random.default_rng(2)
    Xn = sk_scale(column_major(rng.normal(size=(50, 150)) * np.exp(rng.normal(size=150) * 3)))[0]
    sq = distance.squareform(distance.pdist(Xn.T))
    assert sq.flags.c_contiguous
    pairwise = np.array([np.sum(np.ascontiguousarray(sq[:, j])) for j in range(sq.shape[1])])
    _, hdist, _ = host_outlier(exe, Xn)
    assert (bits(pairwise) != bits(hdist)).any()


def host_pool(exe, st, r):
    F, T = st.shape
    return floats(run(exe, "pool %d %d %d %s\n" % (F, T, r, hexes(st)))[0][1:]).reshape(2 * F, T)


@pytest.mark.parametrize("T,r", [(1, 1), (9, 3), (60, 40), (200, 129), (400, 300), (300, 1000)])
def test_pooling_matches_reference_loop(exe, T, r):
    rng = np.random.default_rng(T + r)
    st = pool_bank(rng, 5, T)
    ref = pool_loop(st, r)
    np.testing.assert_array_equal(bits(A.pool_frames(st, r)), bits(ref))
    np.testing.assert_array_equal(bits(host_pool(exe, st.astype(np.float64), r)), bits(ref))


def test_call_site_layouts():
    """The layouts the call sites hand the scaler: the transpose of a C-contiguous matrix (column-major), and what
    scikit-learn returns for it (column-major too), which standardise makes C-contiguous."""
    rng = np.random.default_rng(0)
    mid, post = rng.normal(size=(6, 30)), [rng.random((30, 2))]
    feats = A._with_posteriors(mid, post)
    assert feats.flags.c_contiguous and feats.T.flags.f_contiguous
    assert sk_scale(feats.T)[0].flags.f_contiguous
    pooled = A.pool_frames(rng.normal(size=(4, 30)).astype(np.float32), 3)
    assert A._with_posteriors(pooled, post).T.flags.f_contiguous
    st = rng.normal(size=(68, 40))
    assert np.asarray(st).T.flags.f_contiguous and A.standardise(st).flags.c_contiguous
    feats32 = torch.zeros((2, 68, 40)).transpose(1, 2)
    assert feats32.stride(1) < feats32.stride(2)


def test_abi_refuses_bad_arguments_before_cuda():
    from pyaudioanalysis_b200 import _lib
    try:
        L = _lib.lib()
    except RuntimeError:
        pytest.skip("libb200aa.so not built")
    rows = np.array([4], dtype=np.int64)
    off = np.zeros(1, dtype=np.int64)
    p = ctypes.c_void_p(16)
    r, o = ctypes.c_void_p(rows.ctypes.data), ctypes.c_void_p(off.ctypes.data)
    scale = L.b200aa_standard_scale
    assert scale(None, _lib.DTYPE_F64, 1, 3, r, 0, 3, 1, p, o, 3, 1, p, p, p, None) == _lib.ERR_INVALID
    assert scale(p, 7, 1, 3, r, 0, 3, 1, p, o, 3, 1, p, p, p, None) == _lib.ERR_INVALID
    assert scale(p, _lib.DTYPE_F64, 1, 0, r, 0, 3, 1, p, o, 3, 1, p, p, p, None) == _lib.ERR_INVALID
    assert scale(p, _lib.DTYPE_F64, 1, 3, r, 0, 0, 1, p, o, 3, 1, p, p, p, None) == _lib.ERR_INVALID
    rows[0] = 0
    assert scale(p, _lib.DTYPE_F64, 1, 3, r, 0, 3, 1, p, o, 3, 1, p, p, p, None) == _lib.ERR_INVALID
    outl = L.b200aa_outlier_columns
    assert outl(p, 10, 0, 10, p, p, p, None) == _lib.ERR_INVALID
    assert outl(p, 10, 4097, 10, p, p, p, None) == _lib.ERR_INVALID
    assert outl(p, 10, 3, 9, p, p, p, None) == _lib.ERR_INVALID
    assert outl(None, 10, 3, 10, p, p, p, None) == _lib.ERR_INVALID
    frames = np.array([5], dtype=np.int64)
    fr = ctypes.c_void_p(frames.ctypes.data)
    pool = L.b200aa_pool_frames
    assert pool(p, _lib.DTYPE_F32, 1, 2, 10, 5, fr, 0, p, 5, None) == _lib.ERR_INVALID
    assert pool(p, _lib.DTYPE_F32, 1, 2, 10, 5, fr, 3, p, 4, None) == _lib.ERR_INVALID
    assert pool(p, 9, 1, 2, 10, 5, fr, 3, p, 5, None) == _lib.ERR_INVALID

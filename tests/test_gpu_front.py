"""GPU: kernel 11 (``consumers.standard_scale_batch``, ``outlier_columns``, ``pool_frames_batch``) bit for bit against
scikit-learn 1.9, scipy and the reference's pooling loop: both layouts, the row counts around NumPy's leaves, the value
bank, NaN and +-inf, D around 16 and 64, ragged batches with poisoned padding, strided and float32 inputs, threads on
their own streams; ``diarize`` in both branches against the host-step restatement under one NumPy seed, every array of
its details."""
import threading

import numpy as np
import pytest

from tests import diarization_oracle as O
from tests.front_cases import NS, column_major, outlier_rule, pool_bank, pool_loop, sk_scale, value_bank, with_nans
from tests.host_exe import bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import consumers
    return consumers


def cuda(a):
    import torch
    return torch.from_numpy(a).cuda()


def dev_scale(C, Xl):
    """standard_scale_batch of a NumPy array uploaded with its layout kept."""
    t = cuda(np.ascontiguousarray(Xl.T)).t() if Xl.flags.f_contiguous and not Xl.flags.c_contiguous else cuda(Xl)
    Y, mean, scale = C.standard_scale_batch(t)
    return Y, mean.cpu().numpy(), scale.cpu().numpy()


def check(C, X):
    for Xl in (np.ascontiguousarray(X), column_major(X)):
        want, wmean, wscale = sk_scale(Xl)
        Y, mean, scale = dev_scale(C, Xl)
        if X.shape[0] > 1 and X.shape[1] > 1:
            assert (Y.stride(0) == 1) == want.flags.f_contiguous
        np.testing.assert_array_equal(bits(mean), bits(wmean))
        np.testing.assert_array_equal(bits(scale), bits(wscale))
        np.testing.assert_array_equal(bits(Y.cpu().numpy()), bits(want))


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("D", [11, 16, 64, 65])
def test_scaler_value_bank(C, n, D):
    rng = np.random.default_rng(n * 100 + D)
    check(C, value_bank(rng, n, D))


@pytest.mark.parametrize("n", [1, 9, 129, 8193])
def test_scaler_nan(C, n):
    rng = np.random.default_rng(n)
    check(C, with_nans(rng, value_bank(rng, n, 17), all_nan_col=5))
    check(C, np.full((n, 3), np.nan))


def test_scaler_inf_raises_sklearns_error(C):
    X = np.random.default_rng(1).normal(size=(50, 16))
    X[20, 3] = -np.inf
    for Xl in (X, column_major(X)):
        with pytest.raises(ValueError, match="infinity"):
            dev_scale(C, Xl)


def test_scaler_ragged_batch_with_poisoned_padding_float32_and_strides(C):
    rng = np.random.default_rng(2)
    rows = np.array([1, 129, 8, 300, 7], dtype=np.int64)
    D, n_max = 68, int(rows.max())
    feats = np.full((len(rows), D, n_max), np.inf, dtype=np.float32)       # [B, F, T] as the feature tensor
    for b, n in enumerate(rows):
        feats[b, :, :n] = pool_bank(rng, D, int(n))
    feats[2, 1, n_max - 1] = np.nan
    t = cuda(feats).transpose(1, 2)
    Y, mean, scale = C.standard_scale_batch(t, rows)
    for b, n in enumerate(rows):
        want, wmean, wscale = sk_scale(feats[b, :, :n].astype(np.float64).T)
        np.testing.assert_array_equal(bits(Y[b, :n].cpu().numpy()), bits(want))
        np.testing.assert_array_equal(bits(mean[b].cpu().numpy()), bits(wmean))
        assert not Y[b, n:].any()
    base = rng.normal(size=(400, 90)) * 4 + 2
    tb = cuda(base)
    for sl in (np.s_[::3, 5:6], np.s_[10:300:2, ::7]):
        want = sk_scale(base[sl])[0]
        np.testing.assert_array_equal(bits(C.standard_scale_batch(tb[sl])[0].cpu().numpy()), bits(want))
    tt = cuda(np.ascontiguousarray(base.T))                                # column-major views of the transpose
    for sl in (np.s_[::2, ::5], np.s_[:, 10:250]):
        want = sk_scale(np.ascontiguousarray(base.T)[sl].T)[0]
        np.testing.assert_array_equal(bits(C.standard_scale_batch(tt[sl].t())[0].cpu().numpy()), bits(want))


@pytest.mark.parametrize("M,D", [(1, 1), (7, 2), (300, 16), (129, 64), (1000, 146), (50, 257)])
def test_outlier_rule(C, M, D):
    rng = np.random.default_rng(M + D)
    Xn = sk_scale(column_major(value_bank(rng, M, D) if D < 100 else rng.normal(size=(M, D)) * 3))[0]
    keep, dist_all = outlier_rule(Xn)
    got, got_dist = C.outlier_columns(cuda(np.ascontiguousarray(Xn.T)).t())
    np.testing.assert_array_equal(bits(got_dist.cpu().numpy()), bits(dist_all))
    np.testing.assert_array_equal(got, keep)
    got_c = C.outlier_columns(cuda(np.ascontiguousarray(Xn)))[0]                  # a C-contiguous input is copied
    np.testing.assert_array_equal(got_c, keep)


@pytest.mark.parametrize("T,r", [(1, 1), (50, 3), (700, 40), (400, 129), (300, 1000)])
def test_pooling(C, T, r):
    rng = np.random.default_rng(T * r)
    st = pool_bank(rng, 68, T)
    want = pool_loop(st, r)
    for t in (cuda(st), cuda(st.astype(np.float64))):
        np.testing.assert_array_equal(bits(C.pool_frames_batch(t, r).cpu().numpy()), bits(want))


def test_pooling_ragged_with_poisoned_padding(C):
    rng = np.random.default_rng(4)
    frames = np.array([5, 200, 1, 131], dtype=np.int64)
    st = np.full((4, 12, 200), np.nan, dtype=np.float32)
    for b, T in enumerate(frames):
        st[b, :, :T] = pool_bank(rng, 12, int(T))
    out = C.pool_frames_batch(cuda(st)[:, :, :], 130, frames).cpu().numpy()
    for b, T in enumerate(frames):
        np.testing.assert_array_equal(bits(out[b, :, :T]), bits(pool_loop(st[b, :, :T], 130)))
        assert not out[b, :, T:].any()


def test_threads_on_their_own_streams(C):
    import torch
    rng = np.random.default_rng(8)
    Xs = [rng.normal(size=(int(n), 64)) * 5 for n in rng.integers(100, 3000, 8)]
    want = [(sk_scale(column_major(X))[0], outlier_rule(sk_scale(column_major(X))[0])[0]) for X in Xs]
    got = [None] * 8

    def work(k):
        with torch.cuda.stream(torch.cuda.Stream()):
            t = cuda(np.ascontiguousarray(Xs[k].T)).t()
            for _ in range(3):
                Y = C.standard_scale_batch(t)[0]
                keep = C.outlier_columns(Y)[0]
                pooled = C.pool_frames_batch(t.t().float(), 40)
            got[k] = (Y.cpu().numpy(), keep, pooled.cpu().numpy())

    threads = [threading.Thread(target=work, args=(k,)) for k in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    for k in range(8):
        np.testing.assert_array_equal(bits(got[k][0]), bits(want[k][0]))
        np.testing.assert_array_equal(got[k][1], want[k][1])
        np.testing.assert_array_equal(bits(got[k][2]), bits(pool_loop(Xs[k].T.astype(np.float32), 40)))


def test_diarize_details_both_branches(C):
    """Every array of diarize's details and cls against the host steps under one NumPy seed, with the default k-means:
    a 900-window matrix without LDA, and the LDA branch."""
    from sklearn.cluster import KMeans
    from pyaudioanalysis_b200 import audioSegmentation as S
    from tests.diarization_cases import lda_case
    rng = np.random.default_rng(31)
    models, st, mid_lda, post_lda = lda_case(rng)
    who = np.repeat(rng.integers(0, 3, size=18), 50)
    mid = (rng.normal(size=(3, 136))[who] * 2 + rng.normal(size=(900, 136))).T
    post = [S._posteriors(mid.T, m) for m in models]
    for mid, post, lda in ((mid, post, None), (mid_lda, post_lda, (st, models, 1.0, 0.1, 2))):
        feats = np.concatenate([mid] + [np.asarray(p).T + 1e-4 for p in post])
        keep = outlier_rule(sk_scale(feats.T)[0])[0]
        np.random.seed(5)
        cls, info = S.diarize(mid, models, 0, 0.1, 0.1, 0 if lda is None else 2, st=st, mid_window=1.0,
                              posteriors=post, details=True)
        np.random.seed(5)
        want_cls, sil_all, num, labels = O.diarize(mid, post, 0, lambda x, k: KMeans(n_clusters=k).fit(x).labels_,
                                                   lda=lda)
        np.testing.assert_array_equal(info["i_non_outliers"], keep)
        np.testing.assert_array_equal(bits(info["sil_all"]), bits(sil_all))
        assert info["num_speakers"] == num
        for a, b in zip(info["labels"], labels):
            np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(cls, want_cls)

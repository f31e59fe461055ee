"""GPU: kernel 9 (b200aa_cluster_distance_means, consumers.cluster_distance_means) bit for bit np.mean of scipy's pdist /
cdist on seeded clusterings up to 36 000 rows, strided inputs, a block past 2^31 terms, streams and threads."""
import threading

import numpy as np
import pytest
from scipy.spatial import distance

from tests.diarization_oracle import reference
from tests.host_exe import bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import consumers
    return consumers


def _run(C, X, labels, K, rows=None):
    import torch
    t = X if isinstance(X, torch.Tensor) else torch.from_numpy(X).cuda()
    A, B = C.cluster_distance_means(t, labels, K, rows)
    return A.cpu().numpy(), B.cpu().numpy()


def _same(got, want):
    assert np.array_equal(bits(got[0]), bits(want[0])), (got[0], want[0])
    assert np.array_equal(bits(got[1]), bits(want[1])), (got[1], want[1])


@pytest.mark.parametrize("M,D,K", [(50, 7, 2), (600, 146, 4), (3600, 146, 9), (3600, 1, 3), (36000, 3, 3)])
def test_matches_scipy(C, M, D, K):
    rng = np.random.default_rng(M + D + K)
    X = rng.normal(size=(M, D)) * np.exp(rng.uniform(-4, 4, size=(1, D))) + rng.normal(size=(1, D))
    labels = rng.choice(K, size=M, p=np.arange(1, K + 1) / (K * (K + 1) / 2))
    _same(_run(C, X, labels, K), reference(X, labels, K))


def test_rows_subset_and_small_clusters(C):
    """Only the clusters asked for are computed (the others NaN); a one-row cluster and an empty one."""
    rng = np.random.default_rng(2)
    X = rng.normal(size=(400, 20))
    labels = rng.integers(0, 5, size=400)
    labels[labels == 3] = 0
    labels[11] = 3
    labels[labels == 4] = 1                                      # cluster 4 empty
    rows = [0, 2, 3]
    want = np.zeros(5, dtype=bool)
    want[rows] = True
    _same(_run(C, X, labels, 5, rows), reference(X, labels, 5, want))


def test_strided_rows(C):
    """Rows at a stride of 3 D, and columns sliced from a wider matrix."""
    import torch
    rng = np.random.default_rng(3)
    big = rng.normal(size=(900, 3 * 30))
    labels = rng.integers(0, 3, size=300)
    t = torch.from_numpy(big).cuda()[::3, 10:40]
    X = big[::3, 10:40]
    _same(_run(C, t, labels, 3), reference(X, labels, 3))


def test_block_past_2_31_terms(C):
    """Two clusters of 46 341 one-feature rows: blocks of 2 147 488 281 terms (64-bit offsets).  The reference sums the
    block's pairwise tree down to subtrees of at most 2^24 terms with np.add.reduce (one pairwise sum, so a subtree's sum
    is NumPy's) over the flattened rows of cdist."""
    rng = np.random.default_rng(4)
    n = 46341
    X = rng.normal(size=(2 * n, 1)) * 10.0
    labels = np.repeat([0, 1], n)
    rng.shuffle(labels)

    def block_mean(xa, xb):
        n2 = xb.shape[0]

        def flat(a, b):
            r0, r1 = a // n2, (b - 1) // n2 + 1
            return distance.cdist(xa[r0:r1], xb).ravel()[a - r0 * n2:b - r0 * n2]

        def tree(a, n_terms):
            if n_terms <= 1 << 24:
                return np.add.reduce(flat(a, a + n_terms))
            h = n_terms // 2
            h -= h % 8
            return tree(a, h) + tree(a + h, n_terms - h)
        return tree(0, xa.shape[0] * n2) / (xa.shape[0] * n2)

    A, B = _run(C, X, labels, 2)
    x0, x1 = X[labels == 0], X[labels == 1]
    assert B[0, 1].view(np.uint64) == np.float64(block_mean(x0, x1)).view(np.uint64)
    assert B[1, 0].view(np.uint64) == np.float64(block_mean(x1, x0)).view(np.uint64)
    assert np.isnan(A).all()                                     # one feature: pdist is empty


def test_streams_and_threads(C):
    """Four threads, each on a stream of its own, each its own clustering of one shared matrix."""
    import torch
    rng = np.random.default_rng(5)
    X = rng.normal(size=(2000, 40))
    t = torch.from_numpy(X).cuda()
    labels = [rng.integers(0, k, size=2000) for k in (2, 3, 5, 9)]
    want = [reference(X, lab, k) for lab, k in zip(labels, (2, 3, 5, 9))]
    got = [None] * 4
    errors = []

    def work(i):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(3):
                    A, B = C.cluster_distance_means(t, labels[i], (2, 3, 5, 9)[i])
                got[i] = (A.cpu().numpy(), B.cpu().numpy())
        except Exception as exc:          # reported below
            errors.append(exc)

    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for g, w in zip(got, want):
        _same(g, w)


def test_refusals(C):
    import torch
    X = torch.zeros((4, 3), dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError):
        C.cluster_distance_means(X.float(), [0, 1, 0, 1], 2)
    with pytest.raises(ValueError):
        C.cluster_distance_means(X, [0, 1, 0], 2)
    with pytest.raises(ValueError):
        C.cluster_distance_means(X, [0, 1, 0, 2], 2)                 # a label >= K: B200AA_ERR_INVALID

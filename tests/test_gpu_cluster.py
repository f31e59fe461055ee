"""GPU: kernel 9 (b200aa_cluster_distance_means, consumers.cluster_distance_means) bit for bit np.mean of scipy's pdist /
cdist on seeded clusterings up to 36 000 rows; at the distance kernel's tile and chunk edges; on each path of the plan
(tests/cluster_cases.py); on the adversarial value bank; with subsets of 1 024 clusters packed into other passes; on
strided, column-major and one-row inputs; on a block past 2^31 terms; across streams and threads; and the wrapper's
refusal of labels and rows that are not cluster ids."""
import threading

import numpy as np
import pytest
from scipy.spatial import distance

from tests.cluster_cases import EDGE_D, EDGE_SIZES, PLAN_CASES, adversarial, labels_of
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


def _scaled(rng, n, D):
    return rng.normal(size=(n, D)) * np.exp(rng.uniform(-4, 4, size=(1, D))) + rng.normal(size=(1, D))


@pytest.mark.parametrize("D", EDGE_D)
def test_tile_and_chunk_edges(C, D):
    """Ten clusters of 1 to 129 rows at D below, at and past multiples of 16 and 64: block tiles end at the cluster sizes
    and their 16-term chunks at D; pdist tiles (and the diagonal tiles its triangle keeps) end at D and its chunks at the
    cluster sizes."""
    rng = np.random.default_rng(100 + D)
    labels = labels_of(rng, EDGE_SIZES)
    X = _scaled(rng, labels.size, D)
    _same(_run(C, X, labels, len(EDGE_SIZES)), reference(X, labels, len(EDGE_SIZES)))


@pytest.mark.parametrize("case", PLAN_CASES, ids=lambda c: c.name)
def test_plan_paths(C, case):
    """Clusterings that make the plan take each of its paths (tests/test_cluster_cpu.py checks that they still do): a
    pdist mean just under and just past one segment, two pdist means at D = 4096 filling a pass, blocks of exactly one
    segment and one row past it, and blocks split into segments spread over several passes."""
    rng = np.random.default_rng(sum(case.sizes) + case.D)
    labels = labels_of(rng, case.sizes)
    X = _scaled(rng, labels.size, case.D)
    _same(_run(C, X, labels, len(case.sizes)), reference(X, labels, len(case.sizes)))


@pytest.mark.parametrize("sizes,D", [((1, 16, 17, 65, 130), 17), ((2, 63, 64, 70), 65), ((3, 129, 40), 130),
                                     ((1, 7, 66), 1), ((0, 5, 66, 1), 33)])
def test_extreme_values(C, sizes, D):
    """The adversarial bank (+-0, subnormals, e^-40 to e^40, +-1e300 whose squares overflow, NaN, +-inf) across tile
    edges, with one-row clusters; then again with one cluster's rows all NaN.  A stays NaN for D = 1; for D >= 2 an empty
    cluster has A[c] = +0.0 (scipy's pdist of D points with no coordinates is all zeros) and NaN blocks."""
    rng = np.random.default_rng(sum(sizes) * D)
    K = len(sizes)
    labels = labels_of(rng, sizes)
    X = adversarial(rng, labels.size, D, nonfinite=max(1, labels.size * D // 200))
    X[~np.isfinite(X) & (labels != 1)[:, None]] = -0.0             # NaN and inf in cluster 1 only
    X[(np.abs(X) == 1e300) & (labels > 1)[:, None]] = -0.0         # +-1e300 in clusters 0 and 1 only
    want = reference(X, labels, K)
    tame = np.array([c > 1 and sizes[c] > 0 for c in range(K)])    # their means are finite
    assert np.isfinite(want[1][np.ix_(tame, tame)][~np.eye(tame.sum(), dtype=bool)]).all()
    assert D == 1 or np.isfinite(want[0][tame]).all()
    got = _run(C, X, labels, K)
    _same(got, want)
    if D == 1:
        assert np.isnan(got[0]).all()
    for c in np.flatnonzero(np.asarray(sizes) == 0):
        assert D == 1 or got[0][c].view(np.uint64) == 0
        assert np.isnan(got[1][c]).all() and np.isnan(got[1][:, c]).all()
    X[labels == 2] = np.nan
    _same(_run(C, X, labels, K), reference(X, labels, K))


def test_rows_subsets_pack_other_passes(C):
    """At K = B200AA_CLUSTER_MAX, each requested cluster's A[c] and B[c, :] are the bits of the call over every cluster,
    whose means fill three passes, whichever other clusters are requested with it (so whatever passes its segments land
    in); the clusters not requested stay NaN.  An empty and a one-row cluster are among them."""
    rng = np.random.default_rng(9)
    K = 1024
    labels = rng.integers(0, K, size=6000)
    labels[labels == 7] = 8                                      # cluster 7 empty
    labels[labels == 1023] = 1022
    labels[4321] = 1023                                          # cluster 1023 has one row
    X = _scaled(rng, labels.size, 8)
    A, B = _run(C, X, labels, K)
    for rows, check_reference in (([0, 7, 511, 512, 1023], True), ([3], True), (range(1, K, 2), False)):
        want = np.zeros(K, dtype=bool)
        want[list(rows)] = True
        a, b = _run(C, X, labels, K, rows)
        assert np.isnan(a[~want]).all() and np.isnan(b[~want]).all()
        _same((a[want], b[want]), (A[want], B[want]))
        if check_reference:
            rA, rB = reference(X, labels, K, want)
            _same((a[want], b[want]), (rA[want], rB[want]))


@pytest.mark.parametrize("layout", ["odd_stride_slice", "column_major", "one_row", "cuda_int64_labels"])
def test_input_layouts(C, layout):
    """Columns sliced from a wider matrix at an odd row stride; a column-major tensor (the wrapper copies it); n = 1 (one
    cluster of one row, the others empty); labels given as a CUDA int64 tensor."""
    import torch
    rng = np.random.default_rng(11)
    n, D, K = 333, 20, 4
    labels = rng.integers(0, K, size=n)
    lab = labels
    if layout == "odd_stride_slice":
        big = _scaled(rng, n, 37)
        t = torch.from_numpy(big).cuda()[:, 5:5 + D]
        X = big[:, 5:5 + D]
        assert t.stride(0) == 37
    elif layout == "column_major":
        X = _scaled(rng, n, D)
        t = torch.from_numpy(X.T.copy()).cuda().t()
        assert t.stride() == (1, n)
    elif layout == "one_row":
        X = _scaled(rng, 1, D)
        labels = lab = np.array([2])
        t = torch.from_numpy(X).cuda()
    else:
        X = _scaled(rng, n, D)
        t = torch.from_numpy(X).cuda()
        lab = torch.from_numpy(labels).cuda()
    _same(_run(C, t, lab, K), reference(X, labels, K))


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


@pytest.mark.parametrize("labels,rows", [
    ([0, 1, 0, 2 ** 32], None),                                  # int32 cast: cluster 0
    ([0, 1, 0, 2 ** 32 + 1], None),                              # int32 cast: cluster 1
    (np.array([0, 1, 0, 2 ** 32], dtype=np.uint64), None),
    ([0, 1, -0.5, 1], None),                                     # int32 cast: cluster 0
    ([0, 1.7, 0, 1], None),                                      # int32 cast: cluster 1
    ([0, 1, 0, np.nan], None),
    ([0, 1, 0, 1], [-1]),                                        # NumPy's index: cluster K - 1
    ([0, 1, 0, 1], [2]),
    ([0, 1, 0, 1], [0.5]),
], ids=["label_2^32", "label_2^32+1", "uint64_label_2^32", "label_-0.5", "label_1.7", "label_nan", "row_-1", "row_K",
        "row_0.5"])
def test_refuses_ids_outside_the_clusters(C, labels, rows):
    """Labels and rows that are not integers in [0, K) raise ValueError; the reference's X[labels == c] would leave
    those rows out of every cluster, and a cast or a negative index would put them in one."""
    import torch
    X = torch.ones((4, 3), dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError):
        C.cluster_distance_means(X, labels, 2, rows)


def test_accepts_integer_valued_labels(C):
    """Float labels that hold integers (-0.0 included) are cluster ids, as they are to NumPy's labels == c."""
    rng = np.random.default_rng(12)
    X = _scaled(rng, 30, 5)
    labels = rng.integers(0, 3, size=30).astype(np.float64)
    labels[labels == 0] = -0.0
    _same(_run(C, X, labels, 3), reference(X, labels, 3))

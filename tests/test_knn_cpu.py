"""CPU: the pieces of the kNN kernel (csrc/knn.cuh, __host__ __device__) run on the host by tests/knn_host.cu -- the distance
chain against scipy's cdist, the sort keys, and the radix selection, ordered pass and vote against the stable-sort oracle
and the reference's Knn.classify (tests/golden/knn.npz), bit for bit."""

import numpy as np
import pytest
from scipy.spatial.distance import cdist

from tests import host_exe
from tests.host_exe import bits, floats, hexes, run
from tests.conftest import load_golden
from tests.knn_oracle import knn_oracle, slots_of

pytestmark = pytest.mark.skipif(host_exe.nvcc() is None, reason="nvcc not available")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "knn_host.cu", "-O1")


def _dist(exe, v, x):
    out = run(exe, "dist %d %d %d %s %s\n" % (v.shape[0], v.shape[1], x.shape[0], hexes(v), hexes(x)))
    return np.array([floats(ln[1:]) for ln in out])


def _classify(exe, feats, labels, k, x):
    slots, C = slots_of(labels)
    N, F = feats.shape
    script = "classify %d %d %d %d %s %s %d %s\n" % (N, F, C, k, " ".join(map(str, slots)), hexes(feats), x.shape[0], hexes(x))
    out = run(exe, script)
    ids = np.array([int(ln[1]) for ln in out], dtype=np.int64)
    P = np.array([floats(ln[2:]) for ln in out]).reshape(len(out), C)
    return ids, P


def test_distance_matches_cdist(exe):
    rng = np.random.default_rng(3)
    for F in (1, 2, 7, 136, 138):
        v = rng.normal(size=(23, F)) * rng.choice([1e-3, 1.0, 1e3], size=(23, 1))
        x = rng.normal(size=(9, F))
        got = _dist(exe, v, x)
        assert np.array_equal(bits(got), bits(cdist(x, v))), F
        assert np.array_equal(bits(got), bits(cdist(v, x).T)), F          # the reference's argument order


def test_distance_hard_values(exe):
    rng = np.random.default_rng(4)
    specials = np.array([np.inf, -np.inf, np.nan, 5e-324, -5e-324, 2.2250738585072014e-308 / 3, 1e300, -1e300, 1e154, 0.0,
                         -0.0, 1.0])
    for F in (1, 3, 138):
        v = rng.normal(size=(30, F))
        x = rng.normal(size=(30, F))
        for a in (v, x):
            mask = rng.random(a.shape) < 0.3
            a[mask] = rng.choice(specials, size=mask.sum())
        v[0] = x[0]                                       # a zero distance
        got = _dist(exe, v, x)
        assert np.array_equal(bits(got), bits(cdist(x, v))), F


def test_key_order(exe):
    d = np.array([0.0, 5e-324, 1e-300, 0.5, 1.0, 1.0000000000000002, 1e300, np.inf, np.nan, -np.nan,
                  np.frombuffer(np.uint64(0x7ff0000000000001).tobytes(), dtype=np.float64)[0], -0.0])
    out = run(exe, "key %d %s\n" % (d.size, hexes(d).replace("-nan", "nan")))
    keys = [int(t, 16) for t in out[0][1:]]
    assert keys[:8] == sorted(keys[:8]) and len(set(keys[:8])) == 8          # finite ascending, then +inf
    assert keys[8] == keys[9] == keys[10] == 0x7ff8000000000000 > keys[7]  # every NaN one key, above +inf
    assert keys[11] == keys[0] == 0                                         # -0 == +0


def _selection_cases():
    rng = np.random.default_rng(5)
    cases = []
    feats = rng.normal(size=(40, 6))
    labels = rng.integers(0, 3, size=40).astype(np.float64)
    cases.append((feats, labels, rng.normal(size=(12, 6))))
    grid = rng.integers(0, 3, size=(50, 2)).astype(np.float64)                # integer grid: many exact distance ties
    cases.append((grid, rng.integers(0, 4, size=50).astype(np.float64), rng.integers(0, 3, size=(15, 2)).astype(np.float64)))
    base = rng.normal(size=(15, 4))                                           # duplicated rows under different labels
    cases.append((np.concatenate([base, base, base]), np.repeat([0.0, 1.0, 2.0], 15), np.concatenate([base[:5], rng.normal(size=(5, 4))])))
    lab = rng.choice([0.0, 2.0, 3.0, 0.5], size=30)                           # labels that skip a class or never count
    cases.append((rng.normal(size=(30, 5)), lab, rng.normal(size=(8, 5))))
    nanq = rng.normal(size=(6, 3))                                            # NaN / inf distances
    nanq[0, 1] = np.nan
    nanq[1, 0] = np.inf
    tr = rng.normal(size=(25, 3))
    tr[[3, 7], 2] = np.nan
    tr[11, 0] = -np.inf
    cases.append((tr, rng.integers(0, 2, size=25).astype(np.float64), nanq))
    cases.append((rng.normal(size=(1, 3)), np.array([0.0]), rng.normal(size=(3, 3))))     # N = 1
    return cases


def test_selection_matches_stable_oracle(exe):
    for feats, labels, x in _selection_cases():
        N = feats.shape[0]
        for k in sorted({1, 2, 13, max(N - 1, 1), N, N + 7}):
            ids, P = _classify(exe, feats, labels, k, x)
            ref_ids, ref_P = knn_oracle(feats, labels, k, x)
            assert np.array_equal(ids, ref_ids), (N, k)
            assert np.array_equal(P, ref_P), (N, k)


def test_golden_replay(exe):
    g = load_golden("knn.npz")
    for c in g["cases"]:
        ids, P = _classify(exe, g[c + "_features"], g[c + "_labels"], int(g[c + "_k"]), g[c + "_queries"])
        assert np.array_equal(ids, g[c + "_ids"]), c
        assert np.array_equal(P, g[c + "_P"]), c


def test_stable_oracle_matches_reference_goldens():
    """The oracle the GPU tests use is the reference's Knn.classify on every stored query."""
    g = load_golden("knn.npz")
    for c in g["cases"]:
        ids, P = knn_oracle(g[c + "_features"], g[c + "_labels"], int(g[c + "_k"]), g[c + "_queries"])
        assert np.array_equal(ids, g[c + "_ids"]) and np.array_equal(P, g[c + "_P"]), c
        d = np.sort(cdist(g[c + "_queries"], g[c + "_features"]), axis=1)
        k = int(g[c + "_k"])
        assert np.array_equal(d[:, k - 1], g[c + "_dk"]), c
        assert np.array_equal(d[:, k], g[c + "_dk1"]), c

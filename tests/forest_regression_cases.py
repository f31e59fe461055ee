"""Seeded training problems for kernel 13's regression builder (csrc/forest.cuh, build_regression_tree) and the
comparison of a trained regressor with scikit-learn's RandomForestRegressor fit: every tree's Tree.__getstate__ in bits,
the fitted attributes."""
import numpy as np


def problems():
    """(name, X, y) regression problems: targets whose sums show their order (a large offset plus small noise), tied
    integer ratings, rounded X with duplicated rows, constant and near-constant features, float32 collisions and +-0, a
    root impurity of 4 eps, tie blocks long enough to send update() backwards; n of 1 and 2; F of 1, 2, 136 and 138."""
    out = []
    r = np.random.RandomState(23)
    X = r.randn(300, 11)
    out.append(("offset_noise_11x300", X, 1e6 + r.randn(300) * 1e-3 + X[:, 0]))
    X = r.randn(900, 136)
    out.append(("offset_noise_136x900", X, 1234.5 + r.randn(900) * 1e-2 + 0.1 * X[:, 3]))
    X = r.randn(1500, 138)
    out.append(("gauss_138x1500", X, X[:, 0] * 2 + r.randn(1500)))
    out.append(("ratings_ties", np.round(r.randn(400, 7), 1), r.randint(1, 6, 400).astype(np.float64)))
    X = np.round(r.randn(500, 9), 1)
    X[250:] = X[:250]
    out.append(("dup_rows", X, np.round(r.randn(500) * 3)))
    X = r.randn(400, 8)
    X[:, 2] = 2.5
    X[:, 4] = 1.0 + np.where(r.rand(400) < 0.5, 0.0, 5e-8)
    X[:, 6] = np.where(X[:, 0] < 0, -1.0, X[:, 6])
    out.append(("constants", X, X[:, 1] + (X[:, 0] > 0) + r.randn(400) * 0.1))
    v = 1.0 + np.arange(300) * 2.0 ** -30
    X = np.stack([v, r.permutation(v), np.where(r.rand(300) < 0.5, 0.0, -0.0), r.randn(300)], 1)
    out.append(("f32_collisions_pm0", X, r.randn(300)))
    # root impurity 4 eps: EPSILON (eps) splits it, 10 eps would leave one leaf
    X = np.arange(8, dtype=np.float64).reshape(8, 1)
    out.append(("four_eps", X, 1.0 + np.array([0, 1] * 4) * 2.0 ** -24))
    # long tie blocks at the low end: the first candidates lie past the middle, so update() runs backwards
    X = np.concatenate([np.zeros(300), np.arange(60) * 1.0])[:, None] * np.ones((1, 2))
    X[:, 1] = r.permutation(X[:, 1])
    out.append(("reverse_update", X, r.randn(360) + 100.0))
    out.append(("one_row", r.randn(1, 2), np.array([3.5])))
    out.append(("two_rows_f1", np.array([[0.0], [1.0]]), np.array([1.0, 2.0])))
    out.append(("f1_large", r.randn(2000, 1), r.randn(2000)))
    out.append(("f2_ties", np.round(r.randn(600, 2), 0), r.randint(0, 3, 600) * 0.1))
    return out


def compare(got, ref):
    """Assert the GPU-built regressor equals scikit-learn's fit: trees in bits, every fitted attribute."""
    assert type(got) is type(ref)
    assert len(got.estimators_) == len(ref.estimators_)
    assert set(got.__dict__) == set(ref.__dict__), set(got.__dict__) ^ set(ref.__dict__)
    for k in set(ref.__dict__) - {"estimators_"}:
        a, b = got.__dict__[k], ref.__dict__[k]
        assert type(a) is type(b), k
        assert (a.get_params() == b.get_params()) if hasattr(b, "get_params") else a == b, k
    for i, (ta, tb) in enumerate(zip(got.estimators_, ref.estimators_)):
        assert set(ta.__dict__) == set(tb.__dict__), set(ta.__dict__) ^ set(tb.__dict__)
        for k in set(tb.__dict__) - {"tree_"}:
            assert type(ta.__dict__[k]) is type(tb.__dict__[k]) and ta.__dict__[k] == tb.__dict__[k], (i, k)
        sa, sb = ta.tree_.__getstate__(), tb.tree_.__getstate__()
        assert sa["max_depth"] == sb["max_depth"] and sa["node_count"] == sb["node_count"], (i, sa["node_count"], sb["node_count"])
        for f in sb["nodes"].dtype.names:
            a, b = np.ascontiguousarray(sa["nodes"][f]), np.ascontiguousarray(sb["nodes"][f])
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (i, f)
        assert sa["values"].shape == sb["values"].shape
        assert np.array_equal(sa["values"].view(np.uint64), sb["values"].view(np.uint64)), i


def same_state(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))

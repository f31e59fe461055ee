"""Seeded training problems for kernel 13 (csrc/forest.cuh) and the comparison of a trained forest with scikit-learn's
fit: every tree's Tree.__getstate__ field by field in bits, the estimators' fitted attributes and NumPy's global state."""
import numpy as np


def problems():
    """(name, X, y) training problems: feature counts 1, 2, 11, 136, 138; 1 to a few thousand rows; 1 to 10 classes and
    string labels; duplicated rows and ties; features constant everywhere or only inside a subtree; neighbours closer and
    farther than 1e-7; float64 values that collide as float32; +-0, subnormals and values near float32 max."""
    out = []
    r = np.random.RandomState(7)
    X = r.randn(300, 11)
    out.append(("gauss_11x300_c4", X, r.randint(0, 4, 300)))
    X = r.randn(1000, 136)
    out.append(("gauss_136x1000_c4", X, r.randint(0, 4, 1000)))
    X = r.randn(2500, 138)
    out.append(("gauss_138x2500_c10", X, r.randint(0, 10, 2500)))
    out.append(("one_row", r.randn(1, 2), np.array([3])))
    out.append(("two_rows_f1", np.array([[0.0], [1.0]]), np.array([0, 1])))
    out.append(("single_class", r.randn(40, 2), np.zeros(40, dtype=int)))
    out.append(("strings_f2", r.randn(200, 2), np.array(["speech", "music", "noise"])[r.randint(0, 3, 200)]))
    # duplicated rows and heavy ties
    X = np.round(r.randn(400, 11), 1)
    X[200:] = X[:200]
    out.append(("dups_ties", X, r.randint(0, 3, 400)))
    # constant in the whole matrix, and constant only where feature 0 is below 0 (inside the left subtree)
    X = r.randn(500, 11)
    X[:, 3] = 2.5
    X[:, 5] = np.where(X[:, 0] < 0, 1.0, r.randn(500))
    X[:, 7] = np.where(X[:, 1] > 0.3, -4.0, X[:, 7])
    y = (X[:, 0] > 0).astype(int) + 2 * (X[:, 5] > 0.5)
    out.append(("constants", X, y))
    # neighbours 5e-8 apart (one candidate group) and 3e-7 apart (separate), around 0 and 1
    base = np.repeat(np.arange(40) * 1e-6, 5)
    X = np.stack([base + np.tile([0, 5e-8, 1e-7, 3e-7, 6e-7], 40), 1.0 + base + np.tile([0, 2e-8, 5e-8, 2e-7, 4e-7], 40)], 1)
    out.append(("near_threshold", X, r.randint(0, 2, 200)))
    # float64 values that are equal as float32
    v = 1.0 + np.arange(300) * 2.0 ** -30
    X = np.stack([v, r.permutation(v), r.randn(300)], 1)
    out.append(("f32_collisions", X, r.randint(0, 3, 300)))
    # +-0, subnormals, values near float32 max (the halved-sum threshold)
    fmax = float(np.finfo(np.float32).max)
    sub = float(np.finfo(np.float32).smallest_subnormal)
    pool = np.array([0.0, -0.0, sub, -sub, 3 * sub, 1e-40, -1e-39, fmax, -fmax, fmax * 0.75, 1.0, -1.0])
    X = pool[r.randint(0, pool.size, (300, 2))]
    out.append(("extremes", X, r.randint(0, 2, 300)))
    return out


def palindrome(seed, n=40):
    """n (even) labels symmetric along the sorted values, so splits at p and n - p tie in exact arithmetic: the proxy's
    rounding decides between them (a fused multiply-add breaks the tie the other way for seed 39 at n = 40).  At n of a
    few hundred the tied positions fall in different threads' chunks of a 128-thread team."""
    r = np.random.RandomState(seed)
    h = r.randint(0, 3, n // 2)
    return np.stack([np.arange(float(n)), r.permutation(n).astype(float)], 1), np.concatenate([h, h[::-1]])


# root sizes at the builders' team and padding edges: the 128-thread team, and the bitonic sort's power-of-two padding
ROOT_SIZES = (127, 128, 129, 255, 256, 257, 1025)


def limits(seed=41, n=400):
    """(X, y) at the launchers' limits: 512 features (kMaxFeats) and 32 classes (kMaxClasses), each class present."""
    r = np.random.RandomState(seed)
    X = r.randn(n, 512)
    y = r.permutation(np.arange(n) % 32)
    X[:, :8] += 0.5 * (y[:, None] % 8 == np.arange(8))          # some signal, so the trees grow deep and wide
    return X, y


def duplicated_columns(seed, n=300, F=6, decimals=None):
    """(X, y) whose columns F .. 2F - 1 repeat columns 0 .. F - 1: every split found on one copy ties with the other, and
    the copy visited first must win; `decimals` rounds X so that the values tie within a column too."""
    r = np.random.RandomState(seed)
    X = r.randn(n, F) if decimals is None else np.round(r.randn(n, F), decimals)
    y = (X[:, 0] + X[:, 1] > 0).astype(int) + (X[:, 2] > 0.5)
    return np.hstack([X, X]), y


def compare(got, ref):
    """Assert the GPU-built estimator equals scikit-learn's fit: trees in bits, every fitted attribute."""
    assert type(got) is type(ref)
    assert len(got.estimators_) == len(ref.estimators_)
    assert set(got.__dict__) == set(ref.__dict__), set(got.__dict__) ^ set(ref.__dict__)
    for k in set(ref.__dict__) - {"estimators_", "classes_"}:
        a, b = got.__dict__[k], ref.__dict__[k]
        assert type(a) is type(b), k
        assert (a.get_params() == b.get_params()) if hasattr(b, "get_params") else a == b, k
    assert np.array_equal(got.classes_, ref.classes_) and got.classes_.dtype == ref.classes_.dtype
    for i, (ta, tb) in enumerate(zip(got.estimators_, ref.estimators_)):
        assert set(ta.__dict__) == set(tb.__dict__)
        for k in set(tb.__dict__) - {"tree_", "classes_"}:
            assert type(ta.__dict__[k]) is type(tb.__dict__[k]) and ta.__dict__[k] == tb.__dict__[k], (i, k)
        assert np.array_equal(ta.classes_, tb.classes_) and ta.classes_.dtype == tb.classes_.dtype
        sa, sb = ta.tree_.__getstate__(), tb.tree_.__getstate__()
        assert sa["max_depth"] == sb["max_depth"] and sa["node_count"] == sb["node_count"], (i, sa["node_count"], sb["node_count"])
        for f in sb["nodes"].dtype.names:
            a, b = np.ascontiguousarray(sa["nodes"][f]), np.ascontiguousarray(sb["nodes"][f])
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (i, f)
        assert sa["values"].shape == sb["values"].shape
        assert np.array_equal(sa["values"].view(np.uint64), sb["values"].view(np.uint64)), i


def same_state(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))

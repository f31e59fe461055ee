"""Seeded training problems for kernel 13's gradient boosting (csrc/forest.cuh boost_leaves) and the comparison of a
trained GradientBoostingClassifier with scikit-learn's fit: every tree's Tree.__getstate__ in bits, train_score_, init_,
classes_, and predict / predict_proba / decision_function on held-out rows."""
import numpy as np


def problems():
    """(name, X, y, n_estimators): binary, 3- and 10-class data, non-contiguous and string labels, tied and constant
    features, duplicated rows, tiny n (one-row leaves), trees cut off at depth 3."""
    out = []
    r = np.random.RandomState(31)
    X = r.randn(120, 6)
    out.append(("binary", X, (X[:, 0] + 0.5 * r.randn(120) > 0).astype(int), 6))
    X = r.randn(150, 8)
    out.append(("three_class", X, np.argmax(X[:, :3] + 0.7 * r.randn(150, 3), 1), 5))
    X = r.randn(300, 12)
    out.append(("ten_class", X, r.randint(0, 10, 300), 3))
    X = r.randn(90, 5)
    out.append(("labels_3_7_11", X, np.array([3, 7, 11])[r.randint(0, 3, 90)], 4))
    X = r.randn(80, 4)
    out.append(("string_labels", X, np.array(["music", "speech"])[(X[:, 1] > 0).astype(int)], 5))
    X = np.round(r.randn(140, 5), 1)
    X[:, 2] = 1.5
    X[:, 4] = np.where(X[:, 0] < 0, -1.0, X[:, 4])
    out.append(("ties_constants", X, np.argmax(X[:, :3] + r.randn(140, 3), 1), 5))
    X = np.round(r.randn(100, 4), 1)
    X[50:] = X[:50]
    out.append(("dup_rows", X, r.randint(0, 3, 100), 4))
    out.append(("tiny_binary", r.randn(5, 3), np.array([0, 1, 1, 0, 1]), 4))
    out.append(("tiny_three", r.randn(7, 2), np.array([0, 1, 2, 0, 1, 2, 2]), 3))
    out.append(("two_rows", np.array([[0.0], [1.0]]), np.array([0, 1]), 3))
    X = r.randn(200, 136)
    out.append(("f136_four_class", X, np.argmax(X[:, :4] + r.randn(200, 4), 1), 3))
    return out


def held_out(X, seed=5):
    """Rows near X's range for predict."""
    r = np.random.RandomState(seed)
    return X[r.randint(0, X.shape[0], 40)] + 0.05 * r.randn(40, X.shape[1])


def compare(got, ref, X_test):
    """Assert the GPU-trained classifier equals scikit-learn's fit: trees in bits, every fitted attribute, the same
    predictions."""
    assert type(got) is type(ref)
    assert set(got.__dict__) == set(ref.__dict__), set(got.__dict__) ^ set(ref.__dict__)
    assert got.estimators_.shape == ref.estimators_.shape
    assert np.array_equal(got.classes_, ref.classes_) and got.classes_.dtype == ref.classes_.dtype
    assert np.array_equal(got.train_score_.view(np.uint64), ref.train_score_.view(np.uint64))
    assert type(got._loss) is type(ref._loss) and got._rng is ref._rng
    for k in ("n_classes_", "n_trees_per_iteration_", "n_estimators_", "max_features_", "n_features_in_"):
        assert type(got.__dict__[k]) is type(ref.__dict__[k]) and got.__dict__[k] == ref.__dict__[k], k
    assert got.get_params() == ref.get_params()
    assert np.array_equal(got.init_.predict_proba(X_test[:3]), ref.init_.predict_proba(X_test[:3]))
    for (i, k), tb in np.ndenumerate(ref.estimators_):
        ta = got.estimators_[i, k]
        assert set(ta.__dict__) == set(tb.__dict__), set(ta.__dict__) ^ set(tb.__dict__)
        for a in set(tb.__dict__) - {"tree_"}:
            va, vb = ta.__dict__[a], tb.__dict__[a]
            assert type(va) is type(vb) and (va is vb or va == vb), (i, k, a)
        sa, sb = ta.tree_.__getstate__(), tb.tree_.__getstate__()
        assert sa["max_depth"] == sb["max_depth"] and sa["node_count"] == sb["node_count"], (i, k)
        for f in sb["nodes"].dtype.names:
            a, b = np.ascontiguousarray(sa["nodes"][f]), np.ascontiguousarray(sb["nodes"][f])
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (i, k, f)
        assert np.array_equal(sa["values"].view(np.uint64), sb["values"].view(np.uint64)), (i, k)
    assert np.array_equal(got.predict(X_test), ref.predict(X_test))
    assert np.array_equal(got.predict_proba(X_test).view(np.uint64), ref.predict_proba(X_test).view(np.uint64))
    assert np.array_equal(got.decision_function(X_test).view(np.uint64), ref.decision_function(X_test).view(np.uint64))


def same_state(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))

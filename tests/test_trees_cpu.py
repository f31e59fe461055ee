"""CPU: the pieces of the tree-ensemble kernel (csrc/trees.cuh, __host__ __device__) run on the host by tests/trees_host.cu
over the arrays consumers.flatten_tree_ensemble makes, bit for bit scikit-learn's predict / predict_proba (and gradient
boosting's raw scores) on seeded forests and boosting models and adversarial query banks; the flattening against the
tree_ attributes; the refusals; and the argument checks of b200aa_trees_create / b200aa_trees_classify."""
import ctypes
import subprocess

import numpy as np
import pytest

from tests import host_exe
from tests import tree_models as TM

pytestmark = pytest.mark.skipif(host_exe.nvcc() is None, reason="nvcc not available")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "trees_host.cu", "-O1")


@pytest.fixture(scope="module")
def models():
    return TM.models()


def _flat(model):
    from pyaudioanalysis_b200.consumers import flatten_tree_ensemble
    return flatten_tree_ensemble(model)


def _host(exe, tmp_path, flat, X, dtype=np.float64):
    X = np.ascontiguousarray(X, dtype=dtype)
    C, n = flat["n_classes"], X.shape[0]
    init = flat["init"]
    head = np.array([flat["nodes"].shape[0], flat["roots"].size, flat["values"].shape[0], flat["mode"], C, flat["n_feats"],
                     int(flat["allow_nan"]), 1 if dtype == np.float32 else 2, n, init is not None], dtype=np.int64)
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        for a in (head, flat["nodes"], flat["roots"], flat["values"]) + ((init,) if init is not None else ()) + (X,):
            f.write(np.ascontiguousarray(a).tobytes())
    res = subprocess.run([exe, src, dst], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw = open(dst, "rb").read()
    ids = np.frombuffer(raw, np.int64, n)
    bad = np.frombuffer(raw, np.int32, n, 8 * n)
    scores = np.frombuffer(raw, np.float64, n * C, 12 * n).reshape(n, C)
    return ids, bad, scores


def _check(exe, tmp_path, model, X, dtype=np.float64):
    """Host pieces == scikit-learn on every row it accepts; a flagged row is one scikit-learn refuses."""
    flat = _flat(model)
    ids, bad, scores = _host(exe, tmp_path, flat, X, dtype)
    Xq = np.asarray(X, dtype=dtype)
    for i in np.nonzero(bad)[0][:5]:
        with pytest.raises(ValueError):
            model.predict(Xq[i:i + 1])
    ok = bad == 0
    if not ok.any():
        return ids, bad
    good = Xq[ok]
    assert np.array_equal(model.classes_[ids[ok]], model.predict(good))
    if flat["mode"] == 0:
        assert np.array_equal(scores[ok], model.predict_proba(good))
    else:
        raw = model.decision_function(good)
        assert np.array_equal(scores[ok], raw.reshape(-1, flat["n_classes"]))
        assert np.array_equal(model._loss.predict_proba(scores[ok][:, 0] if flat["n_classes"] == 1 else scores[ok]),
                              model.predict_proba(good))
    return ids, bad


@pytest.mark.parametrize("name", ["rf4", "et4", "gb4", "rf2", "et2", "gb2", "gb2_zero", "rf1", "rf500", "labels_257",
                                  "labels_str", "labels_str_et", "one_leaf", "stump_leaf", "tie", "rf40", "gb40",
                                  "tie40"])
def test_query_bank_bit_for_bit(exe, tmp_path, models, name):
    model = models[name]
    X = TM.query_bank(model, seed=1)
    _, bad = _check(exe, tmp_path, model, X)
    assert not bad.any()
    _, bad = _check(exe, tmp_path, model, X.astype(np.float32), np.float32)
    assert not bad.any()


@pytest.mark.parametrize("name", ["rf_nan", "et_nan", "rf4", "et4"])
def test_nan_in_split_features_of_forests(exe, tmp_path, models, name):
    """Forests take NaN (scikit-learn 1.9 walks it by missing_go_to_left, set even without NaN in training)."""
    model = models[name]
    flat = _flat(model)
    assert flat["allow_nan"]
    X = TM.query_bank(model, seed=2, nan=True)
    _, bad = _check(exe, tmp_path, model, X)
    assert not bad.any()
    _check(exe, tmp_path, model, X.astype(np.float32), np.float32)


@pytest.mark.parametrize("name", ["gb4", "gb2", "rf4", "labels_str"])
def test_refused_rows_flagged(exe, tmp_path, models, name):
    model = models[name]
    X = np.concatenate([TM.refused_rows(), TM.query_bank(model, seed=3)[:50]])
    if name.startswith("gb") or name == "labels_str":
        X[30, 2] = np.nan                                   # boosting refuses NaN
    _, bad = _check(exe, tmp_path, model, X)
    assert bad[:4].all()
    assert bad[30] == (name != "rf4")
    assert bad.sum() == 4 + int(name != "rf4")


def test_argmax_tie_is_first_maximum(exe, tmp_path, models):
    model = models["tie"]
    X = TM.query_bank(model, seed=4)
    flat = _flat(model)
    ids, _, scores = _host(exe, tmp_path, flat, X)
    tied = scores[:, 0] == scores[:, 1]
    assert tied.any() and (ids[tied] == 0).all()
    _check(exe, tmp_path, model, X)


def test_40_class_ties_span_lanes(models):
    """The 40-class tie model exercises the kernel's several classes per lane: some rows' maxima tie between a class
    below 32 and one at or above it, both on one lane (c and c + 32) and on different lanes."""
    model = models["tie40"]
    P = model.predict_proba(TM.query_bank(model, seed=1))
    top = [np.flatnonzero(p == p.max()) for p in P]
    assert any(t[0] < 32 <= t[-1] and any((c - t[0]) % 32 == 0 for c in t[1:]) for t in top)
    assert any(t[0] < 32 <= t[-1] and any((c - t[0]) % 32 != 0 for c in t[1:] if c >= 32) for t in top)


def test_one_leaf_trees_present(models):
    for name in ("one_leaf", "stump_leaf"):
        assert any(e.tree_.node_count == 1 for e in models[name].estimators_), name


def test_flattening_matches_tree_attributes(models):
    for name in ("rf4", "gb4", "gb2", "rf_nan", "one_leaf"):
        model = models[name]
        flat = _flat(model)
        nodes, roots, values = flat["nodes"], flat["roots"], flat["values"]
        trees = [e.tree_ for e in np.ravel(model.estimators_)]
        assert roots.size == len(trees) and roots[0] == 0
        leaf_base = 0
        for t, tr in enumerate(trees):
            nd = nodes[roots[t]:roots[t] + tr.node_count]
            leaf = tr.children_left < 0
            assert np.array_equal(nd[~leaf, 0], tr.children_left[~leaf] + roots[t])
            assert np.array_equal(nd[~leaf, 1], tr.children_right[~leaf] + roots[t])
            assert (nd[leaf, 0] == -1).all()
            assert np.array_equal(nd[leaf, 1], leaf_base + np.arange(leaf.sum()))
            feat = nd[~leaf, 2].view(np.uint32)
            assert np.array_equal(feat & 0x7fffffff, tr.feature[~leaf])
            assert np.array_equal((feat >> 31).astype(bool), tr.missing_go_to_left[~leaf].astype(bool))
            thr = nd[~leaf, 3].view(np.float32)
            t64 = tr.threshold[~leaf]
            assert (thr.astype(np.float64) <= t64).all()
            assert ((thr.astype(np.float64) == t64) | (np.nextafter(thr, np.float32(np.inf)).astype(np.float64) > t64)).all()
            rows = values[leaf_base:leaf_base + leaf.sum()]
            if flat["mode"] == 0:
                assert np.array_equal(rows, tr.value[leaf, 0, :flat["n_classes"]])
            else:
                assert np.array_equal(rows, model.learning_rate * tr.value[leaf, 0, 0])
            leaf_base += int(leaf.sum())
        assert values.shape[0] == leaf_base


def test_thresholds_mostly_not_float32(models):
    """Rounding is exercised: most thresholds of a forest lie strictly between two float32 values."""
    thr = np.concatenate([e.tree_.threshold[e.tree_.children_left >= 0] for e in models["rf4"].estimators_])
    assert np.mean(thr.astype(np.float32).astype(np.float64) != thr) > 0.3


def test_refusals():
    from sklearn.dummy import DummyClassifier
    from sklearn.ensemble import GradientBoostingRegressor, RandomForestRegressor
    from sklearn.svm import SVC
    from pyaudioanalysis_b200.consumers import flatten_tree_ensemble
    from sklearn.ensemble import GradientBoostingClassifier, RandomForestClassifier
    X, y = TM.dataset(n=120)
    bad = [RandomForestClassifier(3, random_state=0).fit(X, np.stack([y, y % 2], axis=1)),
           GradientBoostingClassifier(n_estimators=3, init=DummyClassifier(strategy="most_frequent")).fit(X, y),
           RandomForestRegressor(3).fit(X, y.astype(float)), GradientBoostingRegressor(n_estimators=3).fit(X, y.astype(float)),
           SVC(probability=True).fit(X, y), RandomForestClassifier(3)]
    for m in bad:
        with pytest.raises(ValueError):
            flatten_tree_ensemble(m)


def test_abi_argument_checks():
    """Every argument error of b200aa_trees_create / _classify is B200AA_ERR_INVALID, found before any CUDA call."""
    from pyaudioanalysis_b200._lib import ERR_INVALID, lib
    model = TM.models()["rf2"]
    flat = _flat(model)
    nodes, roots, values = flat["nodes"].copy(), flat["roots"].copy(), flat["values"].copy()

    def create(nodes=nodes, roots=roots, values=values, n_nodes=None, n_trees=None, n_leaves=None, C=2, F=TM.F, mode=0,
               init=None, out=True):
        h = ctypes.c_void_p()
        return lib().b200aa_trees_create(
            ctypes.byref(h) if out else None, None if nodes is None else ctypes.c_void_p(nodes.ctypes.data),
            flat["nodes"].shape[0] if n_nodes is None else n_nodes, None if roots is None else ctypes.c_void_p(roots.ctypes.data),
            flat["roots"].size if n_trees is None else n_trees, None if values is None else ctypes.c_void_p(values.ctypes.data),
            flat["values"].shape[0] if n_leaves is None else n_leaves, C, F, mode,
            None if init is None else ctypes.c_void_p(init.ctypes.data), 0)

    cases = [dict(out=False), dict(nodes=None), dict(roots=None), dict(values=None), dict(n_nodes=0), dict(n_trees=0),
             dict(n_leaves=0), dict(C=0), dict(F=0), dict(mode=2), dict(mode=1)]
    for kw in cases:
        assert create(**kw) == ERR_INVALID, kw
    internal = np.nonzero(nodes[:, 0] >= 0)[0]
    leaves = np.nonzero(nodes[:, 0] < 0)[0]
    i = int(internal[1])
    for col, v in ((0, i), (0, nodes.shape[0]), (1, i), (1, -1), (2, TM.F), (2, TM.F | 0x40000000)):
        bad = nodes.copy()
        bad[i, col] = v
        assert create(nodes=bad) == ERR_INVALID, (col, v)
    bad = nodes.copy()
    bad[int(leaves[0]), 1] = values.shape[0]
    assert create(nodes=bad) == ERR_INVALID
    bad = nodes.copy()
    bad[int(internal[0]), 0] = roots[1]                    # a child in the next tree
    assert create(nodes=bad) == ERR_INVALID
    for r in (roots + 1, roots[::-1].copy(), np.concatenate([roots[:1], roots[:1], roots[2:]]).astype(np.int32)):
        assert create(roots=np.ascontiguousarray(r, dtype=np.int32)) == ERR_INVALID, r
    assert create(n_nodes=int(roots[-1])) == ERR_INVALID     # the last tree empty
    z = np.zeros(8)
    assert lib().b200aa_trees_classify(None, z.ctypes.data, 2, 1, TM.F, TM.F, z.ctypes.data, z.ctypes.data, z.ctypes.data,
                                       None) == ERR_INVALID

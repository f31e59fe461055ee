"""CPU: kernel 13's gradient boosting stage (csrc/forest.cuh build_regression_tree with max_depth 3, boost_leaves) run on
the host by tests/boosting_host.cu with teams of 1, 3 and 8 threads (tests/team_host.h), driven stage by stage with scikit-learn's own loss (pyaudioanalysis_b200.boosting),
against GradientBoostingClassifier.fit on the case bank (tests/boosting_cases.py): every tree in bits, train_score_,
init_, classes_, NumPy's global state and the predictions.  Also: one stage on crafted gradients against scikit-learn's own
_update_terminal_regions, named mutants caught (those of the team-parallel code at a team of 3), a ThreadSanitizer build
free of races that finds a deleted barrier, the refusals, the entry points' argument checks and the scratch refusal."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import boosting_cases as BC
from tests import host_exe

pytestmark = pytest.mark.skipif(host_exe.nvcc() is None, reason="nvcc not available")

CSRC = os.path.join(host_exe.ROOT, "pyaudioanalysis_b200", "csrc")


def _build(tmp_path_factory, replaces=(), flags=("-O1",)):
    """The harness over forest.cuh, or over a copy with (old, new) replacements made (a mutant)."""
    inc = CSRC
    if replaces:
        src = open(os.path.join(CSRC, "forest.cuh")).read()
        for old, new in replaces:
            assert src.count(old) == 1, old
            src = src.replace(old, new)
        d = tmp_path_factory.mktemp("mutant")
        (d / "forest.cuh").write_text(src)
        inc = str(d)
    return host_exe.build(tmp_path_factory, "boosting_host.cu", *flags, "-I" + inc, "-I" + CSRC)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _build(tmp_path_factory)


def stage_input(tmp_path, X32, neg_g, y, raw, seeds, lr=0.1):
    """The harness's input for one stage: (src, dst)."""
    n, F = X32.shape
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        for a in (np.array([n, F, raw.shape[1]], np.int64), X32.astype(np.float32), neg_g.astype(np.float64),
                  np.asarray(y, np.int32), raw.astype(np.float64), np.asarray(seeds, np.uint32), np.float64(lr)):
            f.write(np.ascontiguousarray(a).tobytes())
    return src, dst


def host_stage(exe, tmp_path, X32, neg_g, y, raw, seeds, lr=0.1, team=1):
    """One stage through the harness with a team of `team` threads: ([(node_count, max_depth, nodes, values)] per tree,
    raw after the stage)."""
    from pyaudioanalysis_b200 import forests as FO
    n, F = X32.shape
    K = raw.shape[1]
    src, dst = stage_input(tmp_path, X32, neg_g, y, raw, seeds, lr)
    res = subprocess.run([exe, "stage", src, dst, str(team)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw_out, off, trees = open(dst, "rb").read(), 0, []
    for _ in range(K):
        nc, md = np.frombuffer(raw_out, np.int64, 2, off)
        off += 16
        nodes = np.frombuffer(raw_out, FO.NODE_DTYPE, nc, off)
        off += FO.NODE_DTYPE.itemsize * nc
        vals = np.frombuffer(raw_out, np.float64, nc, off)
        off += 8 * nc
        trees.append(FO.tree_state(nodes, vals, md, 1))
    return trees, np.frombuffer(raw_out, np.float64, n * K, off).reshape(n, K).copy()


def host_fit(exe, tmp_path, X, y, T, team=1):
    """GradientBoostingClassifier(T).fit(X, y) with every stage's trees built by the host harness."""
    from pyaudioanalysis_b200 import boosting as BO
    est, X32, y_enc, raw0 = BO.begin(X, y, T)
    K = est.n_trees_per_iteration_
    seeds = BO.draw_seeds(T * K)
    raw = np.ascontiguousarray(np.broadcast_to(raw0, (X32.shape[0], K)))
    factor, sw = BO.loss_factor(est._loss), np.ones(X32.shape[0])
    for i in range(T):
        states, raw = host_stage(exe, tmp_path, X32, BO.neg_gradient(est._loss, y_enc, raw), y_enc, raw,
                                 seeds[i * K:(i + 1) * K], team=team)
        est.train_score_[i] = factor * est._loss(y_true=y_enc, raw_prediction=raw, sample_weight=sw)
        for k, s in enumerate(states):
            est.estimators_[i, k] = BO.make_tree(est, X32.shape[1], s)
    est.n_estimators_ = T
    return est


def _check(exe, tmp_path, X, y, T, seed=7, team=1):
    from sklearn.ensemble import GradientBoostingClassifier
    np.random.seed(seed)
    got = host_fit(exe, tmp_path, X, y, T, team)
    s_got = np.random.get_state()
    np.random.seed(seed)
    ref = GradientBoostingClassifier(n_estimators=T).fit(X, y)
    assert BC.same_state(s_got, np.random.get_state())
    BC.compare(got, ref, BC.held_out(X))


@pytest.mark.parametrize("case,team", host_exe.team_params(BC.problems()))
def test_fit_equals_sklearn(exe, tmp_path, case, team):
    _, X, y, T = case
    _check(exe, tmp_path, X, y, T, team=team)


def _sk_stage(X32, neg_g, y_enc, raw, seeds, lr=0.1):
    """One stage as _fit_stage runs it, on given negative gradients: scikit-learn's own tree (random_state
    RandomState(seeds[k])) and _update_terminal_regions."""
    from sklearn._loss.loss import HalfBinomialLoss, HalfMultinomialLoss
    from sklearn.ensemble._gb import _update_terminal_regions
    from sklearn.tree import DecisionTreeRegressor
    K = raw.shape[1]
    loss = HalfBinomialLoss() if K == 1 else HalfMultinomialLoss(n_classes=K)
    raw = raw.copy()
    states = []
    for k in range(K):
        t = DecisionTreeRegressor(max_depth=3, random_state=np.random.RandomState(int(seeds[k])))
        t.fit(X32, np.ascontiguousarray(neg_g[:, k]), sample_weight=np.ones(X32.shape[0]), check_input=False)
        yk = y_enc if K == 1 else (y_enc == k).astype(np.float64)
        _update_terminal_regions(loss, t.tree_, X32, yk, neg_g[:, k], raw, np.ones(X32.shape[0]),
                                 np.ones(X32.shape[0], bool), learning_rate=lr, k=k)
        states.append(t.tree_.__getstate__())
    return states, raw


@pytest.mark.parametrize("K", [1, 3])
def test_crafted_gradients_hit_the_guard(exe, tmp_path, K):
    """Gradients with prob = y_k - neg_g in {0, 1} give a zero Hessian: _safe_divide's 1e-150 guard sets the leaf to 0.0
    (0 / 0 would be NaN).  The rows left of x0 = 0 carry such gradients, the others ordinary ones; the stage equals
    scikit-learn's own tree and _update_terminal_regions."""
    r = np.random.RandomState(K)
    n = 64
    X32 = r.randn(n, 3).astype(np.float32)
    y = r.randint(0, 2 if K == 1 else K, n).astype(np.float64)
    left = X32[:, 0] < 0
    y[~left] = 1 if K == 1 else 0                   # one class right of x0 = 0: every column's target has one sign there
    onehot = y[:, None] if K == 1 else (y[:, None] == np.arange(K)).astype(np.float64)
    neg = np.where(left[:, None], 0.0, onehot - r.uniform(0.1, 0.9, (n, K)))       # left: prob = y_k in {0, 1}
    raw = r.randn(n, K)
    seeds = r.randint(0, 2 ** 31 - 1, K)
    rand_r = [np.random.RandomState(int(s)).randint(0, 2147483647) for s in seeds]
    trees, got_raw = host_stage(exe, tmp_path, X32, neg, y.astype(np.int32), raw, rand_r)
    ref_states, ref_raw = _sk_stage(X32, neg, y, raw, seeds)
    zero_leaves = 0
    for a, b in zip(trees, ref_states):
        assert a["node_count"] == b["node_count"] and a["max_depth"] == b["max_depth"]
        for f in b["nodes"].dtype.names:
            assert np.array_equal(np.ascontiguousarray(a["nodes"][f]).view(np.uint8),
                                  np.ascontiguousarray(b["nodes"][f]).view(np.uint8)), f
        assert np.array_equal(a["values"].view(np.uint64), b["values"].view(np.uint64))
        leaf = b["nodes"]["left_child"] == -1
        zero_leaves += int((b["values"][leaf, 0, 0] == 0.0).sum())
    assert zero_leaves >= 1
    assert np.array_equal(got_raw.view(np.uint64), ref_raw.view(np.uint64))


def host_predict(exe, tmp_path, raw):
    src, dst = str(tmp_path / "pin.bin"), str(tmp_path / "pout.bin")
    with open(src, "wb") as f:
        f.write(np.array(raw.shape, np.int64).tobytes() + np.ascontiguousarray(raw, np.float64).tobytes())
    res = subprocess.run([exe, "predict", src, dst], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return np.frombuffer(open(dst, "rb").read(), np.int32)


def test_predict_rule(exe, tmp_path):
    """boost_class is predict's rule: raw >= 0 (0.0 and -0.0 included) for one score, else the first maximum."""
    raw1 = np.array([[0.0], [-0.0], [1e-300], [-1e-300], [-2.0], [3.0]])
    assert host_predict(exe, tmp_path, raw1).tolist() == (raw1[:, 0] >= 0).astype(int).tolist()
    raw3 = np.array([[1.0, 1.0, 0.5], [0.0, 2.0, 2.0], [-1.0, -3.0, -1.0], [0.1, 0.2, 0.3]])
    assert host_predict(exe, tmp_path, raw3).tolist() == np.argmax(raw3, 1).tolist()


def _predict_cases(exe, tmp_path):
    raw1 = np.array([[0.0], [-0.0], [1.0], [-1.0]])
    return host_predict(exe, tmp_path, raw1).tolist() == [1, 1, 1, 0]


# (name, replacements): each mutant must fail at least one case of the bank, the crafted stage or the predict rule (those
# in TEAM_MUTANTS at a team of 3)
MUTANTS = [
    ("no_depth_limit", [("S.leaf = rec.depth >= T.max_depth || m < 2", "S.leaf = m < 2")]),
    ("partition_order", [("            const int32_t s = int32_t(q);\n", "            const int32_t s = T.samples[q];\n")]),
    ("running_sum", [("    return front::np_sum(get, cnt, true);",
                      "    double r = 0.0;\n    for (int64_t i = 0; i < cnt; ++i) r = dadd(r, get(i));\n    return r;")]),
    ("no_k_factor", [("    if (K > 1) num = dmul(num, ddiv(double(K - 1), double(K)));\n", "")]),
    ("no_guard", [("    return fabs(den) < 1e-150 ? 0.0 : ddiv(num, den);", "    return ddiv(num, den);")]),
    ("fma_raw_update", [("        r = dadd(r, dmul(B.lr, T.values[B.leaf_of[s]]));",
                         "        r = std::fma(B.lr, T.values[B.leaf_of[s]], r);")]),
    ("strict_binary_predict", [("    if (K == 1) return raw[0] >= 0.0 ? 1 : 0;", "    if (K == 1) return raw[0] > 0.0 ? 1 : 0;")]),
    # every thread writes its rows of a leaf from offset 0 instead of after the earlier threads' rows
    ("leaf_rows_from_zero", [("        for (int t = 0; t < tm.tid; ++t) o += B.part[t];\n", "")]),
]
TEAM_MUTANTS = {"leaf_rows_from_zero"}


@pytest.mark.parametrize("name", [m[0] for m in MUTANTS])
def test_mutants_are_caught(tmp_path_factory, tmp_path, name):
    exe = _build(tmp_path_factory, dict(MUTANTS)[name])
    team = 3 if name in TEAM_MUTANTS else 1
    failed = []
    if not _predict_cases(exe, tmp_path):
        failed.append("predict")
    for K in (1, 3):
        if team > 1:
            break
        try:
            test_crafted_gradients_hit_the_guard(exe, tmp_path, K)
        except AssertionError:
            failed.append("crafted%d" % K)
    for case, X, y, T in BC.problems():
        if failed:
            break
        try:
            _check(exe, tmp_path, X, y, min(T, 3), team=team)
        except AssertionError:
            failed.append(case)
    assert failed, name


# A barrier deleted from boost_leaves (thread 0 sums a leaf's rows before the other threads have written theirs): a race
# whose outcome depends on timing, so it is ThreadSanitizer's to find
SYNC_MUTANT = ("            if (B.leaf_of[s] == id) B.leaf_rows[o++] = s;\n        }\n        tm.sync();\n",
               "            if (B.leaf_of[s] == id) B.leaf_rows[o++] = s;\n        }\n")


@pytest.mark.parametrize("mutant", [False, True], ids=["builder", "deleted_sync"])
def test_thread_sanitizer(tmp_path_factory, tmp_path, monkeypatch, mutant):
    """The stage built with ThreadSanitizer, at a team of 4 on small binary and multiclass problems: no report (and the
    fit still equals scikit-learn's); with one barrier deleted, a data race is reported on every problem's first stage.
    The mutant's run is judged by its reports alone (host_exe.tsan_reports): after the racing read it may sum rows that
    are not the leaf's, crash or not end, as timing has it."""
    from pyaudioanalysis_b200 import boosting as BO
    tsan = _build(tmp_path_factory, [SYNC_MUTANT] if mutant else (), ("-O1",) + host_exe.tsan_flags())
    for name, X, y, T in [c for c in BC.problems() if c[0] in ("binary", "three_class", "tiny_three", "dup_rows")]:
        if mutant:
            np.random.seed(3)
            est, X32, y_enc, raw0 = BO.begin(X, y, 1)
            K = est.n_trees_per_iteration_
            raw = np.ascontiguousarray(np.broadcast_to(raw0, (X32.shape[0], K)))
            src, dst = stage_input(tmp_path, X32, BO.neg_gradient(est._loss, y_enc, raw), y_enc, raw, BO.draw_seeds(K))
            logs = tmp_path / ("tsan_" + name)
            assert "WARNING: ThreadSanitizer: data race" in host_exe.tsan_reports([tsan, "stage", src, dst, "4"], logs), name
        else:
            monkeypatch.setenv("TSAN_OPTIONS", "exitcode=0 log_path=%s" % (tmp_path / "tsan"))
            _check(tsan, tmp_path, X, y, 2, team=4)
    if not mutant:
        reports = "".join(p.read_text() for p in tmp_path.glob("tsan*"))
        assert reports == "", reports[:4000]


def test_refusals():
    from pyaudioanalysis_b200 import boosting as BO
    r = np.random.RandomState(0)
    X, y = r.randn(20, 3), r.randint(0, 3, 20)
    assert BO.unsupported(X, y, 10) is None
    bad = X.copy()
    bad[0, 0] = np.nan
    assert "NaN" in BO.unsupported(bad, y, 10)
    bad[0, 0] = 1e39                                        # finite in float64, inf as float32
    assert "NaN" in BO.unsupported(bad, y, 10)
    assert "1-d" in BO.unsupported(X, y[:, None], 10)
    assert "classification" in BO.unsupported(X, r.randn(20), 10)
    assert "one class" in BO.unsupported(X, np.zeros(20, int), 10)
    assert "features" in BO.unsupported(r.randn(5, 513), np.array([0, 1, 0, 1, 0]), 10)
    assert "n_estimators" in BO.unsupported(X, y, 0)
    assert "sample weights" in BO.unsupported(X, y, 10, sample_weight=np.ones(20))
    assert "hyper" in BO.unsupported(X, y, 10, learning_rate=0.2)
    import sklearn
    real = sklearn.__version__
    try:
        sklearn.__version__ = "1.8.2"
        assert "1.9" in BO.unsupported(X, y, 10)
    finally:
        sklearn.__version__ = real
    from pyaudioanalysis_b200 import forests as FO
    assert FO.unsupported(X, y, 10, "gradientboosting") is not None
    from pyaudioanalysis_b200 import audioTrainTest as at
    feats = [r.randn(10, 4), r.randn(12, 4)]
    assert at.unsupported(feats, "gradientboosting", [10, 25]) is None
    assert "SMOTE" in at.unsupported(feats, "gradientboosting", [10], smote=True)
    assert "512" in at.unsupported([r.randn(10, 513), r.randn(10, 513)], "gradientboosting", [10])


def test_train_gradient_boosting_refused_goes_to_sklearn():
    """A call the trainer refuses (here NaN in X) goes to scikit-learn unchanged, which raises its own error."""
    from pyaudioanalysis_b200 import audioTrainTest as at
    X = np.random.RandomState(1).randn(10, 3)
    X[0, 0] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        at.train_gradient_boosting(X, np.arange(10) % 2, 5)


def test_install_training_rebinds_boosting_where_present():
    import types
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    mod = types.ModuleType("standin_boosting")
    mod.evaluate_classifier = lambda *a, **k: None
    orig = (lambda *a: "original")
    mod.train_gradient_boosting = orig
    try:
        assert install_training(mod) == ["standin_boosting.evaluate_classifier", "standin_boosting.train_gradient_boosting"]
        assert mod.train_gradient_boosting is at.train_gradient_boosting
    finally:
        uninstall()
    assert mod.train_gradient_boosting is orig


def test_dispatcher_restores_the_state_on_a_single_class_split(monkeypatch):
    """A training split with one class (the reference's fit raises there): evaluate_classifier puts NumPy's state back
    and the dispatcher hands the whole call to the original, which then draws the same splits."""
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200 import boosting as BO
    seen = []

    def original(features, class_names, classifier_name, params, parameter_mode, **kw):
        seen.append(np.random.get_state())
        return "original"
    r = np.random.RandomState(2)
    feats = [r.randn(30, 4), r.randn(1, 4)]         # the second class's one row lands in the test set sometimes
    np.random.seed(3)
    before = np.random.get_state()
    assert at.dispatcher(original)(feats, ["a", "b"], "gradientboosting", [2, 3], 0, n_exp=20) == "original"
    assert len(seen) == 1 and BC.same_state(seen[0], before)
    np.random.seed(3)
    with pytest.raises(BO.SingleClass):
        at.evaluate_classifier(feats, ["a", "b"], "gradientboosting", [2, 3], 0, n_exp=20)
    assert BC.same_state(np.random.get_state(), before)


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _stage_args(n=6, F=2):
    dev = ctypes.c_void_p(16)                              # never dereferenced: every failing call refuses first
    a = dict(X=dev, n_rows=n, F=F, P=1, tro=np.array([0, 4], np.int64), tr=np.array([0, 1, 2, 3], np.int32),
             teo=np.array([0, 2], np.int64), te=np.array([4, 5], np.int32), K=np.array([3], np.int32),
             act=np.array([1], np.int32), y=dev, neg=dev, raw=dev, rawte=dev, seeds=np.ones(3, np.uint32), lr=0.1,
             nodes=None, vals=None, cap=0, cnt=None, dep=None)
    return a


def _stage(lib, a):
    def q(v):
        return _p(v) if isinstance(v, np.ndarray) else v
    return lib.b200aa_boosting_stage(q(a["X"]), a["n_rows"], a["F"], a["P"], q(a["tro"]), q(a["tr"]), q(a["teo"]),
                                     q(a["te"]), q(a["K"]), q(a["act"]), q(a["y"]), q(a["neg"]), q(a["raw"]), q(a["rawte"]),
                                     q(a["seeds"]), a["lr"], q(a["nodes"]), q(a["vals"]), a["cap"], q(a["cnt"]),
                                     q(a["dep"]), None)


def test_stage_argument_checks():
    """b200aa_boosting_stage refuses bad arguments before any CUDA call."""
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    bad = [dict(X=None), dict(tro=None), dict(tr=None), dict(K=None), dict(act=None), dict(y=None), dict(neg=None),
           dict(raw=None), dict(seeds=None), dict(n_rows=0), dict(F=0), dict(P=0), dict(lr=float("nan")),
           dict(lr=float("inf")), dict(te=None), dict(rawte=None), dict(tro=np.array([0, 0], np.int64)),
           dict(tro=np.array([1, 4], np.int64)), dict(tr=np.array([0, 1, 2, 6], np.int32)),
           dict(te=np.array([4, -1], np.int32)), dict(K=np.array([2], np.int32)), dict(K=np.array([33], np.int32)),
           dict(K=np.array([0], np.int32)), dict(act=np.array([2], np.int32)),
           dict(nodes=np.zeros(4, dtype=[("b", "u1", 48)])), dict(cap=-1)]
    for kw in bad:
        a = _stage_args()
        a.update(kw)
        assert _stage(lib, a) == L.ERR_INVALID, kw
    a = _stage_args(F=513)
    assert _stage(lib, a) == L.ERR_UNSUPPORTED
    # a training split of more rows than X has (here 7 of 6, one repeated) is accepted: F = 513 refuses it next
    a = _stage_args(F=513)
    a.update(tro=np.array([0, 7], np.int64), tr=np.array([0, 1, 2, 3, 4, 5, 0], np.int32))
    assert _stage(lib, a) == L.ERR_UNSUPPORTED
    # an input both invalid and over the feature limit is invalid
    for kw in (dict(tr=np.array([0, 1, 2, 6], np.int32)), dict(K=np.array([2], np.int32)), dict(rawte=None)):
        a = _stage_args(F=513)
        a.update(kw)
        assert _stage(lib, a) == L.ERR_INVALID, kw
    # an inactive problem's rows are checked, but it counts toward no size limit: nothing to build returns B200AA_OK
    # before any CUDA call, even for a training set over the scratch bound
    a = _stage_args(F=513)
    a.update(act=np.array([0], np.int32), te=np.array([4, 6], np.int32))
    assert _stage(lib, a) == L.ERR_INVALID
    n = 131073
    a = _stage_args(n=n, F=136)
    a.update(tro=np.array([0, n], np.int64), tr=np.arange(n, dtype=np.int32), teo=None, te=None, rawte=None,
             K=np.array([1], np.int32), act=np.array([0], np.int32), seeds=np.ones(1, np.uint32))
    assert _stage(lib, a) == L.OK


def test_scale_and_count_argument_checks():
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    dev = ctypes.c_void_p(16)
    tro, tr = np.array([0, 4], np.int64), np.array([0, 1, 2, 3], np.int32)
    teo, te = np.array([0, 2], np.int64), np.array([4, 5], np.int32)

    def q(v):
        return _p(v) if isinstance(v, np.ndarray) else v

    def scale(**kw):
        a = dict(X=dev, n=6, F=2, P=1, tro=tro, tr=tr, teo=teo, te=te, out=dev)
        a.update(kw)
        return lib.b200aa_boosting_scale(a["X"], a["n"], a["F"], a["P"], q(a["tro"]), q(a["tr"]), q(a["teo"]), q(a["te"]),
                                         a["out"], None)
    for kw in (dict(X=None), dict(out=None), dict(tr=None), dict(te=None), dict(n=0), dict(F=0), dict(P=0),
               dict(tr=np.array([0, 1, 2, 6], np.int32)), dict(te=np.array([-1, 5], np.int32)),
               dict(tro=np.array([0, 0], np.int64))):
        assert scale(**kw) == L.ERR_INVALID, kw
    K, cls, yt = np.array([1], np.int32), np.zeros((1, 32), np.int32), np.array([0, 1], np.int32)
    cls[0, :2] = [0, 2]

    def count(**kw):
        a = dict(raw=dev, P=1, teo=teo, K=K, cls=cls, yt=yt, C=3, pred=dev, counts=dev)
        a.update(kw)
        return lib.b200aa_boosting_count(a["raw"], a["P"], q(a["teo"]), q(a["K"]), q(a["cls"]), q(a["yt"]), a["C"],
                                         a["pred"], a["counts"], None)
    bad_cls = cls.copy()
    bad_cls[0, 1] = 3
    for kw in (dict(raw=None), dict(pred=None), dict(counts=None), dict(cls=None), dict(P=0), dict(C=1), dict(C=33),
               dict(K=np.array([2], np.int32)), dict(cls=bad_cls), dict(yt=np.array([0, 3], np.int32))):
        assert count(**kw) == L.ERR_INVALID, kw


def test_scratch_bound_refused_before_any_cuda_call():
    """A stage whose single tree's scratch passes the 256 MB bound (its sort keys alone take 8 F pow2(n) bytes: at F =
    136, n = 131 073 needs 285 MB) is B200AA_ERR_UNSUPPORTED before any CUDA call (so also without a GPU)."""
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    n = 131073
    a = _stage_args(n=n, F=136)
    a.update(tro=np.array([0, n], np.int64), tr=np.arange(n, dtype=np.int32), teo=None, te=None, rawte=None,
             K=np.array([1], np.int32), seeds=np.ones(1, np.uint32))
    assert _stage(lib, a) == L.ERR_UNSUPPORTED

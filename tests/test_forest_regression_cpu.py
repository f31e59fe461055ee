"""CPU: kernel 13's regression pieces (csrc/forest.cuh) run on the host by tests/forest_regression_host.cu: the
introsort_3way replay against scikit-learn's own simultaneous_sort permutation for permutation, and the tree builder, with
teams of 1, 3 and 8 threads (tests/team_host.h) fed by pyaudioanalysis_b200.forests' host draws, against
RandomForestRegressor.fit on the case bank (tests/forest_regression_cases.py): every tree's state in bits, the fitted
attributes and NumPy's global state.  Also: named mutants of the builder are caught (those of its team-parallel code at
a team of 3), a ThreadSanitizer build finds no race in the builder and finds a deleted barrier, the refusals, and the
argument checks of both entry points."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import forest_regression_cases as RC
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
    return host_exe.build(tmp_path_factory, "forest_regression_host.cu", *flags, "-I" + inc, "-I" + CSRC)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _build(tmp_path_factory)


def host_sort(exe, tmp_path, values, indices):
    src, dst = str(tmp_path / "sin.bin"), str(tmp_path / "sout.bin")
    n = values.size
    with open(src, "wb") as f:
        f.write(np.int64(n).tobytes() + values.astype(np.float32).tobytes() + indices.astype(np.int32).tobytes())
    res = subprocess.run([exe, "sort", src, dst], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw = open(dst, "rb").read()
    return np.frombuffer(raw, np.float32, n), np.frombuffer(raw, np.int32, n, 4 * n)


def fit_input(tmp_path, X, y, n_estimators):
    """The harness's input for the fit of X, y, drawn from NumPy's global state as fit draws: (src, dst, est, trees)."""
    from pyaudioanalysis_b200 import forests as FO
    n, F = X.shape
    est, trees, w, seeds = FO.draw(n_estimators, FO.REGRESSOR, n)
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        for a in (np.array([n, F, n_estimators], np.int64), X.astype(np.float32), np.asarray(y, np.float64), w, seeds):
            f.write(np.ascontiguousarray(a).tobytes())
    return src, dst, est, trees


def host_fit(exe, tmp_path, X, y, n_estimators, team=1):
    """The regressor fit builds, every tree built by the host harness with a team of `team` threads."""
    from pyaudioanalysis_b200 import forests as FO
    n, F = X.shape
    src, dst, est, trees = fit_input(tmp_path, X, y, n_estimators)
    res = subprocess.run([exe, "fit", src, dst, str(team)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw, off, states = open(dst, "rb").read(), 0, []
    for _ in range(n_estimators):
        nc, md = np.frombuffer(raw, np.int64, 2, off)
        off += 16
        nodes = np.frombuffer(raw, FO.NODE_DTYPE, nc, off)
        off += FO.NODE_DTYPE.itemsize * nc
        vals = np.frombuffer(raw, np.float64, nc, off)
        off += 8 * nc
        states.append(FO.tree_state(nodes, vals, md, 1))
    return FO.assemble_regressor(est, trees, F, n, states)


def _check(exe, tmp_path, X, y, n_estimators=3, seed=5, team=1):
    from sklearn.ensemble import RandomForestRegressor
    np.random.seed(seed)
    got = host_fit(exe, tmp_path, X, y, n_estimators, team)
    s_got = np.random.get_state()
    np.random.seed(seed)
    ref = RandomForestRegressor(n_estimators=n_estimators).fit(X, y)
    RC.compare(got, ref)
    assert RC.same_state(s_got, np.random.get_state())


def _sort_inputs():
    r = np.random.RandomState(3)
    out = [("all_equal_40", np.full(40, 2.5)), ("m15", r.randn(15)), ("m16", r.randn(16)), ("m16_ties", r.randint(0, 3, 16)),
           ("heavy_ties", r.randint(0, 4, 500)), ("pm0", np.where(r.rand(200) < 0.5, 0.0, -0.0)),
           ("pm0_mixed", np.where(r.rand(300) < 0.3, -0.0, np.where(r.rand(300) < 0.5, 0.0, r.randint(-2, 3, 300)))),
           ("distinct", r.randn(1000)), ("f32_collide", 1.0 + np.arange(300) * 2.0 ** -30), ("one", np.array([1.0])),
           ("sorted", np.arange(200.0)), ("reversed", np.arange(200.0)[::-1].copy())]
    # median-of-3 killers exhaust maxd and finish in heapsort: organ pipes and sawtooths with ties
    m = 1024
    out.append(("organ_pipe", np.concatenate([np.arange(m // 2), np.arange(m // 2)[::-1]]).astype(float)))
    out.append(("sawtooth", (np.arange(2000) % 37).astype(float)))
    k = np.arange(m)
    out.append(("m3_killer", np.where(k % 2 == 0, k // 2 + m // 2, k).astype(float)))
    return out


@pytest.mark.parametrize("case", [c[0] for c in _sort_inputs()])
def test_introsort_replay_equals_sklearn(exe, tmp_path, case):
    """introsort_3way restated equals scikit-learn's simultaneous_sort(use_three_way_partition=True): the same
    permutation, from the same (shuffled) starting order."""
    from sklearn.utils._sorting import _py_simultaneous_sort
    v = dict(_sort_inputs())[case].astype(np.float32)
    r = np.random.RandomState(len(case))
    for order in (np.arange(v.size), r.permutation(v.size)):
        vals, idx = v[order].copy(), order.astype(np.intp).copy()
        _py_simultaneous_sort(vals, idx, vals.size, use_three_way_partition=True)
        gv, gi = host_sort(exe, tmp_path, v[order], order)
        assert np.array_equal(gi, idx), case
        assert np.array_equal(gv.view(np.uint32), vals.view(np.uint32)), case


@pytest.mark.parametrize("case,team", host_exe.team_params(RC.problems(), big_rows=1500))
def test_trees_equal_sklearn(exe, tmp_path, case, team):
    name, X, y = case
    _check(exe, tmp_path, X, y, team=team)


# (name, replacements): each mutant must fail at least one problem of the bank (those in TEAM_MUTANTS at a team of 3)
MUTANTS = [
    ("stable_partition", [("    int64_t ps = 0, pe = m;\n",
                           "    int64_t k = 0;\n    for (int64_t p = 0; p < m; ++p)\n        if (double(x(samples[p])) <= threshold) {\n"
                           "            const int32_t t = samples[p];\n            for (int64_t q = p; q > k; --q) samples[q] = samples[q - 1];\n"
                           "            samples[k++] = t;\n        }\n    return;\n    int64_t ps = 0, pe = m;\n")]),
    ("pairwise_sum", [("            S.sum_total = st_;",
                       "            S.sum_total = npy::pairwise_sum([&](int64_t p) { return dmul(T.wv(smp[p]), T.yv(smp[p])); }, 0, m, m);")]),
    ("forward_only_update", [("    if (new_pos - pos <= m - new_pos) {", "    if (true) {")]),
    ("no_tie_replay", [("                    if (!T.tied[v]) continue;", "                    continue;")]),
    ("kEpsilon_leaf_tests", [("constexpr double kLeafEpsilon = DBL_EPSILON; ", "constexpr double kLeafEpsilon = kEpsilon; ")]),
    ("fma_sums", [("            sl = dadd(sl, dmul(w, T.yv(s)));", "            sl = std::fma(w, T.yv(s), sl);")]),
    # only thread 0's positions can mark a visit tied: visits whose ties lie in other threads' positions skip the replay
    ("tie_detection_thread0_only", [("                if (q >= 1 && key_value(T.keys[v * m2 + q - 1])",
                                     "                if (tm.tid == 0 && q >= 1 && key_value(T.keys[v * m2 + q - 1])")]),
]
TEAM_MUTANTS = {"tie_detection_thread0_only"}


@pytest.mark.parametrize("name", [m[0] for m in MUTANTS])
def test_mutants_are_caught(tmp_path_factory, tmp_path, name):
    exe = _build(tmp_path_factory, dict(MUTANTS)[name])
    team = 3 if name in TEAM_MUTANTS else 1
    failed = []
    for case, X, y in RC.problems():
        try:
            _check(exe, tmp_path, X, y, n_estimators=2, team=team)
        except AssertionError:
            failed.append(case)
    assert failed, name


# A barrier deleted from the builder (thread 0 reads every visit's best candidate before the other threads have written
# theirs): a race whose outcome depends on timing, so it is ThreadSanitizer's to find
SYNC_MUTANT = ("                T.vpos[v] = bq;\n            }\n            tm.sync();\n", "                T.vpos[v] = bq;\n            }\n")


@pytest.mark.parametrize("mutant", [False, True], ids=["builder", "deleted_sync"])
def test_thread_sanitizer(tmp_path_factory, tmp_path, monkeypatch, mutant):
    """The builder built with ThreadSanitizer, at a team of 4 on small problems (ties and replays included): no report
    (and the trees still equal scikit-learn's); with one barrier deleted, a data race is reported on every problem.  The
    mutant's run is judged by its reports alone (host_exe.tsan_reports): after the racing read it may index past its
    buffers, crash or not end, as timing has it."""
    tsan = _build(tmp_path_factory, [SYNC_MUTANT] if mutant else (), ("-O1",) + host_exe.tsan_flags())
    for name, X, y in [c for c in RC.problems() if c[0] in ("two_rows_f1", "four_eps", "ratings_ties", "f32_collisions_pm0")]:
        if mutant and X.shape[1] < 4:
            continue                            # one feature: thread 0 writes and reads the only visit's candidate itself
        if mutant:
            np.random.seed(3)
            src, dst = fit_input(tmp_path, X, y, 2)[:2]
            logs = tmp_path / ("tsan_" + name)
            assert "WARNING: ThreadSanitizer: data race" in host_exe.tsan_reports([tsan, "fit", src, dst, "4"], logs), name
        else:
            monkeypatch.setenv("TSAN_OPTIONS", "exitcode=0 log_path=%s" % (tmp_path / "tsan"))
            _check(tsan, tmp_path, X, y, n_estimators=2, team=4)
    if not mutant:
        reports = "".join(p.read_text() for p in tmp_path.glob("tsan*"))
        assert reports == "", reports[:4000]


def test_refusals():
    from pyaudioanalysis_b200 import forests as FO
    r = np.random.RandomState(0)
    X, y = r.randn(20, 3), r.randn(20)
    assert FO.unsupported_regressor(X, y, 10) is None
    bad = X.copy()
    bad[0, 0] = np.nan
    assert "NaN" in FO.unsupported_regressor(bad, y, 10)
    bad[0, 0] = np.inf
    assert "NaN" in FO.unsupported_regressor(bad, y, 10)
    assert "1-d" in FO.unsupported_regressor(X, y[:, None], 10)
    yb = y.copy()
    yb[3] = np.inf
    assert "y" in FO.unsupported_regressor(X, yb, 10)
    assert "features" in FO.unsupported_regressor(r.randn(5, 513), r.randn(5), 10)
    assert "n_estimators" in FO.unsupported_regressor(X, y, 0)
    assert "sample weights" in FO.unsupported_regressor(X, y, 10, sample_weight=np.ones(20))
    assert "hyper" in FO.unsupported_regressor(X, y, 10, max_depth=3)
    import sklearn
    real = sklearn.__version__
    try:
        sklearn.__version__ = "1.8.2"
        assert "1.9" in FO.unsupported_regressor(X, y, 10)
    finally:
        sklearn.__version__ = real
    from pyaudioanalysis_b200 import audioTrainTest as at
    feats, lab = r.randn(30, 4), r.randn(30)
    assert at.unsupported_regression(feats, lab, 2, "randomforest", [5, 10]) is None
    assert "svm" in at.unsupported_regression(feats, lab, 2, "svm", [1.0])
    assert "n_train" in at.unsupported_regression(feats[:2], lab[:2], 2, "randomforest", [5])
    assert "contiguous" in at.unsupported_regression(np.asfortranarray(feats), lab, 2, "randomforest", [5])
    assert "contiguous" in at.unsupported_regression(feats.astype(np.float32), lab, 2, "randomforest", [5])
    assert "integer" in at.unsupported_regression(feats, lab, 2, "randomforest", [5.0])


def test_install_training_rebinds_regression_where_present():
    """install_training rebinds evaluate_regression (through a dispatcher) and train_random_forest_regression only where
    the module has them, and uninstall restores them."""
    import types
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200.install import install_training, uninstall
    mod = types.ModuleType("standin_regression")
    mod.evaluate_classifier = lambda *a, **k: None
    orig_eval, orig_train = (lambda *a: "original"), (lambda *a: "original")
    mod.evaluate_regression, mod.train_random_forest_regression = orig_eval, orig_train
    names = install_training(mod)
    try:
        assert names == ["standin_regression.evaluate_classifier", "standin_regression.evaluate_regression",
                         "standin_regression.train_random_forest_regression"]
        assert mod.train_random_forest_regression is at.train_random_forest_regression
        assert mod.evaluate_regression.original is orig_eval
        r = np.random.RandomState(1)
        assert mod.evaluate_regression(r.randn(20, 3), r.randn(20), 2, "svm", [1.0]) == "original"
    finally:
        uninstall()
    assert mod.evaluate_regression is orig_eval and mod.train_random_forest_regression is orig_train


def test_abi_argument_checks():
    """b200aa_forest_regressor_fit refuses bad arguments before any CUDA call."""
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    n, F, T = 6, 2, 2
    y = np.arange(n, dtype=np.float64)
    w = np.ones((T, n), dtype=np.int32)
    seeds = np.ones(T, dtype=np.uint32)
    nodes = np.zeros(T * (2 * n - 1), dtype=[("b", "u1", 48)])
    vals = np.zeros(T * (2 * n - 1))
    cnt, dep = np.zeros(T, np.int64), np.zeros(T, np.int32)
    dev = ctypes.c_void_p(16)                              # never dereferenced: every call below fails its checks first

    def p(a):
        return ctypes.c_void_p(a.ctypes.data)

    def call(**kw):
        a = dict(d_X=dev, dtype=L.DTYPE_F64, n=n, F=F, stride=F, y=p(y), T=T, w=p(w), seeds=p(seeds), nodes=p(nodes),
                 vals=p(vals), cap=T * (2 * n - 1), cnt=p(cnt), dep=p(dep))
        a.update(kw)
        return lib.b200aa_forest_regressor_fit(a["d_X"], a["dtype"], a["n"], a["F"], a["stride"], a["y"], a["T"], a["w"],
                                               a["seeds"], a["nodes"], a["vals"], a["cap"], a["cnt"], a["dep"], None)
    ynan = y.copy()
    ynan[2] = np.nan
    yinf = y.copy()
    yinf[5] = -np.inf
    wneg = w.copy()
    wneg[1, 2] = -1
    for kw in (dict(d_X=None), dict(y=None), dict(w=None), dict(seeds=None), dict(nodes=None), dict(vals=None),
               dict(cnt=None), dict(dep=None), dict(n=0), dict(F=0), dict(stride=1), dict(T=0), dict(dtype=0), dict(cap=-1),
               dict(y=p(ynan)), dict(y=p(yinf)), dict(w=p(wneg))):
        assert call(**kw) == L.ERR_INVALID, kw
    assert call(F=513, stride=513) == L.ERR_UNSUPPORTED
    # an input both invalid and over the feature limit is invalid
    assert call(F=513, stride=513, y=p(ynan)) == L.ERR_INVALID
    assert call(F=513, stride=513, w=p(wneg)) == L.ERR_INVALID


def test_cross_validate_argument_checks():
    """b200aa_forest_regression_cross_validate refuses bad arguments before any CUDA call."""
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    n = 6
    y = np.arange(n, dtype=np.float64)
    tr_off, te_off = np.array([0, 4], np.int64), np.array([0, 2], np.int64)
    tr, te = np.array([0, 1, 2, 3], np.int32), np.array([4, 5], np.int32)
    nt, w, seeds = np.array([2], np.int32), np.ones((2, 4), np.int32), np.ones(2, np.uint32)
    dev = ctypes.c_void_p(16)

    def p(a):
        return ctypes.c_void_p(a.ctypes.data)

    def call(**kw):
        a = dict(X=dev, n=n, F=2, y=p(y), P=1, tro=p(tr_off), tr=p(tr), teo=p(te_off), te=p(te), nt=p(nt), w=p(w),
                 seeds=p(seeds), pte=dev, ptr=dev)
        a.update(kw)
        return lib.b200aa_forest_regression_cross_validate(a["X"], a["n"], a["F"], a["y"], a["P"], a["tro"], a["tr"],
                                                           a["teo"], a["te"], a["nt"], a["w"], a["seeds"], a["pte"],
                                                           a["ptr"], None)
    ynan = y.copy()
    ynan[0] = np.nan
    bad_tr = np.array([0, 1, 2, 6], np.int32)
    bad_te = np.array([4, -1], np.int32)
    bad_nt = np.array([0], np.int32)
    empty = np.array([0, 0], np.int64)
    wneg = w.copy()
    wneg[0, 0] = -3
    for kw in (dict(X=None), dict(y=None), dict(seeds=None), dict(w=None), dict(pte=None), dict(ptr=None), dict(n=0),
               dict(F=0), dict(P=0), dict(y=p(ynan)), dict(tr=p(bad_tr)), dict(te=p(bad_te)), dict(nt=p(bad_nt)),
               dict(tro=p(empty)), dict(w=p(wneg))):
        assert call(**kw) == L.ERR_INVALID, kw
    assert call(F=513) == L.ERR_UNSUPPORTED
    # a training split of more rows than X has (here 7 of 6, one repeated) is invalid
    long_off, long_tr = np.array([0, 7], np.int64), np.array([0, 1, 2, 3, 4, 5, 0], np.int32)
    assert call(tro=p(long_off), tr=p(long_tr), w=p(np.ones((2, 7), np.int32))) == L.ERR_INVALID
    # an input both invalid and over the feature limit is invalid
    assert call(F=513, y=p(ynan)) == L.ERR_INVALID
    assert call(F=513, te=p(bad_te)) == L.ERR_INVALID
    assert call(F=513, w=p(wneg)) == L.ERR_INVALID


def test_scratch_bound_refused_before_any_cuda_call():
    """A tree whose scratch would pass the 256 MB bound (its sort keys alone take 8 F pow2(n) bytes: at F = 136,
    n = 131 073 needs 8 x 136 x 262 144 = 285 MB) is B200AA_ERR_UNSUPPORTED in both entry points, before any CUDA call
    (so also on a machine without a GPU)."""
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    F, dev = 136, ctypes.c_void_p(16)                  # never dereferenced: both calls refuse first

    def p(a):
        return ctypes.c_void_p(a.ctypes.data)
    n = 131073
    y, w, seeds = np.zeros(n), np.ones((1, n), np.int32), np.ones(1, np.uint32)
    nodes = np.zeros(2 * n - 1, dtype=[("b", "u1", 48)])
    vals, cnt, dep = np.zeros(2 * n - 1), np.zeros(1, np.int64), np.zeros(1, np.int32)
    assert lib.b200aa_forest_regressor_fit(dev, L.DTYPE_F32, n, F, F, p(y), 1, p(w), p(seeds), p(nodes), p(vals),
                                           2 * n - 1, p(cnt), p(dep), None) == L.ERR_UNSUPPORTED
    tr_off, te_off = np.array([0, n], np.int64), np.array([0, 0], np.int64)
    tr, te = np.arange(n, dtype=np.int32), np.zeros(1, np.int32)
    nt = np.array([1], np.int32)
    assert lib.b200aa_forest_regression_cross_validate(dev, n, F, p(y), 1, p(tr_off), p(tr), p(te_off), p(te), p(nt), p(w),
                                                       p(seeds), dev, dev, None) == L.ERR_UNSUPPORTED


def test_dispatcher_restores_the_state_on_a_scratch_refusal(monkeypatch):
    """When the batched call refuses (a tree over the scratch bound), evaluate_regression puts NumPy's global state back
    as it was before its draws and the dispatcher hands the call to the original, which then draws the same problems."""
    from pyaudioanalysis_b200 import audioTrainTest as at
    from pyaudioanalysis_b200 import consumers
    from pyaudioanalysis_b200 import forests as FO

    def refuse(*a, **k):
        np.random.rand(5)
        raise FO.Unsupported("over the bound")
    monkeypatch.setattr(consumers, "forest_regression_cross_validate", refuse)
    seen = []

    def original(features, labels, n_exp, method_name, params):
        seen.append(np.random.get_state())
        return "original"
    r = np.random.RandomState(2)
    X, y = r.randn(30, 4), r.randn(30)
    np.random.seed(8)
    before = np.random.get_state()
    assert at.regression_dispatcher(original)(X, y, 2, "randomforest", [3, 4]) == "original"
    assert len(seen) == 1 and RC.same_state(seen[0], before)
    np.random.seed(8)
    with pytest.raises(FO.Unsupported):
        at.evaluate_regression(X, y, 2, "randomforest", [3, 4])
    assert RC.same_state(np.random.get_state(), before)

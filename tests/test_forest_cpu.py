"""CPU: kernel 13's tree builder (csrc/forest.cuh, build_tree) run on the host by tests/forest_host.cu with teams of 1, 3
and 8 threads (tests/team_host.h), fed by the host draws of pyaudioanalysis_b200.forests, against scikit-learn 1.9's
RandomForestClassifier / ExtraTreesClassifier fit on seeded problems: every tree's state in bits, the estimators' fitted
attributes and NumPy's global state afterwards.  Also: named mutants of the builder are caught (those of its
team-parallel code at a team of 3), a ThreadSanitizer build finds no race in the builder and finds a deleted barrier, the
refusals, and the argument checks of b200aa_forest_fit."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import forest_cases as FC
from tests import host_exe

pytestmark = pytest.mark.skipif(host_exe.nvcc() is None, reason="nvcc not available")

CSRC = os.path.join(host_exe.ROOT, "pyaudioanalysis_b200", "csrc")


def _build(tmp_path_factory, replace=None, flags=("-O1",)):
    """The harness over forest.cuh, or over a copy with one (old, new) replacement made (a mutant)."""
    inc = CSRC
    if replace is not None:
        src = open(os.path.join(CSRC, "forest.cuh")).read()
        old, new = replace
        assert src.count(old) == 1, old
        d = tmp_path_factory.mktemp("mutant")
        (d / "forest.cuh").write_text(src.replace(old, new))
        inc = str(d)
    return host_exe.build(tmp_path_factory, "forest_host.cu", *flags, "-I" + inc, "-I" + CSRC)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _build(tmp_path_factory)


def fit_input(tmp_path, X, y, n_estimators, kind):
    """The harness's input for the fit of X, y, drawn from NumPy's global state as fit draws: (src, dst, est, trees,
    classes)."""
    from pyaudioanalysis_b200 import forests as FO
    classes, y_idx = np.unique(y, return_inverse=True)
    n, F = X.shape
    est, trees, w, seeds = FO.draw(n_estimators, kind, n)
    head = np.array([n, F, len(classes), FO.KINDS[kind], n_estimators, max(1, int(np.sqrt(F))), w is not None],
                    dtype=np.int64)
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        for a in (head, X.astype(np.float32), y_idx.astype(np.int32)) + ((w,) if w is not None else ()) + (seeds,):
            f.write(np.ascontiguousarray(a).tobytes())
    return src, dst, est, trees, classes


def host_fit(exe, tmp_path, X, y, n_estimators, kind, team=1):
    """The estimator fit builds, every tree built by the host harness with a team of `team` threads."""
    from pyaudioanalysis_b200 import forests as FO
    n, F = X.shape
    src, dst, est, trees, classes = fit_input(tmp_path, X, y, n_estimators, kind)
    C = len(classes)
    res = subprocess.run([exe, src, dst, str(team)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    raw, off, states = open(dst, "rb").read(), 0, []
    for _ in range(n_estimators):
        nc, md = np.frombuffer(raw, np.int64, 2, off)
        off += 16
        nodes = np.frombuffer(raw, FO.NODE_DTYPE, nc, off)
        off += FO.NODE_DTYPE.itemsize * nc
        vals = np.frombuffer(raw, np.float64, nc * C, off)
        off += 8 * nc * C
        states.append(FO.tree_state(nodes, vals, md, C))
    return FO.assemble(est, trees, F, n, classes, states)


def _sklearn(kind):
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    return RandomForestClassifier if kind == "randomforest" else ExtraTreesClassifier


def _check(exe, tmp_path, X, y, kind, n_estimators=4, seed=11, team=1):
    np.random.seed(seed)
    ref = _sklearn(kind)(n_estimators=n_estimators).fit(X, y)
    ref_state = np.random.get_state()
    np.random.seed(seed)
    got = host_fit(exe, tmp_path, X, y, n_estimators, kind, team)
    assert FC.same_state(np.random.get_state(), ref_state)
    FC.compare(got, ref)
    return got, ref


@pytest.mark.parametrize("kind", ["randomforest", "extratrees"])
@pytest.mark.parametrize("case,team", host_exe.team_params(FC.problems()))
def test_trees_equal_sklearn(exe, tmp_path, kind, case, team):
    _, X, y = case
    got, ref = _check(exe, tmp_path, X, y, kind, team=team)
    assert np.array_equal(got.predict_proba(X), ref.predict_proba(X))
    assert np.array_equal(got.feature_importances_, ref.feature_importances_)


# Named mutants of the builder: each must change some tree of these problems (those in TEAM_MUTANTS at a team of 3).
MUTANTS = {
    # every node draws from a fresh 0..F-1 permutation with no known constants, instead of the carried splitter state
    "sequential_feature_state": (
        "S.n_const_out = draw_features(T.features, T.constf, T.F, T.max_features, T.kind, rec.n_const,",
        "for (int f = 0; f < T.F; ++f) T.features[f] = f;\n"
        "                S.n_const_out = draw_features(T.features, T.constf, T.F, T.max_features, T.kind, 0,"),
    # ties of the proxy keep the last position instead of the first
    "ge_instead_of_gt": ("if (pr > bp) {", "if (pr >= bp) {"),
    # a fused multiply-add in the proxy
    "fma_in_proxy": ("return dsub(dmul(-wr, gr), dmul(wl, gl));", "return std::fma(-wl, gl, dmul(-wr, gr));"),
    # the cross-thread reduction of eval_best keeps the last thread of a tied proxy instead of the first
    "reduction_keeps_last_tie": ("if (T.red_pos[t] >= 0 && T.red_proxy[t] > fp) {", "if (T.red_pos[t] >= 0 && T.red_proxy[t] >= fp) {"),
    # eval_best starts every thread's chunk at zero counts instead of the earlier chunks' sums
    "chunk_counts_from_zero": ("for (int t = 0; t < tm.tid; ++t) a += T.cnt[int64_t(t) * T.C + c];", ""),
    # partition places every chunk's right-hand samples as if no earlier chunk had any
    "partition_drops_right_offsets": ("rb += len - T.red_pos[t2];", "(void)len;"),
}
TEAM_MUTANTS = {"reduction_keeps_last_tie", "chunk_counts_from_zero", "partition_drops_right_offsets"}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_mutants_are_caught(tmp_path_factory, tmp_path, name):
    mexe = _build(tmp_path_factory, MUTANTS[name])
    team = 3 if name in TEAM_MUTANTS else 1
    kinds = ["randomforest"] if name != "sequential_feature_state" else ["randomforest", "extratrees"]
    cases = [(5, X, y) for _, X, y in FC.problems() if X.shape[0] >= 3] + [(39, *FC.palindrome(39))]
    if team > 1:
        cases = [c for c in cases if c[1].shape[0] <= 1000]
    caught = 0
    for kind in kinds:
        for seed, X, y in cases:
            np.random.seed(seed)
            ref = _sklearn(kind)(n_estimators=3).fit(X, y)
            np.random.seed(seed)
            got = host_fit(mexe, tmp_path, X, y, 3, kind, team)
            try:
                FC.compare(got, ref)
            except AssertionError:
                caught += 1
    assert caught > 0, name


# A barrier deleted from the builder (class_counts sums the per-thread counts before every thread has written its own):
# a race whose outcome depends on timing, so it is ThreadSanitizer's to find, not the comparison's
SYNC_MUTANT = ("    T.red_pos[tm.tid] = k;\n    tm.sync();\n", "    T.red_pos[tm.tid] = k;\n")


@pytest.mark.parametrize("mutant", [False, True], ids=["builder", "deleted_sync"])
def test_thread_sanitizer(tmp_path_factory, tmp_path, monkeypatch, mutant):
    """The builder built with ThreadSanitizer, at a team of 4 on small problems of both kinds: no report (and the trees
    still equal scikit-learn's); with one barrier deleted, a data race is reported on every problem.  The mutant's run
    is judged by its reports alone (host_exe.tsan_reports): after the racing read it may build a wrong tree, crash or
    not end, as timing has it."""
    tsan = _build(tmp_path_factory, SYNC_MUTANT if mutant else None, ("-O1",) + host_exe.tsan_flags())
    cases = [c for c in FC.problems() if c[0] in ("one_row", "single_class", "strings_f2", "gauss_11x300_c4")]
    if mutant:
        cases = cases[2:]                       # one_row and single_class build no split: nothing to count
    for kind in ("randomforest", "extratrees"):
        for name, X, y in cases + [("palindrome", *FC.palindrome(39))]:
            if mutant:
                np.random.seed(3)
                src, dst = fit_input(tmp_path, X, y, 2, kind)[:2]
                logs = tmp_path / ("tsan_%s_%s" % (kind, name))
                assert "WARNING: ThreadSanitizer: data race" in host_exe.tsan_reports([tsan, src, dst, "4"], logs), (kind, name)
            else:
                monkeypatch.setenv("TSAN_OPTIONS", "exitcode=0 log_path=%s" % (tmp_path / "tsan"))
                _check(tsan, tmp_path, X, y, kind, n_estimators=2, team=4)
    if not mutant:
        reports = "".join(p.read_text() for p in tmp_path.glob("tsan*"))
        assert reports == "", reports[:4000]


def test_global_state_after_many_trees(exe, tmp_path):
    r = np.random.RandomState(3)
    X, y = r.randn(120, 5), r.randint(0, 3, 120)
    for kind in ("randomforest", "extratrees"):
        _check(exe, tmp_path, X, y, kind, n_estimators=25, seed=99)
        # the next draw after fit is the reference's too
        np.random.seed(99)
        _sklearn(kind)(n_estimators=25).fit(X, y)
        a = np.random.rand(4)
        np.random.seed(99)
        host_fit(exe, tmp_path, X, y, 25, kind)
        assert np.array_equal(np.random.rand(4), a)


def test_refusals():
    from pyaudioanalysis_b200 import forests as FO
    X, y = np.random.RandomState(0).randn(10, 3), np.arange(10) % 2
    assert FO.unsupported(X, y, 10, "randomforest") is None
    assert FO.unsupported(X, y, 10, "extratrees") is None
    bad = X.copy()
    bad[1, 1] = np.nan
    assert "NaN" in FO.unsupported(bad, y, 10, "randomforest")
    bad[1, 1] = 1e300                                      # inf once cast to float32
    assert "inf" in FO.unsupported(bad, y, 10, "randomforest")
    assert "sample weights" in FO.unsupported(X, y, 10, "randomforest", sample_weight=np.ones(10))
    assert "hyper-parameters" in FO.unsupported(X, y, 10, "randomforest", class_weight="balanced")
    assert "hyper-parameters" in FO.unsupported(X, y, 10, "extratrees", max_depth=3)
    assert "shared-memory" in FO.unsupported(np.zeros((4, FO.MAX_FEATS + 1)), y[:4], 10, "randomforest")
    assert "shared-memory" in FO.unsupported(np.zeros((40, 2)), np.arange(40), 10, "randomforest")
    assert "classification" in FO.unsupported(X, y + 0.5, 10, "randomforest")
    assert "gradientboosting" in FO.unsupported(X, y, 10, "gradientboosting")
    assert "n_estimators" in FO.unsupported(X, y, 0, "randomforest")
    import sklearn
    real = sklearn.__version__
    try:
        sklearn.__version__ = "1.8.2"
        assert "1.9" in FO.unsupported(X, y, 10, "randomforest")
    finally:
        sklearn.__version__ = real


def test_abi_argument_checks():
    """b200aa_forest_fit refuses bad arguments before any CUDA call (so also on a machine without a GPU)."""
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    n, F, T = 6, 2, 2
    y = np.array([0, 1, 0, 1, 0, 1], dtype=np.int32)
    w = np.ones((T, n), dtype=np.int32)
    seeds = np.ones(T, dtype=np.uint32)
    nodes = np.zeros(T * (2 * n - 1), dtype=[("b", "u1", 48)])
    vals = np.zeros(T * (2 * n - 1) * 2)
    cnt, dep = np.zeros(T, np.int64), np.zeros(T, np.int32)
    dev = ctypes.c_void_p(16)                              # never dereferenced: every call below fails its checks first

    def p(a):
        return ctypes.c_void_p(a.ctypes.data)

    def call(**kw):
        a = dict(d_X=dev, dtype=L.DTYPE_F64, n=n, F=F, stride=F, y=p(y), C=2, kind=0, T=T, mf=1, w=p(w), seeds=p(seeds),
                 nodes=p(nodes), vals=p(vals), cap=T * (2 * n - 1), cnt=p(cnt), dep=p(dep))
        a.update(kw)
        return lib.b200aa_forest_fit(a["d_X"], a["dtype"], a["n"], a["F"], a["stride"], a["y"], a["C"], a["kind"], a["T"],
                                     a["mf"], a["w"], a["seeds"], a["nodes"], a["vals"], a["cap"], a["cnt"], a["dep"], None)
    for kw in (dict(d_X=None), dict(y=None), dict(seeds=None), dict(nodes=None), dict(vals=None), dict(cnt=None),
               dict(dep=None), dict(n=0), dict(F=0), dict(stride=1), dict(C=0), dict(T=0), dict(kind=2), dict(mf=0),
               dict(mf=3), dict(dtype=0), dict(cap=-1), dict(C=1)):     # C=1: class index 1 is out of range
        assert call(**kw) == L.ERR_INVALID, kw
    wneg = w.copy()
    wneg[1, 2] = -1
    assert call(w=p(wneg)) == L.ERR_INVALID
    assert call(F=513, stride=513, mf=1) == L.ERR_UNSUPPORTED
    ybig = np.arange(n, dtype=np.int32) % 33
    assert call(y=p(ybig), C=33) == L.ERR_UNSUPPORTED
    # an input both invalid and over the feature or class limit is invalid
    assert call(F=513, stride=513, mf=1, w=p(wneg)) == L.ERR_INVALID
    assert call(F=513, stride=513, mf=1, C=1) == L.ERR_INVALID
    assert call(y=p(ybig), C=33, w=p(wneg)) == L.ERR_INVALID


def test_cross_validate_argument_checks():
    """b200aa_forest_cross_validate refuses bad arguments before any CUDA call."""
    from pyaudioanalysis_b200 import _lib as L
    lib = L.lib()
    n = 6
    y = np.array([0, 1, 0, 1, 0, 1], dtype=np.int32)
    tr_off, te_off = np.array([0, 4], np.int64), np.array([0, 2], np.int64)
    tr, te = np.array([0, 1, 2, 3], np.int32), np.array([4, 5], np.int32)
    nt, w, seeds = np.array([2], np.int32), np.ones((2, 4), np.int32), np.ones(2, np.uint32)
    dev = ctypes.c_void_p(16)                              # never dereferenced: every call below fails its checks first

    def p(a):
        return ctypes.c_void_p(a.ctypes.data)

    def call(**kw):
        a = dict(X=dev, n=n, F=2, y=p(y), C=2, kind=0, P=1, tro=p(tr_off), tr=p(tr), teo=p(te_off), te=p(te), nt=p(nt),
                 w=p(w), seeds=p(seeds), pred=dev, counts=dev)
        a.update(kw)
        return lib.b200aa_forest_cross_validate(a["X"], a["n"], a["F"], a["y"], a["C"], a["kind"], a["P"], a["tro"],
                                                a["tr"], a["teo"], a["te"], a["nt"], a["w"], a["seeds"], a["pred"],
                                                a["counts"], None)
    bad_tr = np.array([0, 1, 2, 6], np.int32)
    bad_nt = np.array([0], np.int32)
    empty = np.array([0, 0], np.int64)
    for kw in (dict(X=None), dict(y=None), dict(seeds=None), dict(pred=None), dict(counts=None), dict(n=0), dict(F=0),
               dict(C=1), dict(P=0), dict(kind=2), dict(w=None), dict(kind=1), dict(tr=p(bad_tr)), dict(nt=p(bad_nt)),
               dict(tro=p(empty))):
        assert call(**kw) == L.ERR_INVALID, kw
    assert call(F=513) == L.ERR_UNSUPPORTED
    # a training split of more rows than X has (here 7 of 6, one repeated) is invalid
    long_off, long_tr = np.array([0, 7], np.int64), np.array([0, 1, 2, 3, 4, 5, 0], np.int32)
    assert call(tro=p(long_off), tr=p(long_tr), w=p(np.ones((2, 7), np.int32))) == L.ERR_INVALID
    # an input both invalid and over the feature limit is invalid
    assert call(F=513, tr=p(bad_tr)) == L.ERR_INVALID
    assert call(F=513, te=p(np.array([4, 6], np.int32))) == L.ERR_INVALID

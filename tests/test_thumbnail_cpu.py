"""CPU: kernel 10 (csrc/thumb.cuh) run on the host by tests/thumb_host.cu -- the similarity entries, the diagonal filter
with its NaN box rule, the min and argmax keys, the masks and the walk -- against scipy and the reference's own steps,
compared as float64 bit patterns, and against the goldens of the unmodified reference; the host path of the sizes the
kernel does not take; the C ABI's argument checks, which return before any CUDA call; install_thumbnailing."""
import ctypes
import types

import numpy as np
import pytest
import scipy.signal
from scipy.spatial import distance

from tests import host_exe
from tests.host_exe import bits, floats, hexes, run
from tests.thumb_cases import STUB_CASES, golden
from pyaudioanalysis_b200 import audioSegmentation as A
from pyaudioanalysis_b200.consumers import _limit_bounds, thumbnail_host


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "thumb_host.cu", "-O2")


def scipy_sim(X):
    with np.errstate(all="ignore"):
        return 1.0 - distance.squareform(distance.pdist(X, "cosine"))


def reference_steps(S, m, gap, limit_1=0, limit_2=1):
    """audioSegmentation.py:1145-1177 restated statement by statement on a similarity matrix."""
    C = scipy.signal.convolve2d(S, np.eye(m, m), "valid")
    min_sm = np.min(C)
    for i in range(C.shape[0]):
        for j in range(C.shape[1]):
            if abs(i - j) < gap or i > j:
                C[i, j] = min_sm
    C[0:int(limit_1 * C.shape[0]), :] = min_sm
    C[:, 0:int(limit_1 * C.shape[0])] = min_sm
    C[int(limit_2 * C.shape[0])::, :] = min_sm
    C[:, int(limit_2 * C.shape[0])::] = min_sm
    rows, cols = np.unravel_index(C.argmax(), C.shape)
    i1, i2, j1, j2 = rows, rows, cols, cols
    while i2 - i1 < m:
        if i1 <= 0 or j1 <= 0 or i2 >= C.shape[0] - 2 or j2 >= C.shape[1] - 2:
            break
        if C[i1 - 1, j1 - 1] > C[i2 + 1, j2 + 1]:
            i1 -= 1
            j1 -= 1
        else:
            i2 += 1
            j2 += 1
    return (i1, i2, j1, j2), C


def host_sim(exe, X):
    T, F = X.shape
    return floats(run(exe, "sim %d %d %s\n" % (T, F, hexes(X)))[0][1:]).reshape(T, T)


def host_thumb(exe, X, m, gap, limit_1=0, limit_2=1):
    T, F = X.shape
    R = T - m + 1
    lo, hi = _limit_bounds(R, limit_1, limit_2)
    out = run(exe, "thumb %d %d %d %s %d %d %s\n" % (T, F, m, float(gap).hex(), lo, hi, hexes(X)))
    return tuple(int(v) for v in out[0][1:]), floats(out[1][1:]).reshape(R, R)


def value_bank(rng, T, F):
    """Rows at scales from subnormal to near overflow, with +-0, zero rows, NaN and inf."""
    X = rng.normal(size=(T, F)) * np.exp(rng.uniform(-700, 700, size=(T, 1)))
    X[rng.random(size=(T, F)) < 0.05] = 0.0
    X[rng.random(size=(T, F)) < 0.05] = -0.0
    X[1] = 0.0
    X[2] = rng.normal(size=F) * 5e-324
    if T > 6:
        X[5, F // 2] = np.nan
        X[6, 0] = np.inf
    return X


@pytest.mark.parametrize("F", [1, 2, 3, 5, 67, 68, 69, 136, 137])
def test_similarity_matches_scipy(exe, F):
    """Every entry of S, bit for bit scipy's cosine pdist, on the value bank and on standardised normal rows."""
    rng = np.random.default_rng(F)
    for X in (value_bank(rng, 24, F), rng.normal(size=(30, F)), A.standardise(rng.normal(size=(F, 40)) * 7 + 3)):
        got, want = host_sim(exe, X), scipy_sim(X)
        assert np.array_equal(bits(got), bits(want)), F
        assert np.array_equal(bits(got), bits(got.T))


def test_neither_sequential_nor_fma_dot_matches():
    """The two-accumulator order is the one scipy uses: a plain sequential dot misses it somewhere on the bank."""
    rng = np.random.default_rng(7)
    X = rng.normal(size=(60, 68)) * np.exp(rng.uniform(-3, 3, size=(1, 68)))
    S = scipy_sim(X)
    seq = np.empty_like(S)
    nrm = [np.sqrt(sum(x * x for x in u)) for u in X]
    for i in range(60):
        for j in range(60):
            d = 0.0
            for a, b in zip(X[i], X[j]):
                d += a * b
            c = d / (nrm[i] * nrm[j])
            seq[i, j] = 1.0 - (1.0 - (np.copysign(1.0, c) if abs(c) > 1 else c))
    np.fill_diagonal(seq, 1.0)
    assert not np.array_equal(bits(seq), bits(S))


@pytest.mark.parametrize("T,F,m,step,limits", [(40, 68, 20, 0.5, (0, 1)), (33, 3, 4, 0.25, (0, 1)), (64, 5, 10, 0.5, (0.2, 0.9)),
                                               (50, 1, 7, 1.0, (0.6, 0.2)), (30, 68, 30, 0.5, (0, 1)), (21, 2, 1, 0.5, (0, 1)),
                                               (45, 68, 20, 0.5, (-0.4, -0.1))])
def test_filter_mask_and_walk_match_reference(exe, T, F, m, step, limits):
    """C, its masks, the argmax and the walk equal the reference's statements on standardised rows."""
    rng = np.random.default_rng(T * F + m)
    st = rng.normal(size=(F, T)) + np.sin(np.arange(T) / 3.0)
    X = A.standardise(st)
    idx, C = host_thumb(exe, X, m, 5.0 / step, *limits)
    ridx, rC = reference_steps(scipy_sim(X), m, 5.0 / step, *limits)
    assert idx == tuple(int(v) for v in ridx)
    assert np.array_equal(bits(C), bits(rC))


@pytest.mark.parametrize("where", ["nan_feature", "zero_row", "overflow"])
def test_nan_box_rule(exe, where):
    """A NaN anywhere in an entry's m x m box, not only on its diagonal, makes the entry NaN; the min is NaN, every
    masked entry becomes NaN, and the argmax is the first NaN."""
    rng = np.random.default_rng(len(where))
    X = rng.normal(size=(40, 6))
    if where == "nan_feature":
        X[17, 2] = np.nan
    elif where == "zero_row":
        X[23] = 0.0
    else:
        X[11:13] *= 1e300                               # dot overflows: inf / inf between them, 0 / inf elsewhere
    ridx, rC = reference_steps(scipy_sim(X), 8, 3.0)
    idx, C = host_thumb(exe, X, 8, 3.0)
    assert np.isnan(rC).any()
    assert idx == tuple(int(v) for v in ridx)
    assert np.array_equal(bits(C), bits(rC))


def _stub_inputs(g, name):
    F, T, step, thumb, l1, l2, _ = STUB_CASES[name]
    return A.standardise(g[name + "_st"]), int(round(thumb / step)), step, l1, l2


def test_goldens_through_host_harness(exe):
    """The stubbed-feature goldens of the unmodified reference, in bits: S where stored, and C with the four times where
    the kernel takes the size."""
    g = golden()
    ran = 0
    for name in STUB_CASES:
        X, m, step, l1, l2 = _stub_inputs(g, name)
        if name + "_S" in g.files:
            assert np.array_equal(bits(host_sim(exe, X)), bits(g[name + "_S"])), name
        if str(g[name + "_error"]) or not (1 <= m <= X.shape[0]):
            continue
        idx, C = host_thumb(exe, X, m, 5.0 / step, l1, l2)
        assert np.array_equal(bits(C), bits(g[name + "_C"])), name
        assert np.array_equal(bits(step * np.array(idx, dtype=np.int64)), bits(g[name + "_times"])), name
        ran += 1
    assert ran >= 10


def test_host_path_sizes_match_goldens():
    """The sizes left to the host (filter_len < 1, T < filter_len) give the reference's matrix and times, or its
    exception, from the reference's similarity matrix."""
    g = golden()
    for name in ("shorter_than_filter", "one_frame", "filter_zero", "filter_negative"):
        X, m, step, l1, l2 = _stub_inputs(g, name)
        assert not (1 <= m <= X.shape[0])
        err = str(g[name + "_error"])
        if err:
            with pytest.raises(ValueError):
                thumbnail_host(scipy_sim(X), m, 5.0 / step, l1, l2)
            continue
        idx, C = thumbnail_host(scipy_sim(X), m, 5.0 / step, l1, l2)
        assert np.array_equal(bits(C), bits(g[name + "_C"])), name
        times = [step * i for i in idx]
        assert all(type(t) is np.float64 for t in times)
        assert np.array_equal(bits(np.array(times)), bits(g[name + "_times"])), name


@pytest.mark.parametrize("R", [1, 2, 7, 100])
def test_limit_bounds_follow_python_slices(R):
    for l1 in (0, 0.1, 0.5, 1, 1.7, -0.3, -2):
        for l2 in (1, 0.9, 0.3, 0, -0.2, 3):
            lo, hi = _limit_bounds(R, l1, l2)
            keep = np.ones(R, dtype=bool)
            keep[0:int(l1 * R)] = False
            keep[int(l2 * R)::] = False
            assert np.array_equal(keep, (np.arange(R) >= lo) & (np.arange(R) < hi)), (R, l1, l2)


# ------------------------------------------------------------------ C ABI argument checks (no CUDA call is made)
@pytest.fixture(scope="module")
def L():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib


def test_thumbnail_rejects_bad_arguments(L):
    lib = L.lib()
    d = ctypes.c_void_p(16)
    frames = np.array([30, 25], dtype=np.int64)
    limits = np.array([[0, 11], [0, 6]], dtype=np.int64)

    def call(X=d, F=68, stride=68, frames=frames, B=2, m=20, limits=limits, sim=None, out=d, idx=d):
        fr = None if frames is None else ctypes.c_void_p(np.ascontiguousarray(frames, dtype=np.int64).ctypes.data)
        li = None if limits is None else ctypes.c_void_p(np.ascontiguousarray(limits, dtype=np.int64).ctypes.data)
        return lib.b200aa_music_thumbnail(X, F, stride, fr, B, m, 10.0, li, sim, out, idx, None)

    assert call(X=None) == L.ERR_INVALID
    assert call(frames=None) == L.ERR_INVALID
    assert call(F=0, stride=0) == L.ERR_INVALID
    assert call(stride=67) == L.ERR_INVALID
    assert call(B=0) == L.ERR_INVALID
    assert call(out=None) == L.ERR_INVALID
    assert call(idx=None) == L.ERR_INVALID
    assert call(limits=None) == L.ERR_INVALID
    assert call(m=0) == L.ERR_INVALID
    assert call(m=26) == L.ERR_INVALID                                  # T < filter_len
    assert call(frames=np.array([30, 0])) == L.ERR_INVALID
    assert call(limits=np.array([[0, 12], [0, 6]])) == L.ERR_INVALID    # hi > R
    assert call(limits=np.array([[-1, 11], [0, 6]])) == L.ERR_INVALID
    assert call(sim=d) == L.ERR_INVALID                                 # both modes at once
    assert call(sim=d, out=None) == L.ERR_INVALID
    assert call(frames=np.array([1 << 29, 1]), sim=d, out=None, idx=None) == L.ERR_INVALID


def test_install_thumbnailing_and_uninstall():
    import importlib
    install = importlib.import_module("pyaudioanalysis_b200.install")
    names = ("music_thumbnailing", "self_similarity_matrix")
    originals = {n: (lambda n: lambda *a: n)(n) for n in names + ("speaker_diarization",)}
    mod = types.ModuleType("pyAudioAnalysis.audioSegmentation")
    for n, f in originals.items():
        setattr(mod, n, f)
    try:
        done = install.install_thumbnailing(mod)
        assert sorted(done) == sorted("pyAudioAnalysis.audioSegmentation." + n for n in names)
        for n in names:
            assert getattr(mod, n) is getattr(A, n)
        assert mod.speaker_diarization is originals["speaker_diarization"]
    finally:
        install.uninstall()
    for n in originals:
        assert getattr(mod, n) is originals[n]

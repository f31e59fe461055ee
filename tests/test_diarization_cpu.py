"""CPU: the host steps of the drop-in speaker diarization -- the silhouette from the cluster distance means, the
diarize pipeline with kernel 9 replaced by its NumPy statement and the HMM left out, evaluate_speaker_diarization, the
missing-model error -- and install_diarization / uninstall."""
import types
import warnings

import numpy as np
import pytest

from tests import diarization_oracle as O
from tests.diarization_cases import fixed, lda_case
from tests.diarization_oracle import reference
from pyaudioanalysis_b200 import audioSegmentation as S


def test_silhouette_from_means_matches_restatement():
    rng = np.random.default_rng(1)
    x = rng.normal(size=(500, 12))
    for k in (2, 4, 9):
        cls = rng.integers(0, k, size=500)
        cls[cls == k - 1] = 0
        cls[:5] = k - 1                                         # a cluster below the 2 % share
        A, B = reference(x, cls, k)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            got = S._silhouette(cls, k, A, B)
        assert np.float64(got).view(np.uint64) == np.float64(O.silhouette(x, cls, k)).view(np.uint64)


@pytest.mark.parametrize("n_speakers", [3, 0])
def test_diarize_host_steps(n_speakers):
    """sil_all, the chosen count and the labels of every count through diarize's host steps with NumPy's means, the
    HMM and median filter left out (they need kernel 7)."""
    rng = np.random.default_rng(2 + n_speakers)
    mid = rng.normal(size=(30, 400)) + np.repeat(rng.normal(size=(30, 8)) * 3, 50, axis=1)
    post = [rng.dirichlet(np.ones(4), size=400), rng.dirichlet(np.ones(2), size=400)]
    cluster = (lambda x, k: (np.arange(x.shape[0]) // 50) % k)

    def means(x, cls, k, rows):
        want = np.zeros(k, dtype=bool)
        want[list(rows)] = True
        return reference(x, cls, k, want)
    seen = {}
    real_smooth = S._hmm_smooth
    S._hmm_smooth = lambda x, cls: seen.setdefault("cls", np.asarray(cls, dtype=np.int64))
    try:
        _, info = S.diarize(mid, None, n_speakers, 0.1, 0.1, 0, posteriors=post, cluster=cluster, means=means, details=True)
    finally:
        S._hmm_smooth = real_smooth
    import sklearn.preprocessing
    feats = np.concatenate([mid] + [p.T + 1e-4 for p in post])
    x = sklearn.preprocessing.StandardScaler().fit_transform(feats.T)
    from scipy.spatial import distance
    d = np.sum(distance.squareform(distance.pdist(x.T)), axis=0)
    x = x[:, np.nonzero(d < 1.1 * np.mean(d))[0]]
    s_range = range(2, 10) if n_speakers <= 0 else [n_speakers]
    sil_all = np.array([O.silhouette(x, cluster(x, k), k) for k in s_range])
    assert np.array_equal(info["sil_all"].view(np.uint64), sil_all.view(np.uint64))
    assert info["num_speakers"] == s_range[int(np.argmax(sil_all))]
    assert np.array_equal(seen["cls"], cluster(x, s_range[-1]))          # the LAST count's labels are smoothed


def test_evaluate_speaker_diarization_matches_loop():
    rng = np.random.default_rng(3)
    for _ in range(20):
        a = rng.integers(0, 4, size=int(rng.integers(1, 60))).astype(np.float64)
        b = rng.integers(0, 3, size=int(rng.integers(1, 60)))
        n = min(len(a), len(b))
        fa, fb = np.unique(a[:n]), np.unique(b[:n])
        t = np.zeros((len(fa), len(fb)))
        for i in range(n):
            t[int(np.nonzero(fa == a[i])[0][0]), int(np.nonzero(fb == b[i])[0][0])] += 1.0
        rs, cs = t.sum(axis=0), t.sum(axis=1)
        pc = np.sum(np.array([t[i].max() / cs[i] for i in range(len(fa))]) * cs) / t.sum()
        ps = np.sum(np.array([t[:, j].max() / rs[j] for j in range(len(fb))]) * rs) / t.sum()
        assert S.evaluate_speaker_diarization(a, b) == (pc, ps)


def test_missing_models_raise(tmp_path):
    with pytest.raises(FileNotFoundError, match="svm_rbf_speaker_male_female"):
        S.speaker_diarization(str(tmp_path / "x.wav"), 2, models_dir=str(tmp_path))


def test_install_diarization_and_uninstall():
    import importlib
    install = importlib.import_module("pyaudioanalysis_b200.install")
    names = ("speaker_diarization", "speaker_diarization_evaluation", "evaluate_speaker_diarization")
    originals = {n: (lambda n: lambda *a: n)(n) for n in names + ("hmm_segmentation",)}
    mod = types.ModuleType("pyAudioAnalysis.audioSegmentation")
    for n, f in originals.items():
        setattr(mod, n, f)
    try:
        done = install.install_diarization(mod)
        assert sorted(done) == sorted("pyAudioAnalysis.audioSegmentation." + n for n in names)
        for n in names:
            assert getattr(mod, n) is getattr(S, n)
        assert mod.hmm_segmentation is originals["hmm_segmentation"]
    finally:
        install.uninstall()
    for n in originals:
        assert getattr(mod, n) is originals[n]


# ------------------------------------------------------------------ the LDA branch (:881-932)
def test_pool_frames_matches_reference_loop():
    """The per-frame pooling equals the reference's per-row loop of np.mean / np.std over each cut window, in bits."""
    rng = np.random.default_rng(20)
    st = rng.normal(size=(68, 300)) * np.exp(rng.uniform(-20, 20, size=(68, 1)))
    st = st.astype(np.float32).astype(np.float64)
    for ratio in (1, 3, 8, 10, 40, 130, 400):
        got, want = S.pool_frames(st, ratio), O.pool_frames(st, ratio)
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), ratio


@pytest.mark.parametrize("n_speakers,lda_dim", [(3, 2), (0, 3)])
def test_diarize_lda_host_steps(n_speakers, lda_dim):
    """diarize with lda_dim > 0 (no HMM, so every step runs on the host once kernel 9 is replaced by its NumPy statement)
    against the restatement of the reference's LDA branch: sil_all, the chosen count and cls, in bits."""
    rng = np.random.default_rng(21 + n_speakers)
    models, st, mid, post = lda_case(rng)

    def means(x, cls, k, rows):
        want = np.zeros(k, dtype=bool)
        want[list(rows)] = True
        return reference(np.asarray(x), cls, k, want)
    cls, info = S.diarize(mid, models, n_speakers, 0.1, 0.1, lda_dim, st=st, mid_window=1.0, posteriors=post,
                          cluster=fixed, means=means, details=True)
    want_cls, sil_all, num, _ = O.diarize(mid, post, n_speakers, fixed, lda=(st, models, 1.0, 0.1, lda_dim))
    assert cls.shape == (st.shape[1],)
    assert np.array_equal(info["sil_all"].view(np.uint64), sil_all.view(np.uint64))
    assert info["num_speakers"] == num
    assert np.array_equal(cls, want_cls)


def test_diarize_lda_needs_models():
    rng = np.random.default_rng(22)
    _, st, mid, post = lda_case(rng)
    with pytest.raises(ValueError, match="lda_dim > 0 needs models"):
        S.diarize(mid, None, 3, 0.1, 0.1, 2, st=st, mid_window=1.0, posteriors=post, cluster=fixed)

"""GPU: kernel 7's float64 decode against tests/hmm_oracle.py's predict in both window layouts; ``diarize`` against the
host-only restatement (tests/diarization_oracle.py) with fixed labels and with the default k-means under one NumPy seed;
and speaker_diarization end to end on a generated WAV with seeded SVM models, against diarize on the drop-in's own
mid-term features."""
import pickle
import types

import numpy as np
import pytest

from tests import diarization_oracle as O
from tests import hmm_oracle as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def S():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import audioSegmentation
    return audioSegmentation


def _hmm(rng, C, F):
    start, trans = rng.random(C) + 0.05, rng.random((C, C)) + 0.05
    return types.SimpleNamespace(startprob_=start / start.sum(), transmat_=trans / trans.sum(axis=1, keepdims=True),
                                 means_=rng.normal(size=(C, F)), covars_=rng.random((C, F)) + 0.3)


@pytest.mark.parametrize("C,F,M", [(2, 146, 1), (3, 146, 2000), (9, 20, 36000), (4, 1, 500)])
def test_decode_f64_matches_oracle(S, C, F, M):
    import torch
    from pyaudioanalysis_b200.consumers import hmm_decode_batch
    rng = np.random.default_rng(C * F + M)
    hmm = _hmm(rng, C, F)
    X = rng.normal(size=(M, F)) + hmm.means_[rng.integers(0, C, size=M)]
    t = torch.from_numpy(X).cuda()
    # window-major: predict(X) of a C-contiguous X (pairwise density sums)
    ids, bad = hmm_decode_batch(t.unsqueeze(0).transpose(1, 2), hmm)
    path, ties = H.predict(X.T, hmm.startprob_, hmm.transmat_, hmm.means_, hmm.covars_, ties=True)
    assert ties == 0 and not bool(bad[0])
    assert np.array_equal(ids[0].cpu().numpy(), path)
    # feature-major: predict(features.T) of a C-contiguous [F, M] matrix (sequential sums)
    feats = np.ascontiguousarray(X.T)
    ids, _ = hmm_decode_batch(torch.from_numpy(feats).cuda().unsqueeze(0), hmm)
    path, ties = H.predict(feats, hmm.startprob_, hmm.transmat_, hmm.means_, hmm.covars_, ties=True)
    assert ties == 0
    assert np.array_equal(ids[0].cpu().numpy(), path)


def _mid(rng, M, speakers=3, F=136):
    """A mid-term-like matrix [F, M]: runs of windows from a few 'speakers', each a mean vector plus noise."""
    centres = rng.normal(size=(speakers, F)) * np.exp(rng.uniform(-2, 2, size=(1, F)))
    who = np.repeat(rng.integers(0, speakers, size=M // 50 + 1), 50)[:M]
    return (centres[who] + 0.3 * rng.normal(size=(M, F)) * np.exp(rng.uniform(-2, 2, size=(1, F)))).T, who


def _posteriors(rng, who, C):
    p = rng.random((who.shape[0], C)) + np.eye(C)[who % C] * 3.0
    return p / p.sum(axis=1, keepdims=True)


@pytest.mark.parametrize("n_speakers", [4, 0])
def test_diarize_fixed_labels(S, n_speakers):
    """Fixed labels per count (seeded, with a cluster below the 2 % share): every step but k-means compared."""
    rng = np.random.default_rng(10 + n_speakers)
    mid, who = _mid(rng, 1200)
    post = [_posteriors(rng, who, 10), _posteriors(rng, who, 2)]
    fixed = {}

    def cluster(x, k):
        if k not in fixed:
            lab = (np.arange(who.shape[0]) // 40 + who) % k           # every label in [0, k) present
            if k > 3:
                lab[lab == k - 1] = 0
                lab[:10] = k - 1                                    # a cluster below the 2 % share
            fixed[k] = lab
        return fixed[k]

    cls, info = S.diarize(mid, None, n_speakers, 0.1, 0.1, 0, posteriors=post, cluster=cluster, details=True)
    want_cls, sil_all, num, _ = O.diarize(mid, post, n_speakers, cluster)
    assert np.array_equal(info["sil_all"].view(np.uint64), sil_all.view(np.uint64))
    assert info["num_speakers"] == num
    assert np.array_equal(cls, want_cls)


def test_diarize_default_kmeans(S):
    """The default k-means under one NumPy seed, against the restatement under the same seed on the same machine."""
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(12)
    mid, who = _mid(rng, 900)
    post = [_posteriors(rng, who, 10), _posteriors(rng, who, 2)]
    np.random.seed(7)
    cls, info = S.diarize(mid, None, 0, 0.1, 0.1, 0, posteriors=post, details=True)
    np.random.seed(7)
    want_cls, sil_all, num, _ = O.diarize(mid, post, 0, lambda x, k: KMeans(n_clusters=k).fit(x).labels_)
    assert np.array_equal(info["sil_all"].view(np.uint64), sil_all.view(np.uint64))
    assert info["num_speakers"] == num
    assert np.array_equal(cls, want_cls)


def _write_models(tmp_path, rng):
    """Two seeded SVC(probability=True) models on 136 features with the reference's model-file layout."""
    from sklearn.svm import SVC
    for name, C in (("svm_rbf_speaker_10", 4), ("svm_rbf_speaker_male_female", 2)):
        X = rng.normal(size=(120, 136))
        y = np.arange(120) % C
        X += y[:, None] * 0.5
        mean, std = X.mean(axis=0), X.std(axis=0)
        clf = SVC(C=1.0, kernel="rbf", probability=True, random_state=0).fit((X - mean) / std, y)
        with open(tmp_path / name, "wb") as f:
            pickle.dump(clf, f)
        with open(tmp_path / (name + "MEANS"), "wb") as f:
            for obj in (mean.tolist(), std.tolist(), ["c%d" % i for i in range(C)], 1.0, 0.1, 0.05, 0.05, False):
                pickle.dump(obj, f)


def test_speaker_diarization_end_to_end(S, tmp_path):
    from tests import wavgen
    from pyaudioanalysis_b200.MidTermFeatures import mid_feature_extraction
    rng = np.random.default_rng(13)
    fs = 16000
    parts = []
    for f0 in (140.0, 220.0, 140.0, 300.0, 220.0):               # speaker-like harmonic tones, 2 s each
        t = np.arange(2 * fs) / fs
        x = sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 6)) * (1 + 0.3 * np.sin(2 * np.pi * 3 * t))
        parts.append(x + 0.05 * rng.normal(size=t.shape))
    sig = np.round(np.concatenate(parts) / 4 * 32767).astype(np.int16)
    wav = tmp_path / "talk.wav"
    wav.write_bytes(wavgen.wav_bytes(fs, wavgen.encode(sig, "s16"), 1, 1, 16))
    (tmp_path / "talk.segments").write_text("0.0\t2.0\ta\n2.0\t4.0\tb\n4.0\t6.0\ta\n6.0\t8.0\tc\n8.0\t10.0\tb\n")
    _write_models(tmp_path, rng)
    np.random.seed(3)
    cls, purity_c, purity_s = S.speaker_diarization(str(wav), 3, models_dir=str(tmp_path))
    mid, _, _ = mid_feature_extraction(sig, fs, 1.0 * fs, 0.1 * fs, round(fs * 0.05), round(fs * 0.05))
    models = [S._load_svm(str(tmp_path / n))[:3] for n in S._DIARIZATION_MODELS]
    np.random.seed(3)
    want = S.diarize(mid, models, 3, 0.1, 0.1, 0)
    assert np.array_equal(cls, want)
    assert 0 < purity_c <= 1 and 0 < purity_s <= 1
    with pytest.raises(FileNotFoundError, match="svm_rbf_speaker_10"):
        S.speaker_diarization(str(wav), 3, models_dir=str(tmp_path / "missing"))


@pytest.mark.parametrize("n_speakers,lda_dim", [(3, 2), (0, 3)])
def test_diarize_lda_on_kernel9(S, n_speakers, lda_dim):
    """The LDA branch with the silhouette means on kernel 9, against the restatement of the reference's branch."""
    from tests.diarization_cases import fixed, lda_case
    rng = np.random.default_rng(21 + n_speakers)
    models, st, mid, post = lda_case(rng)
    cls, info = S.diarize(mid, models, n_speakers, 0.1, 0.1, lda_dim, st=st, mid_window=1.0, posteriors=post,
                          cluster=fixed, details=True)
    want_cls, sil_all, num, _ = O.diarize(mid, post, n_speakers, fixed, lda=(st, models, 1.0, 0.1, lda_dim))
    assert np.array_equal(info["sil_all"].view(np.uint64), sil_all.view(np.uint64))
    assert info["num_speakers"] == num
    assert np.array_equal(cls, want_cls)


def test_empty_means_warn_as_numpy(S):
    """Every mean of no terms warns as np.mean of an empty array does, in the reference's order: one feature column
    (pdist empty) and an empty cluster (cdist empty)."""
    import warnings
    from scipy.spatial import distance
    rng = np.random.default_rng(30)
    x = rng.normal(size=(200, 1))
    cls = rng.integers(0, 4, size=200)
    cls[cls == 2] = 3
    rows = [0, 1, 3]

    def record(fn):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            with np.errstate(all="warn"):
                fn()
        return [(type(m.message), str(m.message)) for m in w]

    def reference():
        for c in rows:
            xc = x[cls == c, :]
            np.mean(distance.pdist(xc.T))
            for c2 in range(4):
                if c2 != c:
                    np.mean(distance.cdist(xc, x[cls == c2, :]))
    want = record(reference)
    assert len(want) == 2 * (3 + 3)
    assert record(lambda: S.cluster_means_gpu(x, cls, 4, rows)) == want


def test_speaker_diarization_evaluation_mono_and_stereo(S, tmp_path):
    """A folder of one mono and one stereo WAV with .segments files: the evaluation prints what speaker_diarization
    prints file by file (the stereo file downmixed, as the reference does), for LDA dimensions 0 and 1."""
    import contextlib
    import io
    from tests import wavgen
    rng = np.random.default_rng(31)
    fs = 16000

    def tones(freqs, seconds):
        out = []
        for f0 in freqs:
            t = np.arange(seconds * fs) / fs
            out.append(sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 6)) * (1 + 0.3 * np.sin(2 * np.pi * 3 * t))
                       + 0.1 * rng.normal(size=t.shape))
        return np.concatenate(out) / 5
    a = np.round(tones((150.0, 260.0, 150.0), 8) * 32767).astype(np.int16)
    b = np.stack([tones((180.0, 320.0, 240.0), 8), tones((180.0, 330.0, 250.0), 8)], axis=1)
    b = np.round(b * 32767).astype(np.int16)
    (tmp_path / "a.wav").write_bytes(wavgen.wav_bytes(fs, wavgen.encode(a, "s16"), 1, 1, 16))
    (tmp_path / "b.wav").write_bytes(wavgen.wav_bytes(fs, wavgen.encode(b, "s16"), 2, 1, 16))
    (tmp_path / "a.segments").write_text("0.0\t8.0\tx\n8.0\t16.0\ty\n16.0\t24.0\tx\n")
    (tmp_path / "b.segments").write_text("0.0\t8.0\tx\n8.0\t16.0\ty\n16.0\t24.0\tz\n")
    models = tmp_path / "models"
    models.mkdir()
    _write_models(models, rng)
    out = io.StringIO()
    np.random.seed(5)
    with contextlib.redirect_stdout(out):
        S.speaker_diarization_evaluation(str(tmp_path), [0, 1], models_dir=str(models))
    want = io.StringIO()
    np.random.seed(5)
    with contextlib.redirect_stdout(want):
        for dim in (0, 1):
            print("LDA = {0:d}".format(dim))
            for name, n in (("a.wav", 2), ("b.wav", 3)):
                S.speaker_diarization(str(tmp_path / name), n, 2.0, 0.2, 0.05, dim, models_dir=str(models))
    assert out.getvalue() == want.getvalue()
    assert out.getvalue().count("\t") == 4

"""Golden kNN classifications of the UNMODIFIED reference (run where the reference tree exists):

    python -m oracle.make_golden_knn

The reference's `Knn` class (audioTrainTest.py:33-49) is executed from its source text, as in make_golden_consumers.py
(audioTrainTest cannot be imported here), on models unpickled from the reference's data/models in load_model_knn's order
(:492-520).  Writes tests/golden/knn.npz; for case <c> (listed in `cases`):

* <c>_features [N, F], <c>_labels [N] float64, <c>_k: the model, a row subset of each shipped model (the rows of
  knn_musical_genre_6 alone take 580 KB compressed; the file stays small, and the kernel's sizes are covered by the GPU
  tests' seeded models);
* <c>_mean / <c>_std [F]: the shipped model's normalisation (real models only);
* <c>_queries [n, F]: mid-term windows of the reference's small test WAVs by its own mid_feature_extraction (for the
  138-dim model followed by the file's beat_extraction pair, as file_classification appends it), normalised in float64
  with the model's mean / std; then training rows as they are and with small noise;
* <c>_ids [n], <c>_P [n, C]: Knn.classify of each query; <c>_dk / <c>_dk1 [n]: its k-th and (k+1)-th distance (inf when
  there is no such place).

A query whose k-th place is an exact distance tie between different labels is not stored: the reference's argsort is
not stable, so its result there depends on the CPU's sort.
"""
import os
import pickle
import warnings

import numpy as np
from scipy.io import wavfile
from scipy.spatial import distance

from oracle.ref_import import REFERENCE_ROOT, load_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "knn.npz")
REF = os.path.join(REFERENCE_ROOT, "pyAudioAnalysis")
WAVS = ("count.wav", "doremi.wav", "speech_music_sample.wav")


def _exec_between(path, start, stop, env):
    src = open(path).read()
    a = src.index(start)
    b = src.index(stop, a)
    exec(src[a:b], env)
    return env


def _load_model(name):
    """load_model_knn's fields: features, labels, mean, std, classes, neighbors, mid / short windows, compute_beat."""
    with open(os.path.join(REF, "data", "models", name), "rb") as fo:
        vals = [pickle.load(fo) for _ in range(11)]
    feats, labels, mean, std = (np.array(v) for v in vals[:4])
    return feats, labels, mean, std, int(vals[5]), vals[6:10], bool(vals[10])


def _windows(M, mean, std, mid_window, mid_step, short_window, short_step, beat, per_wav):
    out = []
    for w in WAVS:
        fs, x = wavfile.read(os.path.join(REF, "data", w))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mid, st, _ = M.mid_feature_extraction(x, fs, mid_window * fs, mid_step * fs, round(fs * short_window),
                                                  round(fs * short_step))
            v = np.asarray(mid, dtype=np.float64).T[:per_wav]
            if beat:
                b, c = M.beat_extraction(st, short_step)
                v = np.concatenate([v, np.tile([b, c], (v.shape[0], 1))], axis=1)
        out.append((v - mean) / std)
    return np.concatenate(out)


def _ambiguous(d, labels, k):
    """The k-th place is an exact tie between different labels: the reference's unstable argsort decides."""
    if k >= d.size:
        return False
    dk = np.sort(d)[k - 1]
    tied = labels[d == dk]
    return (d < dk).sum() + tied.size > k and np.unique(tied).size > 1


def main():
    _, M, _ = load_reference()
    np.Inf, np.NaN = np.inf, np.nan             # utilities.peakdet (beat_extraction) still spells them the NumPy 1 way
    knn_env = _exec_between(os.path.join(REF, "audioTrainTest.py"), "class Knn", "def classifier_wrapper",
                            {"np": np, "distance": distance})
    Knn = knn_env["Knn"]
    rng = np.random.default_rng(20261016)
    g, cases = {}, []

    def add(name, feats, labels, k, queries, mean=None, std=None):
        knn = Knn(feats, labels, k)
        keep, ids, P, dk, dk1 = [], [], [], [], []
        for q in queries:
            d = distance.cdist(feats, q.reshape(1, -1), "euclidean")[:, 0]
            if _ambiguous(d, labels, k):
                continue
            i, p = knn.classify(q)
            s = np.sort(d)
            keep.append(q)
            ids.append(i)
            P.append(p)
            dk.append(s[k - 1] if k <= s.size else np.inf)
            dk1.append(s[k] if k < s.size else np.inf)
        print(name, feats.shape, "k", k, "queries", len(keep), "of", len(queries))
        g.update({name + "_features": feats, name + "_labels": labels, name + "_k": np.int64(k),
                  name + "_queries": np.asarray(keep), name + "_ids": np.asarray(ids, dtype=np.int64),
                  name + "_P": np.asarray(P), name + "_dk": np.asarray(dk), name + "_dk1": np.asarray(dk1)})
        if mean is not None:
            g.update({name + "_mean": mean, name + "_std": std})
        cases.append(name)

    def train_queries(feats, n):
        rows = feats[rng.choice(feats.shape[0], size=n, replace=False)]
        return np.concatenate([rows[: n // 2], rows[n // 2:] + rng.normal(scale=0.01, size=rows[n // 2:].shape)])

    for name, rows in (("knn_musical_genre_6", 110), ("knn_4class", 80), ("knn_speaker_male_female", 40)):
        feats, labels, mean, std, k, (mw, ms, sw, ss), beat = _load_model(name)
        sub = np.sort(rng.choice(feats.shape[0], size=rows, replace=False))
        feats, labels = feats[sub], labels[sub]
        q = np.concatenate([_windows(M, mean, std, mw, ms, sw, ss, beat, 6), train_queries(feats, 16)])
        add(name, feats, labels, k, q, mean, std)

    # labels {0, 2, 3}: C = 3, so label 3 never counts and class 1 never wins
    feats = rng.normal(size=(200, 10))
    labels = rng.choice([0.0, 2.0, 3.0], size=200)
    feats += labels[:, None] * 0.3
    add("skip_class", feats, labels, 7, np.concatenate([rng.normal(size=(40, 10)) + 0.5, train_queries(feats, 20)]))

    # duplicated training rows under different labels
    base = rng.normal(size=(40, 8))
    feats = np.concatenate([base, base, base[:20]])
    labels = np.concatenate([np.zeros(40), np.ones(40), np.full(20, 2.0)])
    add("duplicates", feats, labels, 5, np.concatenate([rng.normal(size=(40, 8)), train_queries(feats, 20)]))

    g["cases"] = np.asarray(cases)
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()

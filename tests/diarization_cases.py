"""Seeded inputs of the diarization tests that run the library's host steps (speaker_diarization's LDA branch): two SVM
models with their scaling, the short- and mid-term matrices with the models' posteriors, and a fixed clustering."""
import numpy as np


def svm_models(rng, F=136):
    from sklearn.svm import SVC
    models = []
    for C in (4, 2):
        X = rng.normal(size=(60 * C, F)) + (np.arange(60 * C) % C)[:, None] * 0.4
        y = np.arange(60 * C) % C
        mean, std = X.mean(axis=0), X.std(axis=0)
        models.append((SVC(probability=True, random_state=0).fit((X - mean) / std, y), mean, std))
    return models


def lda_case(rng, T=450):
    from pyaudioanalysis_b200 import audioSegmentation as S
    models = svm_models(rng)
    st = (rng.normal(size=(68, T)) + np.repeat(rng.normal(size=(68, T // 50 + 1)), 50, axis=1)[:, :T]).astype(np.float32)
    mid = rng.normal(size=(136, T // 10))
    post = [S._posteriors(mid.T, m) for m in models]
    return models, st.astype(np.float64), mid, post


def fixed(x, k):
    lab = (np.arange(x.shape[0]) // 20) % k
    if k > 3:
        lab[lab == k - 1] = 0
        lab[:5] = k - 1                                          # a cluster below the 2 % share
    return lab

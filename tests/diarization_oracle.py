"""Host-only NumPy / scipy / scikit-learn restatement of speaker_diarization's steps after the mid-term features
(reference audioSegmentation.py:848-1012): posteriors, StandardScaler, the feature-outlier rule, k-means per candidate
count, the silhouette from np.mean of pdist / cdist, then for lda_dim = 0 the HMM smoothing of the last count's labels
(tests/hmm_oracle.py's predict, the statistics in NumPy), for lda_dim > 0 the per-frame pooling of the short-term
features written as the reference's loop, posteriors, StandardScaler and LinearDiscriminantAnalysis before the
clustering; and the median filter."""
import warnings

import numpy as np
from scipy.signal import medfilt
from scipy.spatial import distance
from sklearn.preprocessing import StandardScaler

from tests import hmm_oracle as H


def reference(X, labels, K, want=None):
    """(A [K], B [K, K]) as speaker_diarization computes them (audioSegmentation.py:958-972), NaN where not computed."""
    A, B = np.full(K, np.nan), np.full((K, K), np.nan)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for c in range(K):
            if want is not None and not want[c]:
                continue
            xc = X[labels == c, :]
            A[c] = np.mean(distance.pdist(xc.T))
            for c2 in range(K):
                if c2 != c:
                    B[c, c2] = np.mean(distance.cdist(xc, X[labels == c2, :]))
    return A, B


def statistics(features, labels):
    """train_hmm_compute_statistics (:287-344) in NumPy: priors, transitions, means, std of features [F, n]."""
    u_label = np.unique(labels)
    C = len(u_label)
    priors = np.array([np.count_nonzero(labels == u) for u in u_label], dtype=np.float64)
    priors = priors / priors.sum()
    trans = np.zeros((C, C))
    for i in range(labels.shape[0] - 1):
        trans[int(labels[i]), int(labels[i + 1])] += 1
    for i in range(C):
        trans[i, :] /= trans[i, :].sum()
    means = np.array([features[:, np.nonzero(labels == u)[0]].mean(axis=1) for u in u_label])
    cov = np.array([np.std(features[:, np.nonzero(labels == u)[0]], axis=1) for u in u_label])
    return priors, trans, means, cov


def silhouette(x, cls, k):
    sil_1, sil_2 = [], []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for c in range(k):
            share = np.nonzero(cls == c)[0].shape[0] / float(len(cls))
            if share < 0.020:
                sil_1.append(0.0)
                sil_2.append(0.0)
                continue
            xc = x[cls == c, :]
            sil_1.append(np.mean(distance.pdist(xc.T)) * share)
            temp = []
            for c2 in range(k):
                if c2 != c:
                    share_2 = np.nonzero(cls == c2)[0].shape[0] / float(len(cls))
                    temp.append(np.mean(distance.cdist(xc, x[cls == c2, :])) * (share + share_2) / 2.0)
            sil_2.append(min(np.array(temp)))
    sil_1, sil_2 = np.array(sil_1), np.array(sil_2)
    return np.mean([(sil_2[c] - sil_1[c]) / (max(sil_2[c], sil_1[c]) + 1e-5) for c in range(k)])


def pool_frames(st_feats, window_ratio):
    """:884-906 as the reference writes it: per feature row, the mean then the std of every window of window_ratio frames
    starting at each frame, cut at the end."""
    num_of_features = len(st_feats)
    red = [[] for _ in range(2 * num_of_features)]
    for index in range(num_of_features):
        cur_pos, feat_len = 0, len(st_feats[index])
        while cur_pos < feat_len:
            n2 = min(cur_pos + window_ratio, feat_len)
            short_features = st_feats[index][cur_pos:n2]
            red[index].append(np.mean(short_features))
            red[index + num_of_features].append(np.std(short_features))
            cur_pos += 1
    return np.array(red)


def lda_features(st, models, mid_window, short_window, lda_dim):
    """:881-932: the pooled frames with their posteriors (+1e-4), standardised, projected by LDA onto lda_dim axes."""
    import sklearn.discriminant_analysis
    red = pool_frames(np.asarray(st, dtype=np.float64), int(round(mid_window / short_window)))
    red2 = np.zeros((red.shape[0] + sum(m[0].predict_proba(np.zeros((1, red.shape[0]))).shape[1] for m in models),
                     red.shape[1]))
    limit = red.shape[0]
    for index in range(red.shape[1]):
        red2[0:red.shape[0], index] = red[:, index]
        at = limit
        for classifier, mean, std in models:
            p = classifier.predict_proba(((red[:, index] - mean) / std).reshape(1, -1))[0]
            red2[at:at + p.shape[0], index] = p + 1e-4
            at += p.shape[0]
    red = StandardScaler().fit_transform(red2.T).T
    labels = np.zeros((red.shape[1],))
    lda_step_ratio = 1.0 / short_window
    for index in range(labels.shape[0]):
        labels[index] = int(index * short_window / lda_step_ratio)
    clf = sklearn.discriminant_analysis.LinearDiscriminantAnalysis(n_components=lda_dim)
    return clf.fit_transform(red.T, labels)


def diarize(mid, posteriors, n_speakers, cluster, lda=None):
    """(cls, sil_all, num_speakers, labels per count) for mid [F, M] and the two posterior matrices [M, C];
    lda = (st, models, mid_window, short_window, lda_dim) for the LDA branch."""
    feats = np.concatenate([mid] + [np.asarray(p).T + 1e-4 for p in posteriors])
    x = StandardScaler().fit_transform(feats.T)
    dist_all = np.sum(distance.squareform(distance.pdist(x.T)), axis=0)
    keep = np.nonzero(dist_all < 1.1 * np.mean(dist_all))[0]
    x_or, x = x, x[:, keep]
    if lda is not None:
        x = lda_features(*lda)
    s_range = range(2, 10) if n_speakers <= 0 else [n_speakers]
    sil_all, labels = [], []
    for k in s_range:
        cls = cluster(x, k)
        labels.append(cls)
        sil_all.append(silhouette(x, cls, k))
    num_speakers = s_range[int(np.argmax(sil_all))]
    if lda is None:
        start, trans, means, cov = statistics(x_or.T, cls)
        cls = H.predict(x_or.T, start, trans, means, cov)
    return medfilt(cls, 5), np.array(sil_all), num_speakers, labels

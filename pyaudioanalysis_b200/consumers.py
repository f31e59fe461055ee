"""Consumers of the mid-term matrix (SURVEY.md 8f rank 4): the per-window normalise-and-classify loops of the reference,
batched.

The reference walks the mid-term (or short-term) matrix one column at a time:

    feature_vector = (mt_feats[:, col_index] - mean) / std              # audioSegmentation.py:581-584
    label, posterior = classifier_wrapper(classifier, model_type, feature_vector)   # audioTrainTest.py:52-93

Here all columns are normalised and transposed in ONE kernel (``b200aa_normalize_windows``: [F x M] -> [M x F] feature
vectors) and the classifier sees the whole matrix at once (scikit-learn's ``predict`` / ``predict_proba`` are row-wise, the
library's kNN runs as one kernel over a CUDA matrix of test vectors, ``b200aa_knn_classify``, and is restated below for a
NumPy one), so the results are the loop's results.  The classifiers themselves (training, model files, HMMs) stay out of
scope; any object with the reference's interface works.
"""
import ctypes

import numpy as np
import torch

from ._lib import DTYPE_F32, DTYPE_F64, check, lib
from .batch import _require_cuda, _stream, beat_extraction_batch, long_term_mean_batch, mid_feature_extraction_batch

_SKLEARN_TYPES = ("svm", "randomforest", "gradientboosting", "extratrees", "svm_rbf")


def normalize_windows_batch(mid, mean, std):
    """CUDA float32 [B, F, M] -> [B, M, F]: vector j of clip b = (mid[b, :, j] - mean) / std."""
    _require_cuda(mid, "mid")
    if mid.dim() != 3 or mid.dtype != torch.float32 or not mid.is_contiguous():
        raise ValueError("mid must be contiguous float32 [B, F, M]")
    B, F, M = mid.shape
    mean = torch.as_tensor(np.asarray(mean, dtype=np.float32)).to(mid.device)
    std = torch.as_tensor(np.asarray(std, dtype=np.float32)).to(mid.device)
    if mean.numel() != F or std.numel() != F:
        raise ValueError("mean / std must hold one value per feature row (%d)" % F)
    with torch.cuda.device(mid.device):
        out = torch.empty((B, M, F), dtype=torch.float32, device=mid.device)
        check(lib().b200aa_normalize_windows(ctypes.c_void_p(mid.data_ptr()), B, F, M, ctypes.c_void_p(mean.data_ptr()),
                                             ctypes.c_void_p(std.data_ptr()), ctypes.c_void_p(out.data_ptr()), _stream()))
    return out


def knn_classify_matrix(classifier, vectors):
    """The library's kNN (audioTrainTest.py:33-49) for a matrix of test vectors [n x F]: (class ids [n], P [n x classes]).
    `classifier` needs .features [N x F], .labels [N], .neighbors (the reference's Knn object or a look-alike)."""
    feats = np.asarray(classifier.features, dtype=np.float64)
    labels = np.asarray(classifier.labels)
    k = int(classifier.neighbors)
    n_classes = np.unique(labels).shape[0]
    v = np.asarray(vectors, dtype=np.float64)
    d = np.sqrt(np.maximum(((v[:, None, :] - feats[None, :, :]) ** 2).sum(axis=2), 0.0))     # cdist(..., 'euclidean')
    order = np.argsort(d, axis=1)[:, :k]
    near = labels[order]
    P = np.stack([(near == i).sum(axis=1) / float(k) for i in range(n_classes)], axis=1)
    return np.argmax(P, axis=1), P


class KnnModel:
    """A kNN model (the reference's ``Knn`` object, audioTrainTest.py:33-49, or anything with .features [N x F], .labels [N]
    and .neighbors) uploaded once to one CUDA device for ``knn_classify_batch``: the float64 features, and per training row
    the class it votes for -- its label when that is an integer in [0, C), else -1, since Knn.classify counts
    ``labels == i`` for i in range(C), C = len(np.unique(labels))."""

    def __init__(self, classifier, device=None):
        feats = np.asarray(classifier.features, dtype=np.float64)
        labels = np.asarray(classifier.labels)
        if feats.ndim != 2 or feats.shape[0] < 1 or feats.shape[1] < 1:
            raise ValueError("kNN features must be a non-empty [N x F] matrix, got shape %s" % (feats.shape,))
        if labels.shape != (feats.shape[0],):
            raise ValueError("kNN labels must hold one label per training row (%d), got shape %s" % (feats.shape[0], labels.shape))
        self.k = int(classifier.neighbors)
        if self.k < 1:
            raise ValueError("kNN neighbors must be >= 1, got %d" % self.k)
        self.n_train, self.n_feats = feats.shape
        self.n_classes = int(np.unique(labels).shape[0])
        slots = np.full(self.n_train, -1, dtype=np.int32)
        if labels.dtype.kind in "biuf":
            lf = labels.astype(np.float64)
            ok = (lf == np.floor(lf)) & (lf >= 0) & (lf < self.n_classes)
            slots[ok] = lf[ok].astype(np.int32)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise TypeError("a KnnModel lives on a CUDA device (there is no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.features = torch.from_numpy(np.ascontiguousarray(feats)).to(self.device)
        self.slots = torch.from_numpy(slots).to(self.device)


def knn_classify_batch(model, vectors):
    """Knn.classify (audioTrainTest.py:33-49) of every row of a CUDA float32 / float64 [n, F] tensor, in one kernel on the
    current stream: CUDA (ids int64 [n], P float64 [n, C]), bit for bit the reference's per-row results (DESIGN.md, kernel 5).
    `model`: a KnnModel, or a Knn-like object, uploaded for this call."""
    _require_cuda(vectors, "vectors")
    if not isinstance(model, KnnModel):
        model = KnnModel(model, vectors.device)
    if vectors.dim() != 2 or vectors.dtype not in (torch.float32, torch.float64):
        raise ValueError("vectors must be float32 / float64 [n, F]")
    if vectors.shape[1] != model.n_feats:
        raise ValueError("vectors have %d features, the model %d" % (vectors.shape[1], model.n_feats))
    if vectors.device != model.device:
        raise ValueError("vectors are on %s, the model on %s" % (vectors.device, model.device))
    n = vectors.shape[0]
    if (model.n_feats > 1 and vectors.stride(1) != 1) or (n > 1 and vectors.stride(0) < model.n_feats):
        vectors = vectors.contiguous()
    with torch.cuda.device(vectors.device):
        ids = torch.empty(n, dtype=torch.int64, device=vectors.device)
        P = torch.empty((n, model.n_classes), dtype=torch.float64, device=vectors.device)
        if n == 0:
            return ids, P
        check(lib().b200aa_knn_classify(
            ctypes.c_void_p(model.features.data_ptr()), ctypes.c_void_p(model.slots.data_ptr()), model.n_train, model.n_feats,
            model.n_classes, model.k, ctypes.c_void_p(vectors.data_ptr()),
            DTYPE_F32 if vectors.dtype == torch.float32 else DTYPE_F64, n, vectors.stride(0) if n > 1 else model.n_feats,
            ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(P.data_ptr()), _stream()))
    return ids, P


def classify_vectors(classifier, model_type, vectors):
    """classifier_wrapper (audioTrainTest.py:52-93) over the rows of `vectors` [n x F]: (class ids [n], probabilities [n x classes]).
    A CUDA tensor goes to the kNN kernel (``knn_classify_batch``; `classifier` a KnnModel or a Knn-like object) and only the
    results come back; NumPy input runs on the host."""
    if isinstance(vectors, torch.Tensor):
        if model_type == "knn" and vectors.is_cuda:
            ids, P = knn_classify_batch(classifier, vectors)
            return ids.cpu().numpy(), P.cpu().numpy()
        vectors = vectors.cpu().numpy()
    vectors = np.asarray(vectors, dtype=np.float64)
    if model_type == "knn":
        return knn_classify_matrix(classifier, vectors)
    if model_type in _SKLEARN_TYPES:
        return np.asarray(classifier.predict(vectors)), np.asarray(classifier.predict_proba(vectors))
    n = vectors.shape[0]
    return np.full(n, -1), np.full(n, -1)                       # the reference's answer for an unknown type


def classify_windows(mid, mean, std, classifier, model_type):
    """Every column of a mid-term (or short-term) matrix [F x M] (NumPy, or a CUDA float32 [F, M] tensor) normalised and
    classified: (labels [M], probabilities [M x classes]) = the loop of audioSegmentation.py:579-590 / :744-748."""
    t = mid if isinstance(mid, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(mid, dtype=np.float32)).cuda()
    vec = normalize_windows_batch(t.reshape(1, t.shape[0], t.shape[1]).contiguous(), mean, std)[0]
    return classify_vectors(classifier, model_type, vec)


def mid_term_classification(signal, sampling_rate, classifier, model_type, mean, std, mt_win, mid_step, st_win, st_step):
    """The feature + classification part of audioSegmentation.mid_term_file_classification (:571-591) for a mono signal:
    returns (labels [M], max posterior per window [M]); times in seconds as in the reference's model files."""
    sig = torch.from_numpy(np.ascontiguousarray(signal)).cuda().reshape(1, -1)
    mid, _ = mid_feature_extraction_batch(sig, sampling_rate, mt_win * sampling_rate, mid_step * sampling_rate,
                                          round(sampling_rate * st_win), round(sampling_rate * st_step))
    labels, post = classify_windows(mid[0], mean, std, classifier, model_type)
    return np.asarray(labels), np.max(np.asarray(post, dtype=np.float64).reshape(len(labels), -1), axis=1)


def file_classification_vector(signal, sampling_rate, classifier, model_type, mean, std, mid_window, mid_step, short_window,
                               short_step, compute_beat=False):
    """The feature + classification part of audioTrainTest.file_classification (:1074-1095) for a mono signal:
    long-term average of the mid-term statistics (+ beat, beat confidence), normalised, classified: (class id, probabilities)."""
    n = np.asarray(signal).shape[0]
    if n / float(sampling_rate) < mid_window:
        mid_window = n / float(sampling_rate)
    sig = torch.from_numpy(np.ascontiguousarray(signal)).cuda().reshape(1, -1)
    mid, st = mid_feature_extraction_batch(sig, sampling_rate, mid_window * sampling_rate, mid_step * sampling_rate,
                                           round(sampling_rate * short_window), round(sampling_rate * short_step))
    vec = long_term_mean_batch(mid)[0].double().cpu().numpy()
    if compute_beat:
        beat, beat_conf = beat_extraction_batch(st, short_step)[0].tolist()
        vec = np.append(np.append(vec, beat), beat_conf)
    vec = (vec - np.asarray(mean, dtype=np.float64)) / np.asarray(std, dtype=np.float64)
    ids, post = classify_vectors(classifier, model_type, vec.reshape(1, -1))
    return ids[0], post[0]


def labels_to_segments(labels, window):
    """audioSegmentation.labels_to_segments (:58-99): runs of equal window labels -> (segments [n x 2] in seconds, classes)."""
    labels = list(labels)
    if len(labels) == 1:
        return [0, window], labels
    ends, classes = [], []
    start = 0
    for i in range(1, len(labels)):
        if labels[i] != labels[start] or i == len(labels) - 1:
            ends.append(i * window)
            classes.append(labels[start])
            start = i
    seg = np.zeros((len(ends), 2))
    for i, e in enumerate(ends):
        if i > 0:
            seg[i, 0] = ends[i - 1]
        seg[i, 1] = e
    return seg, classes

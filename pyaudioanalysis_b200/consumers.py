"""Consumers of the mid-term matrix (SURVEY.md 8f rank 4): the per-window normalise-and-classify loops of the reference,
batched.

The reference walks the mid-term (or short-term) matrix one column at a time:

    feature_vector = (mt_feats[:, col_index] - mean) / std              # audioSegmentation.py:581-584
    label, posterior = classifier_wrapper(classifier, model_type, feature_vector)   # audioTrainTest.py:52-93

Here all columns are normalised and transposed in ONE kernel (``b200aa_normalize_windows``: [F x M] -> [M x F] feature
vectors) and the classifier sees the whole matrix at once (scikit-learn's ``predict`` / ``predict_proba`` are row-wise, the
library's kNN runs as one kernel over a CUDA matrix of test vectors, ``b200aa_knn_classify``, and is restated below for a
NumPy one), so the results are the loop's results.  The classifiers themselves (training, model files) stay out of scope; any
object with the reference's interface works.  The library's HMMs decode a whole ragged batch in one launch pair
(``hmm_decode_batch``, ``b200aa_hmm_decode``) and train from ``hmm_statistics_batch`` (audioSegmentation.py here).  The
random forest, extra trees and gradient boosting classifiers run as one kernel over a CUDA matrix (``tree_classify_batch``,
``b200aa_trees_classify``), bit for bit scikit-learn's predict / predict_proba.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import DTYPE_F32, DTYPE_F64, ERR_UNSUPPORTED, check, lib
from .batch import _require_cuda, _stream, beat_extraction_batch, long_term_mean_batch, mid_feature_extraction_batch

_SKLEARN_TYPES = ("svm", "randomforest", "gradientboosting", "extratrees", "svm_rbf")


def _cuda_device(device, what):
    """The CUDA device `what` (a model class, with its article) is uploaded to: `device`, else the current device."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise TypeError("%s lives on a CUDA device (there is no CPU fallback)" % what)
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


def _query_matrix(model, vectors):
    """A CUDA [n, F] query tensor checked against `model` (its n_feats and device): (the tensor, made contiguous where the
    kernel cannot read its strides; its row stride; its dtype code)."""
    if vectors.dim() != 2 or vectors.dtype not in (torch.float32, torch.float64):
        raise ValueError("vectors must be float32 / float64 [n, F]")
    if vectors.shape[1] != model.n_feats:
        raise ValueError("vectors have %d features, the model %d" % (vectors.shape[1], model.n_feats))
    if vectors.device != model.device:
        raise ValueError("vectors are on %s, the model on %s" % (vectors.device, model.device))
    n = vectors.shape[0]
    if (model.n_feats > 1 and vectors.stride(1) != 1) or (n > 1 and vectors.stride(0) < model.n_feats):
        vectors = vectors.contiguous()
    return (vectors, vectors.stride(0) if n > 1 else model.n_feats,
            DTYPE_F32 if vectors.dtype == torch.float32 else DTYPE_F64)


def _concat_indices(lists, dtype):
    """A list of 1-D int64 index arrays -> (int64 offsets [len + 1], their concatenation as a contiguous `dtype` array)."""
    off = np.concatenate([[0], np.cumsum([a.size for a in lists])]).astype(np.int64)
    return off, np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0), dtype=dtype)


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
        self.device = _cuda_device(device, "a KnnModel")
        self.features = torch.from_numpy(np.ascontiguousarray(feats)).to(self.device)
        self.slots = torch.from_numpy(slots).to(self.device)


def knn_classify_batch(model, vectors):
    """Knn.classify (audioTrainTest.py:33-49) of every row of a CUDA float32 / float64 [n, F] tensor, in one kernel on the
    current stream: CUDA (ids int64 [n], P float64 [n, C]), bit for bit the reference's per-row results (DESIGN.md, kernel 5).
    `model`: a KnnModel, or a Knn-like object, uploaded for this call."""
    _require_cuda(vectors, "vectors")
    if not isinstance(model, KnnModel):
        model = KnnModel(model, vectors.device)
    vectors, stride, dtype = _query_matrix(model, vectors)
    n = vectors.shape[0]
    with torch.cuda.device(vectors.device):
        ids = torch.empty(n, dtype=torch.int64, device=vectors.device)
        P = torch.empty((n, model.n_classes), dtype=torch.float64, device=vectors.device)
        if n == 0:
            return ids, P
        check(lib().b200aa_knn_classify(
            ctypes.c_void_p(model.features.data_ptr()), ctypes.c_void_p(model.slots.data_ptr()), model.n_train, model.n_feats,
            model.n_classes, model.k, ctypes.c_void_p(vectors.data_ptr()), dtype, n, stride, ctypes.c_void_p(ids.data_ptr()),
            ctypes.c_void_p(P.data_ptr()), _stream()))
    return ids, P


def knn_cross_validate(X, y, splits, ks, n_classes=None):
    """Knn(X_train, y_train, k).classify of every test row of every (train, test) split, each split's rows standardised by
    its own StandardScaler fit (audioTrainTest.evaluate_classifier, :631-699), as one batch on the GPU
    (``b200aa_knn_cross_validate``, DESIGN.md kernel 6).

    X: float64 [n, F] (a CUDA tensor, or host data uploaded to the current device); y: the n class indices in
    [0, n_classes); splits: (train row indices, test row indices) per problem, in split order; ks: the k of each problem.
    Returns CUDA (pred int32 [sum of the test counts], the predicted class of each test row, problem after problem;
    counts int64 [P, n_classes, n_classes], counts[p, y_test, y_pred])."""
    if not isinstance(X, torch.Tensor):
        X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float64)).cuda()
    _require_cuda(X, "X")
    if X.dim() != 2 or X.dtype != torch.float64:
        raise ValueError("X must be float64 [n, F]")
    X = X.contiguous()
    n = X.shape[0]
    y = np.asarray(y.cpu() if isinstance(y, torch.Tensor) else y)
    if y.shape != (n,) or not np.array_equal(y, np.floor(y)) or (n and y.min() < 0):
        raise ValueError("y must hold one class index >= 0 per row of X")
    y = y.astype(np.int64)
    n_classes = int(y.max()) + 1 if n_classes is None else int(n_classes)
    if len(splits) != len(ks):
        raise ValueError("one k per split: %d splits, %d ks" % (len(splits), len(ks)))
    train = [np.asarray(tr, dtype=np.int64).ravel() for tr, _ in splits]
    test = [np.asarray(te, dtype=np.int64).ravel() for _, te in splits]
    train_off, train_idx = _concat_indices(train, np.int32)
    test_off, test_idx = _concat_indices(test, np.int32)
    k = np.ascontiguousarray(ks, dtype=np.int64)
    # Knn.classify's class count: len(np.unique(y_train)) of the split
    classes = np.array([np.unique(y[t[(t >= 0) & (t < n)]]).size for t in train], dtype=np.int32)
    with torch.cuda.device(X.device):
        d_y = torch.from_numpy(y.astype(np.int32)).to(X.device)
        pred = torch.empty(int(test_off[-1]), dtype=torch.int32, device=X.device)
        counts = torch.empty((len(splits), n_classes, n_classes), dtype=torch.int64, device=X.device)

        def ptr(a):
            return ctypes.c_void_p(a.ctypes.data)
        check(lib().b200aa_knn_cross_validate(
            ctypes.c_void_p(X.data_ptr()), ctypes.c_void_p(d_y.data_ptr()), n, X.shape[1], n_classes, len(splits),
            ptr(train_off), ptr(train_idx), ptr(test_off), ptr(test_idx), ptr(k), ptr(classes),
            ctypes.c_void_p(pred.data_ptr()), ctypes.c_void_p(counts.data_ptr()), _stream()))
    return pred, counts


def hmm_model_arrays(hmm):
    """(startprob [C], transmat [C, C], means [C, F], diagonal covariances [C, F]) of a diagonal GaussianHMM: hmmlearn's
    object (whose covars_ property expands the diagonal into full matrices; the stored diagonal is _covars_) or anything
    with its attribute names."""
    if getattr(hmm, "covariance_type", "diag") != "diag":
        raise ValueError("only diagonal-covariance HMMs are supported, got covariance_type %r" % (hmm.covariance_type,))
    cov = getattr(hmm, "_covars_", None)
    if cov is None:
        cov = hmm.covars_
    return (np.asarray(hmm.startprob_, dtype=np.float64), np.asarray(hmm.transmat_, dtype=np.float64),
            np.asarray(hmm.means_, dtype=np.float64), np.asarray(cov, dtype=np.float64))


def hmm_check(start, trans, means, cov):
    """hmmlearn's model checks before a decode, with its ValueError texts."""
    C = start.shape[0] if start.ndim == 1 else -1
    if C < 1:
        raise ValueError("startprob_ must have shape (n_components,)")
    if not np.allclose(start.sum(), 1.0):
        raise ValueError("startprob_ must sum to 1 (got {:.4f})".format(start.sum()))
    if trans.shape != (C, C):
        raise ValueError("transmat_ must have shape (n_components, n_components)")
    if not np.allclose(trans.sum(axis=1), 1.0):
        raise ValueError("rows of transmat_ must sum to 1 (got {})".format(trans.sum(axis=1)))
    if means.ndim != 2 or means.shape[0] != C or means.shape[1] < 1:
        raise ValueError("means_ must have shape (n_components, n_features)")
    if cov.shape != means.shape:
        raise ValueError("'diag' covars must have shape (n_components, n_dim)")
    if np.any(cov <= 0):
        raise ValueError("'diag' covars must be positive")


class HmmModel:
    """A diagonal GaussianHMM (hmmlearn's, or a look-alike: ``hmm_model_arrays``) checked as hmmlearn checks it before a
    decode and uploaded once to one CUDA device for ``hmm_decode_batch``.  The logarithms are taken here, with NumPy, as
    hmmlearn takes them: log pi and log A (-inf for a zero probability), and per state F log 2pi + sum_f log var with
    var = max(covars, tiny)."""

    def __init__(self, hmm, device=None):
        start, trans, means, cov = hmm_model_arrays(hmm)
        hmm_check(start, trans, means, cov)
        self.n_states, self.n_feats = means.shape
        var = np.maximum(cov, np.finfo(float).tiny)
        with np.errstate(divide="ignore"):
            log_start, log_trans = np.log(start), np.log(trans)
        const = self.n_feats * np.log(2 * np.pi) + np.log(var).sum(axis=-1)
        self.device = _cuda_device(device, "an HmmModel")

        def up(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(self.device)
        self.log_start, self.log_trans, self.means, self.vars, self.const = (up(a) for a in (log_start, log_trans, means, var,
                                                                                          const))


def _host_counts(n_windows, B, M, lo):
    if n_windows is None:
        return np.full(B, M, dtype=np.int64)
    n = np.ascontiguousarray(n_windows.cpu().numpy() if isinstance(n_windows, torch.Tensor) else n_windows, dtype=np.int64)
    if n.shape != (B,) or (B and (n.min() < lo or n.max() > M)):
        raise ValueError("n_windows must hold one count in [%d, %d] per clip" % (lo, M))
    return n


def hmm_decode_batch(mid, model, n_windows=None):
    """GaussianHMM.predict (hmmlearn's Viterbi) of the windows of every clip of a CUDA float32 or float64 [B, F, M]
    mid-term batch, in one launch pair on the current stream (DESIGN.md, kernel 7).  float32 is contiguous; float64 is
    contiguous, or the transpose of a contiguous [B, M, F] batch of one window per row (``X.T`` of a C-contiguous X): a
    window's density terms are then added pairwise, as predict(X) adds them, else in sequence, as predict(features.T)
    does.  ``n_windows``: each clip's window count (>= 1), host integers or a CUDA tensor; None: all M.  Returns CUDA
    (ids int32 [B, M], each clip's states and zeros past its count; bad bool [B], True for a clip with a non-finite
    feature, whose ids are left unwritten -- hmmlearn raises ValueError for it).  `model`: an HmmModel, or an HMM
    uploaded for this call."""
    _require_cuda(mid, "mid")
    window_major = (mid.dim() == 3 and mid.dtype == torch.float64 and not mid.is_contiguous()
                    and mid.transpose(1, 2).is_contiguous())
    if mid.dim() != 3 or mid.dtype not in (torch.float32, torch.float64) or not (mid.is_contiguous() or window_major):
        raise ValueError("mid must be contiguous float32 / float64 [B, F, M], or float64 [B, M, F] transposed")
    if not isinstance(model, HmmModel):
        model = HmmModel(model, mid.device)
    B, F, M = mid.shape
    if F != model.n_feats:
        raise ValueError("mid has %d features, the model %d" % (F, model.n_feats))
    if mid.device != model.device:
        raise ValueError("mid is on %s, the model on %s" % (mid.device, model.device))
    counts = _host_counts(n_windows, B, M, 1)
    with torch.cuda.device(mid.device):
        ids = torch.zeros((B, M), dtype=torch.int32, device=mid.device)
        bad = torch.zeros((B,), dtype=torch.int32, device=mid.device)
        if B and mid.dtype == torch.float64:
            check(lib().b200aa_hmm_decode_f64(
                ctypes.c_void_p(mid.data_ptr()), B, F, M, int(window_major), ctypes.c_void_p(counts.ctypes.data),
                model.n_states, ctypes.c_void_p(model.log_start.data_ptr()), ctypes.c_void_p(model.log_trans.data_ptr()),
                ctypes.c_void_p(model.means.data_ptr()), ctypes.c_void_p(model.vars.data_ptr()),
                ctypes.c_void_p(model.const.data_ptr()), ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(bad.data_ptr()),
                _stream()))
        elif B:
            check(lib().b200aa_hmm_decode(
                ctypes.c_void_p(mid.data_ptr()), B, F, M, ctypes.c_void_p(counts.ctypes.data), model.n_states,
                ctypes.c_void_p(model.log_start.data_ptr()), ctypes.c_void_p(model.log_trans.data_ptr()),
                ctypes.c_void_p(model.means.data_ptr()), ctypes.c_void_p(model.vars.data_ptr()),
                ctypes.c_void_p(model.const.data_ptr()), ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(bad.data_ptr()),
                _stream()))
    return ids, bad.bool()


def hmm_statistics_batch(mid, class_windows, n_windows=None):
    """The means and standard deviations of train_hmm_compute_statistics (audioSegmentation.py:328-342) on the GPU.

    mid: a CUDA float32 / float64 [B, F, M] batch whose clips' first n_windows[b] columns (None: all M) form one
    concatenated sequence of windows; class_windows: per class the indices of its windows in that sequence, in order.
    Returns CUDA float64 [4, C, F]: per (class, feature) the sum, mean, sum of squared deviations and population std,
    bit for bit NumPy's features[:, idx].mean(axis=1) / np.std(features[:, idx], axis=1) (DESIGN.md, kernel 7)."""
    _require_cuda(mid, "mid")
    if mid.dim() != 3 or mid.dtype not in (torch.float32, torch.float64) or not mid.is_contiguous():
        raise ValueError("mid must be contiguous float32 / float64 [B, F, M]")
    B, F, M = mid.shape
    counts = _host_counts(n_windows, B, M, 0)
    lists = [np.asarray(w, dtype=np.int64).ravel() for w in class_windows]
    off, idx = _concat_indices(lists, np.int64)
    with torch.cuda.device(mid.device):
        out = torch.empty((4, len(lists), F), dtype=torch.float64, device=mid.device)
        check(lib().b200aa_hmm_statistics(
            ctypes.c_void_p(mid.data_ptr()), DTYPE_F32 if mid.dtype == torch.float32 else DTYPE_F64, B, F, M,
            ctypes.c_void_p(counts.ctypes.data), len(lists), ctypes.c_void_p(off.ctypes.data),
            ctypes.c_void_p(idx.ctypes.data), ctypes.c_void_p(out.data_ptr()), _stream()))
    return out


def _cluster_ids(values, K, what):
    """values as int32 cluster ids, or ValueError unless each is an integer in [0, K).  Checked before any conversion:
    a cast would silently move 2**32, -0.5 or 1.7 into a cluster that NumPy's ``labels == c`` leaves them out of, and
    a negative index would mark a cluster from the end."""
    if values.dtype.kind not in "biuf" or (values.dtype.kind == "f" and not np.all(np.floor(values) == values)):
        raise ValueError("%s must be integer cluster ids" % what)
    if values.size and (values.min() < 0 or values.max() >= K):
        raise ValueError("%s must lie in [0, %d)" % (what, K))
    return values.astype(np.int32)


def cluster_distance_means(X, labels, K, rows=None):
    """The cluster distance means of speaker_diarization's silhouette (audioSegmentation.py:958-972) for one clustering,
    in one call on the current stream (``b200aa_cluster_distance_means``, DESIGN.md kernel 9).

    X: CUDA float64 [n, D] (rows at any stride; a non-unit column stride is copied); labels: n integers in [0, K), host
    or a tensor; rows: the clusters c to compute (None: all).  A label or row that is not an integer in [0, K) raises
    ValueError.  Returns CUDA float64 (A [K], B [K, K]): A[c] =
    np.mean(pdist(X[labels == c].T)), B[c, c2] = np.mean(cdist(X[labels == c], X[labels == c2])), bit for bit; NaN on the
    diagonal of B, for clusters not asked for and for a mean of no terms (D < 2, an empty cluster), where NumPy warns."""
    _require_cuda(X, "X")
    if X.dim() != 2 or X.dtype != torch.float64:
        raise ValueError("X must be float64 [n, D]")
    n, D = X.shape
    if D > 1 and X.stride(1) != 1:
        X = X.contiguous()
    labels = np.ascontiguousarray(labels.cpu().numpy() if isinstance(labels, torch.Tensor) else labels)
    if labels.shape != (n,):
        raise ValueError("labels must hold one cluster per row of X (%d)" % n)
    labels = _cluster_ids(labels, K, "labels")
    want = np.ones(K, dtype=np.uint8)
    if rows is not None:
        want[:] = 0
        want[_cluster_ids(np.asarray(list(rows)), K, "rows")] = 1
    with torch.cuda.device(X.device):
        A = torch.empty(K, dtype=torch.float64, device=X.device)
        B = torch.empty((K, K), dtype=torch.float64, device=X.device)
        check(lib().b200aa_cluster_distance_means(
            ctypes.c_void_p(X.data_ptr()), n, D, X.stride(0) if n > 1 else D, ctypes.c_void_p(labels.ctypes.data), int(K),
            ctypes.c_void_p(want.ctypes.data), ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(B.data_ptr()), _stream()))
    return A, B


def _track_rows(X, frames):
    """A CUDA float64 [sum T_b, F] matrix of tracks and its per-track frame counts: (X, made contiguous where the kernel
    cannot read its strides; its row stride; frames as int64)."""
    _require_cuda(X, "X")
    if X.dim() != 2 or X.dtype != torch.float64:
        raise ValueError("X must be float64 [frames, F]")
    n, F = X.shape
    frames = np.ascontiguousarray(np.asarray(frames).ravel())
    if frames.dtype.kind not in "iu" or frames.size < 1 or frames.min() < 1 or int(frames.sum()) != n or F < 1:
        raise ValueError("frames must be positive per-track row counts of X, summing to %d" % n)
    if F > 1 and X.stride(1) != 1:
        X = X.contiguous()
    return X, frames.astype(np.int64), X.stride(0) if n > 1 else F


def _packed(buf, sides):
    """Square [s, s] views of one packed buffer, one per side, in order."""
    off = np.concatenate([[0], np.cumsum(sides.astype(np.int64) ** 2)])
    return [buf[int(off[b]):int(off[b + 1])].view(int(s), int(s)) for b, s in enumerate(sides)]


def self_similarity_batch(X, frames):
    """The self-similarity matrices of a ragged batch of standardised tracks, in one call on the current stream
    (``b200aa_music_thumbnail``, DESIGN.md kernel 10).  X: CUDA float64 [sum T_b, F], track b the frames[b] rows after the
    tracks before it, one frame per row.  Returns a list of CUDA float64 [T_b, T_b]: 1 - squareform(pdist(X_b, 'cosine')),
    bit for bit scipy's (NaN for a zero-norm or NaN frame, 1.0 on the diagonal)."""
    X, frames, stride = _track_rows(X, frames)
    with torch.cuda.device(X.device):
        S = torch.empty(int((frames ** 2).sum()), dtype=torch.float64, device=X.device)
        check(lib().b200aa_music_thumbnail(ctypes.c_void_p(X.data_ptr()), X.shape[1], stride,
                                           ctypes.c_void_p(frames.ctypes.data), frames.size, 0, 0.0, None,
                                           ctypes.c_void_p(S.data_ptr()), None, None, _stream()))
    return _packed(S, frames)


def _limit_bounds(R, limit_1, limit_2):
    """The rows and columns [lo, hi) the reference's limit slices leave alone (audioSegmentation.py:1158-1161): ``0:int(limit_1
    * R)`` and ``int(limit_2 * R)::`` resolved by Python's slice rules."""
    return slice(0, int(limit_1 * R)).indices(R)[1], slice(int(limit_2 * R), None).indices(R)[0]


def thumbnail_host(S, filter_len, diag_gap, limit_1, limit_2):
    """The reference's steps after the similarity matrix (audioSegmentation.py:1145-1177) on the host, for the sizes the
    kernel does not take: filter_len < 1 (np.eye raises for a negative size; eye(0) gives a (T + 1)^2 matrix of zeros) and
    T < filter_len (convolve2d swaps its inputs in 'valid' mode).  Those matrices hold at most max(T + 1, filter_len)^2
    entries.  Returns ((i1, i2, j1, j2), the masked matrix)."""
    import scipy.signal
    C = scipy.signal.convolve2d(S, np.eye(filter_len, filter_len), "valid")
    min_sm = np.min(C)
    i, j = np.indices(C.shape)
    C[(np.abs(i - j) < diag_gap) | (i > j)] = min_sm
    R = C.shape[0]
    lo, hi = _limit_bounds(R, limit_1, limit_2)
    C[0:lo, :] = min_sm
    C[:, 0:lo] = min_sm
    C[hi:, :] = min_sm
    C[:, hi:] = min_sm
    r, c = np.unravel_index(C.argmax(), C.shape)
    i1, i2, j1, j2 = r, r, c, c
    while i2 - i1 < filter_len:
        if i1 <= 0 or j1 <= 0 or i2 >= C.shape[0] - 2 or j2 >= C.shape[1] - 2:
            break
        if C[i1 - 1, j1 - 1] > C[i2 + 1, j2 + 1]:
            i1, j1 = i1 - 1, j1 - 1
        else:
            i2, j2 = i2 + 1, j2 + 1
    return (i1, i2, j1, j2), C


def thumbnail_batch(X, frames, filter_len, diag_gap, limit_1=0, limit_2=1):
    """music_thumbnailing's steps after the scaler (audioSegmentation.py:1140-1177) for a ragged batch of standardised
    tracks, in one call on the current stream (``b200aa_music_thumbnail``, DESIGN.md kernel 10).  X and frames as for
    ``self_similarity_batch``; filter_len = int(round(thumb_size / short_step)); diag_gap = 5.0 / short_step.  Returns
    (idx int64 [B, 4]: i1, i2, j1, j2 of each track, frame indices; a list of CUDA float64 [R_b, R_b], the masked filtered
    matrices), bit for bit the reference's.  A track shorter than filter_len, and every track when filter_len < 1, runs
    its filter, mask and walk on the host (``thumbnail_host``) from the kernel's similarity matrix."""
    X, frames, stride = _track_rows(X, frames)
    m = int(filter_len)
    device = (frames >= m) & (m >= 1)
    B = frames.size
    idx = np.zeros((B, 4), dtype=np.int64)
    out = [None] * B
    with torch.cuda.device(X.device):
        if device.any():
            row0 = np.concatenate([[0], np.cumsum(frames)])
            rows = np.concatenate([np.arange(row0[b], row0[b + 1]) for b in np.flatnonzero(device)])
            Xd = X if device.all() else X[torch.as_tensor(rows, device=X.device)]
            fd = frames[device]
            R = fd - m + 1
            limits = np.ascontiguousarray([_limit_bounds(int(r), limit_1, limit_2) for r in R], dtype=np.int64)
            C = torch.empty(int((R ** 2).sum()), dtype=torch.float64, device=X.device)
            d_idx = torch.empty((fd.size, 4), dtype=torch.int64, device=X.device)
            check(lib().b200aa_music_thumbnail(
                ctypes.c_void_p(Xd.data_ptr()), X.shape[1], Xd.stride(0) if Xd is not X else stride,
                ctypes.c_void_p(fd.ctypes.data), fd.size, m, float(diag_gap), ctypes.c_void_p(limits.ctypes.data), None,
                ctypes.c_void_p(C.data_ptr()), ctypes.c_void_p(d_idx.data_ptr()), _stream()))
            idx[device] = d_idx.cpu().numpy()
            for b, c in zip(np.flatnonzero(device), _packed(C, R)):
                out[b] = c
        if not device.all():
            host = np.flatnonzero(~device)
            row0 = np.concatenate([[0], np.cumsum(frames)])
            Xh = X[torch.as_tensor(np.concatenate([np.arange(row0[b], row0[b + 1]) for b in host]), device=X.device)]
            for b, S in zip(host, self_similarity_batch(Xh, frames[host])):
                (i1, i2, j1, j2), C = thumbnail_host(S.cpu().numpy(), m, diag_gap, limit_1, limit_2)
                idx[b] = (i1, i2, j1, j2)
                out[b] = torch.from_numpy(C).to(X.device)
    return idx, out


def _scale_into(X, rows, out, out_off, out_row_stride, out_col_stride):
    """b200aa_standard_scale of X [B, n_max, D] (CUDA float32 / float64, strides >= 1) into `out` at the element offsets
    out_off [B]: (mean, scale) CUDA float64 [B, D].  A matrix holding +-inf is handed to scikit-learn, which raises."""
    B, n_max, D = X.shape
    with torch.cuda.device(X.device):
        mean = torch.empty((B, D), dtype=torch.float64, device=X.device)
        scale = torch.empty((B, D), dtype=torch.float64, device=X.device)
        bad = torch.empty(B, dtype=torch.int32, device=X.device)
        check(lib().b200aa_standard_scale(
            ctypes.c_void_p(X.data_ptr()), DTYPE_F32 if X.dtype == torch.float32 else DTYPE_F64, B, D,
            ctypes.c_void_p(rows.ctypes.data), X.stride(0), X.stride(1), X.stride(2), ctypes.c_void_p(out.data_ptr()),
            ctypes.c_void_p(out_off.ctypes.data), out_row_stride, out_col_stride, ctypes.c_void_p(mean.data_ptr()),
            ctypes.c_void_p(scale.data_ptr()), ctypes.c_void_p(bad.data_ptr()), _stream()))
    for b in np.flatnonzero(bad.cpu().numpy()):
        from sklearn.preprocessing import StandardScaler
        StandardScaler().fit_transform(X[b, :rows[b]].cpu().numpy().astype(np.float64))
        raise ValueError("Input X contains infinity or a value too large for dtype('float64').")
    return mean, scale


def _scale_input(X, rows):
    """X as a CUDA [B, n_max, D] float tensor with strides >= 1 and its row counts as int64 [B]."""
    _require_cuda(X, "X")
    if X.dim() not in (2, 3) or X.dtype not in (torch.float32, torch.float64):
        raise ValueError("X must be float32 / float64 [n, D] or [B, n, D]")
    X3 = X.unsqueeze(0) if X.dim() == 2 else X
    B, n_max, D = X3.shape
    if B < 1 or n_max < 1 or D < 1:
        raise ValueError("X must hold at least one matrix of one row and one column")
    if min(X3.stride()) < 1:
        X3 = X3.contiguous()
    rows = np.full(B, n_max, dtype=np.int64) if rows is None else np.ascontiguousarray(np.asarray(rows).ravel())
    if rows.dtype.kind not in "iu" or rows.shape != (B,) or rows.min() < 1 or rows.max() > n_max:
        raise ValueError("rows must be one count in [1, %d] per matrix" % n_max)
    return X3, rows.astype(np.int64)


def standard_scale_batch(X, rows=None):
    """StandardScaler().fit_transform of every matrix of a batch, in one call on the current stream
    (``b200aa_standard_scale``, DESIGN.md kernel 11), bit for bit scikit-learn 1.9.

    X: CUDA float32 (widened) or float64, one matrix [n, D] or a batch [B, n_max, D] at any strides, matrix b its first
    rows[b] rows (default: all).  As NumPy's axis-0 sums, a matrix whose row stride is below its column stride (a
    column-major matrix, such as the transpose of a C-contiguous [D, n] array) has each column summed pairwise, any other
    row by row.  NaN is left out of the statistics and passes through; a matrix holding +-inf raises scikit-learn's
    ValueError.  Returns (Y, mean, scale): Y CUDA float64 of X's shape in the layout scikit-learn returns (column-major
    matrices for a column-major X, else C-contiguous), zero past each matrix's rows; mean and scale CUDA float64 [B, D]
    (or [D]), scikit-learn's mean_ and scale_."""
    X3, rows = _scale_input(X, rows)
    B, n_max, D = X3.shape
    column_major = D == 1 or X3.stride(1) < X3.stride(2)
    with torch.cuda.device(X3.device):
        if column_major:
            Y = torch.zeros((B, D, n_max), dtype=torch.float64, device=X3.device).transpose(1, 2)
        else:
            Y = torch.zeros((B, n_max, D), dtype=torch.float64, device=X3.device)
    mean, scale = _scale_into(X3, rows, Y, np.arange(B, dtype=np.int64) * n_max * D, Y.stride(1), Y.stride(2))
    if X.dim() == 2:
        return Y[0], mean[0], scale[0]
    return Y, mean, scale


def outlier_columns(X):
    """The feature-outlier rule of speaker_diarization (audioSegmentation.py:861-865) for a normalised CUDA float64 [M, D]
    matrix, in one call on the current stream (``b200aa_outlier_columns``, DESIGN.md kernel 11): dist_all =
    np.sum(squareform(pdist(X.T)), axis=0) and the columns with dist_all < 1.1 * np.mean(dist_all), bit for bit.  A
    matrix whose columns are not contiguous is copied.  Returns (i_non_outliers int64 NumPy, dist_all CUDA float64 [D])."""
    _require_cuda(X, "X")
    if X.dim() != 2 or X.dtype != torch.float64 or X.shape[0] < 1 or X.shape[1] < 1:
        raise ValueError("X must be float64 [M, D] with M, D >= 1")
    M, D = X.shape
    if M > 1 and X.stride(0) != 1 or D > 1 and X.stride(1) < M:
        X = X.t().contiguous().t()
    with torch.cuda.device(X.device):
        dist_all = torch.empty(D, dtype=torch.float64, device=X.device)
        mean = torch.empty(1, dtype=torch.float64, device=X.device)
        keep = torch.empty(D, dtype=torch.uint8, device=X.device)
        check(lib().b200aa_outlier_columns(ctypes.c_void_p(X.data_ptr()), M, D, X.stride(1) if D > 1 else M,
                                           ctypes.c_void_p(dist_all.data_ptr()), ctypes.c_void_p(mean.data_ptr()),
                                           ctypes.c_void_p(keep.data_ptr()), _stream()))
    return np.flatnonzero(keep.cpu().numpy()).astype(np.int64), dist_all


def pool_frames_batch(st, ratio, frames=None):
    """The LDA branch's pooling of speaker_diarization (audioSegmentation.py:884-906, ``audioSegmentation.pool_frames``)
    for a ragged batch, in one call on the current stream (``b200aa_pool_frames``, DESIGN.md kernel 11).  st: CUDA
    float32 (widened) or float64 [F, T] or [B, F, T], clip b its first frames[b] frames (default: all).  Returns CUDA
    float64 [2F, T] / [B, 2F, T]: row f at frame i the np.mean and row F + f the np.std of frames [i, min(i + ratio, T_b))
    of row f, bit for bit; zero past each clip's frames.  ratio < 1 raises ValueError."""
    _require_cuda(st, "st")
    if st.dim() not in (2, 3) or st.dtype not in (torch.float32, torch.float64):
        raise ValueError("st must be float32 / float64 [F, T] or [B, F, T]")
    s3 = st.unsqueeze(0) if st.dim() == 2 else st
    B, F, T = s3.shape
    if B < 1 or F < 1 or T < 1:
        raise ValueError("st must hold at least one clip of one row and one frame")
    if (T > 1 and s3.stride(2) != 1) or min(s3.stride()) < 0:
        s3 = s3.contiguous()
    frames = np.full(B, T, dtype=np.int64) if frames is None else np.ascontiguousarray(np.asarray(frames).ravel())
    if frames.dtype.kind not in "iu" or frames.shape != (B,) or frames.min() < 1 or frames.max() > T:
        raise ValueError("frames must be one count in [1, %d] per clip" % T)
    frames = frames.astype(np.int64)
    if int(ratio) != ratio or ratio < 1:
        raise ValueError("ratio must be an integer >= 1")
    with torch.cuda.device(s3.device):
        out = torch.zeros((B, 2 * F, T), dtype=torch.float64, device=s3.device)
        check(lib().b200aa_pool_frames(ctypes.c_void_p(s3.data_ptr()), DTYPE_F32 if s3.dtype == torch.float32 else DTYPE_F64,
                                       B, F, s3.stride(0), s3.stride(1), ctypes.c_void_p(frames.ctypes.data), int(ratio),
                                       ctypes.c_void_p(out.data_ptr()), T, _stream()))
    return out[0] if st.dim() == 2 else out


TREE_FOREST, TREE_BOOST = 0, 1
_TREE_TYPES = ("randomforest", "extratrees", "gradientboosting")


def _threshold_down(t):
    """Each float64 threshold rounded toward -inf to float32: for float32 x, x <= t exactly when x <= the result."""
    with np.errstate(over="ignore"):
        f = t.astype(np.float32)
    below = f.astype(np.float64) > t
    f[below] = np.nextafter(f[below], np.float32(-np.inf))
    return f


def flatten_tree_ensemble(model):
    """The arrays kernel 8 walks (include/b200aa.h, b200aa_trees_create) of a fitted RandomForestClassifier,
    ExtraTreesClassifier or GradientBoostingClassifier, in NumPy: a dict of nodes int32 [n_nodes, 4] (left, right, feature
    with bit 31 set where a NaN goes left, float32 threshold bits; a leaf has left -1 and right its row of values), roots
    int32 [n_trees], values float64 ([n_leaves, C] class fractions for a forest; [n_leaves] learning rate x leaf value for
    boosting), mode, n_classes (C, or K raw scores for boosting), n_feats, init (boosting's constant raw start) and
    allow_nan.  Raises ValueError for anything else: regressors, multi-output forests, a boosting init that is not
    constant per row."""
    from sklearn.dummy import DummyClassifier
    from sklearn.ensemble import ExtraTreesClassifier, GradientBoostingClassifier, RandomForestClassifier

    if isinstance(model, (RandomForestClassifier, ExtraTreesClassifier)):
        if not hasattr(model, "estimators_"):
            raise ValueError("the forest is not fitted")
        if model.n_outputs_ != 1:
            raise ValueError("multi-output forests are not supported (n_outputs_ = %d)" % model.n_outputs_)
        mode, C, scale = TREE_FOREST, int(model.n_classes_), None
        trees = [e.tree_ for e in model.estimators_]
        init = None
        allow_nan = bool(model.estimators_[0]._support_missing_values(np.zeros((1, model.n_features_in_), np.float32)))
    elif isinstance(model, GradientBoostingClassifier):
        if not hasattr(model, "estimators_"):
            raise ValueError("the model is not fitted")
        init_ = model.init_
        if not (isinstance(init_, str) and init_ == "zero") and not (
                isinstance(init_, DummyClassifier) and init_.strategy == "prior"):
            raise ValueError("only a 'zero' or DummyClassifier(strategy='prior') init is supported, got %r" % (init_,))
        mode, C, scale = TREE_BOOST, int(model.estimators_.shape[1]), float(model.learning_rate)
        trees = [e.tree_ for e in model.estimators_.ravel()]       # stage-major: tree s * K + k adds to raw score k
        init = np.ascontiguousarray(model._raw_predict_init(np.zeros((1, model.n_features_in_), np.float32))[0],
                                    dtype=np.float64)
        allow_nan = False
    else:
        raise ValueError("tree inference supports RandomForestClassifier, ExtraTreesClassifier and "
                         "GradientBoostingClassifier, got %s" % type(model).__name__)
    nodes, values, roots = [], [], []
    base = leaf_base = 0
    for tr in trees:
        left = tr.children_left.astype(np.int64)
        leaf = left < 0
        n_leaf = int(leaf.sum())
        nd = np.zeros((tr.node_count, 4), dtype=np.int32)
        leaf_row = np.cumsum(leaf) - 1 + leaf_base
        nd[:, 0] = np.where(leaf, -1, left + base)
        nd[:, 1] = np.where(leaf, leaf_row, tr.children_right.astype(np.int64) + base)
        feat = np.where(leaf, 0, tr.feature).astype(np.int64)
        missing = np.asarray(tr.missing_go_to_left, dtype=bool) & ~leaf
        nd[:, 2] = (feat | np.where(missing, 1 << 31, 0)).astype(np.uint32).view(np.int32)
        nd[:, 3] = np.where(leaf, np.float32(0), _threshold_down(tr.threshold)).astype(np.float32).view(np.int32)
        v = tr.value[leaf, 0, :]
        values.append(v[:, :C] if mode == TREE_FOREST else scale * v[:, 0])
        nodes.append(nd)
        roots.append(base)
        base += tr.node_count
        leaf_base += n_leaf
    return {"nodes": np.ascontiguousarray(np.concatenate(nodes)), "roots": np.asarray(roots, dtype=np.int32),
            "values": np.ascontiguousarray(np.concatenate(values), dtype=np.float64), "mode": mode, "n_classes": C,
            "n_feats": int(model.n_features_in_), "init": init, "allow_nan": allow_nan}


class TreeEnsembleModel:
    """A fitted RandomForestClassifier, ExtraTreesClassifier or GradientBoostingClassifier (``flatten_tree_ensemble``)
    uploaded once to one CUDA device for ``tree_classify_batch`` (kernel 8).  Raises ValueError for a model it cannot
    reproduce bit for bit."""

    def __init__(self, model, device=None):
        flat = flatten_tree_ensemble(model)
        self.estimator = model
        self.classes = np.asarray(model.classes_)
        self.mode, self.n_classes, self.n_feats = flat["mode"], flat["n_classes"], flat["n_feats"]
        self.device = _cuda_device(device, "a TreeEnsembleModel")
        nodes, roots, values, init = flat["nodes"], flat["roots"], flat["values"], flat["init"]
        _lib.refuse_capture("b200aa_trees_create", "allocates and uploads the model; create it outside capture")
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            status = lib().b200aa_trees_create(
                ctypes.byref(h), ctypes.c_void_p(nodes.ctypes.data), nodes.shape[0], ctypes.c_void_p(roots.ctypes.data),
                roots.shape[0], ctypes.c_void_p(values.ctypes.data), values.shape[0], self.n_classes, self.n_feats,
                self.mode, None if init is None else ctypes.c_void_p(init.ctypes.data), int(flat["allow_nan"]))
        if status == ERR_UNSUPPORTED:
            raise ValueError("a row of %d features and %d classes needs more shared memory than the tree kernel takes"
                             % (self.n_feats, self.n_classes))
        check(status)
        self.handle = h

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            lib().b200aa_trees_destroy(h)


def _ptr(a):
    """A host array's address for the C ABI (None: NULL)."""
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def _forest_X(X, Xh):
    """X as the forest trainers read it: a CUDA float32 / float64 tensor with unit column stride as it is (cast to float32
    on the device, round to nearest, as fit casts), anything else through fit's own cast straight to float32 (any
    integer or float dtype rounds once)."""
    if isinstance(X, torch.Tensor) and X.is_cuda and X.dtype in (torch.float32, torch.float64) and X.stride(1) == 1:
        return X
    return torch.from_numpy(np.ascontiguousarray(Xh, dtype=np.float32)).cuda()


def _tree_states(nodes, values, counts, depth, n_outputs):
    """Tree.__getstate__ of every tree of a fit, its nodes and values following the trees before it."""
    from . import forests as FO
    states, off = [], 0
    for nc, d in zip(counts, depth):
        nc = int(nc)
        states.append(FO.tree_state(nodes[off:off + nc], values[off:off + nc], d, n_outputs))
        off += nc
    return states


def _cv_X(X):
    """A model selection's X as a C-contiguous CUDA float64 [n, F] tensor."""
    if not isinstance(X, torch.Tensor):
        X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float64)).cuda()
    _require_cuda(X, "X")
    if X.dim() != 2 or X.dtype != torch.float64:
        raise ValueError("X must be float64 [n, F]")
    return X.contiguous()


def _cv_splits(splits, seeds, n_estimators, what):
    """A model selection's (train, test) splits, one seed list and one `what` count per split: the training and test row
    lists, and both as (offsets int64, indices int32)."""
    if not len(splits) == len(seeds) == len(n_estimators):
        raise ValueError("one seed list and one %s count per split" % what)
    train = [np.asarray(tr, dtype=np.int64).ravel() for tr, _ in splits]
    test = [np.asarray(te, dtype=np.int64).ravel() for _, te in splits]
    return train, test, _concat_indices(train, np.int32), _concat_indices(test, np.int32)


def _forest_draws(seeds, n_trees, train, kind):
    """Every problem's bootstrap weights (int32, None for extra trees) and splitter seeds (uint32) from its tree seeds."""
    from . import forests as FO
    if any(len(s) != t for s, t in zip(seeds, n_trees)):
        raise ValueError("every problem needs one seed per tree")
    ws, rs = [], []
    for s, tr in zip(seeds, train):
        w, r = FO.derive(s, kind, tr.size)
        if w is not None:
            ws.append(w.ravel())
        rs.append(r)
    weights = np.ascontiguousarray(np.concatenate(ws), dtype=np.int32) if ws else None
    return weights, np.ascontiguousarray(np.concatenate(rs), dtype=np.uint32)


def _scratch_refusal(status, what, rows, F, state=None):
    """forests.Unsupported for a tree over the trainer's scratch bound (NumPy's global state put back to `state` first,
    when given), else check(status).  rows: the tree's rows, as the message names them."""
    from . import forests as FO
    if status == ERR_UNSUPPORTED:
        if state is not None:
            np.random.set_state(state)
        raise FO.Unsupported("%s on the GPU: one tree of %s x %d features needs more scratch than the trainer's 256 MB "
                             "bound" % (what, rows, F))
    check(status)


def forest_fit(X, y, n_estimators, kind):
    """``RandomForestClassifier(n_estimators).fit(X, y)`` (kind "randomforest") or ``ExtraTreesClassifier`` (kind
    "extratrees") trained on the GPU (``b200aa_forest_fit``, DESIGN.md kernel 13), tree for tree scikit-learn 1.9's under
    the same NumPy global state, which it leaves as ``fit`` leaves it.  Returns the fitted scikit-learn estimator.

    X: float64 / float32 [n, F] host array (or a CUDA tensor, which is read from the device); y: n labels.  Raises
    ValueError with ``forests.unsupported``'s reason for what it does not reproduce; ``train_random_forest`` /
    ``train_extra_trees`` hand those calls to scikit-learn."""
    from . import forests as FO
    Xh = X.detach().cpu().numpy() if isinstance(X, torch.Tensor) else X
    why = FO.unsupported(Xh, y, n_estimators, kind)
    if why is not None:
        raise ValueError("forest_fit on the GPU: " + why)
    n, F = Xh.shape
    classes, y_idx = np.unique(np.asarray(y), return_inverse=True)
    C = len(classes)
    d_X = _forest_X(X, Xh)
    est, trees, weights, seeds = FO.draw(int(n_estimators), kind, n)
    cap = int(n_estimators) * (2 * n - 1)
    nodes = np.empty(cap, dtype=FO.NODE_DTYPE)
    values = np.empty((cap, C), dtype=np.float64)
    counts = np.empty(int(n_estimators), dtype=np.int64)
    depth = np.empty(int(n_estimators), dtype=np.int32)
    y32 = np.ascontiguousarray(y_idx, dtype=np.int32)
    with torch.cuda.device(d_X.device):
        check(lib().b200aa_forest_fit(
            ctypes.c_void_p(d_X.data_ptr()), DTYPE_F32 if d_X.dtype == torch.float32 else DTYPE_F64, n, F, d_X.stride(0),
            _ptr(y32), C, FO.KINDS[kind], int(n_estimators), max(1, int(np.sqrt(F))), _ptr(weights), _ptr(seeds),
            _ptr(nodes), _ptr(values), cap, _ptr(counts), _ptr(depth), _stream()))
    return FO.assemble(est, trees, F, n, classes, _tree_states(nodes, values, counts, depth, C))


def forest_cross_validate(X, y, splits, seeds, n_estimators, kind, n_classes=None):
    """The forest branch of evaluate_classifier's model selection (audioTrainTest.py:631-699) as one batch on the GPU
    (``b200aa_forest_cross_validate``, DESIGN.md kernel 13): per (train, test) split, StandardScaler fit on the training
    rows, ``RandomForestClassifier`` / ``ExtraTreesClassifier(n_estimators[p]).fit`` (kind "randomforest" /
    "extratrees") on them, and predict of every test row, bit for bit scikit-learn's.  The forests stay on the device.

    X: float64 [n, F] (host, or a CUDA tensor); y: the n class indices in [0, n_classes); splits: (train, test) row
    indices per problem; seeds: per problem the tree seeds fit would draw (``forests.tree_seeds``); n_estimators: the tree
    count per problem.  Returns CUDA (pred int32 [sum of the test counts], counts int64 [P, n_classes, n_classes])."""
    from . import forests as FO
    if kind not in FO.KINDS:
        raise ValueError("kind must be 'randomforest' or 'extratrees', got %r" % (kind,))
    X = _cv_X(X)
    n = X.shape[0]
    y = np.asarray(y.cpu() if isinstance(y, torch.Tensor) else y)
    if y.shape != (n,) or not np.array_equal(y, np.floor(y)) or (n and y.min() < 0):
        raise ValueError("y must hold one class index >= 0 per row of X")
    y = y.astype(np.int32)
    n_classes = int(y.max()) + 1 if n_classes is None else int(n_classes)
    train, _, (train_off, train_idx), (test_off, test_idx) = _cv_splits(splits, seeds, n_estimators, "tree")
    n_trees = np.ascontiguousarray(n_estimators, dtype=np.int32)
    weights, rand_r = _forest_draws(seeds, n_trees, train, kind)
    with torch.cuda.device(X.device):
        pred = torch.empty(int(test_off[-1]), dtype=torch.int32, device=X.device)
        counts = torch.empty((len(splits), n_classes, n_classes), dtype=torch.int64, device=X.device)
        check(lib().b200aa_forest_cross_validate(
            ctypes.c_void_p(X.data_ptr()), n, X.shape[1], _ptr(y), n_classes, FO.KINDS[kind], len(splits),
            _ptr(train_off), _ptr(train_idx), _ptr(test_off), _ptr(test_idx), _ptr(n_trees), _ptr(weights), _ptr(rand_r),
            ctypes.c_void_p(pred.data_ptr()), ctypes.c_void_p(counts.data_ptr()), _stream()))
    return pred, counts


def forest_regressor_fit(X, y, n_estimators):
    """``RandomForestRegressor(n_estimators).fit(X, y)`` trained on the GPU (``b200aa_forest_regressor_fit``, DESIGN.md
    kernel 13, regression), tree for tree scikit-learn 1.9's under the same NumPy global state, which it leaves as ``fit``
    leaves it.  Returns the fitted scikit-learn estimator.

    X: float64 / float32 [n, F] host array (or a CUDA tensor, which is read from the device); y: n finite targets.
    Raises ValueError with ``forests.unsupported_regressor``'s reason for what it does not reproduce, and
    ``forests.Unsupported`` (a ValueError), with NumPy's global state as before the call, when one tree's scratch would
    exceed the trainer's 256 MB bound (at 136 features, more than 131 072 rows); ``train_random_forest_regression`` hands
    those calls to scikit-learn."""
    from . import forests as FO
    Xh = X.detach().cpu().numpy() if isinstance(X, torch.Tensor) else X
    why = FO.unsupported_regressor(Xh, y, n_estimators)
    if why is not None:
        raise ValueError("forest_regressor_fit on the GPU: " + why)
    n, F = Xh.shape
    d_X = _forest_X(X, Xh)
    T = int(n_estimators)
    state = np.random.get_state()
    est, trees, weights, seeds = FO.draw(T, FO.REGRESSOR, n)
    cap = T * (2 * n - 1)
    nodes = np.empty(cap, dtype=FO.NODE_DTYPE)
    values = np.empty(cap, dtype=np.float64)
    counts = np.empty(T, dtype=np.int64)
    depth = np.empty(T, dtype=np.int32)
    y64 = np.ascontiguousarray(y, dtype=np.float64)
    with torch.cuda.device(d_X.device):
        status = lib().b200aa_forest_regressor_fit(
            ctypes.c_void_p(d_X.data_ptr()), DTYPE_F32 if d_X.dtype == torch.float32 else DTYPE_F64, n, F, d_X.stride(0),
            _ptr(y64), T, _ptr(weights), _ptr(seeds), _ptr(nodes), _ptr(values), cap, _ptr(counts), _ptr(depth), _stream())
    _scratch_refusal(status, "forest_regressor_fit", "%d rows" % n, F, state)
    return FO.assemble_regressor(est, trees, F, n, _tree_states(nodes, values, counts, depth, 1))


def forest_regression_cross_validate(X, y, splits, seeds, n_estimators):
    """The "randomforest" branch of evaluate_regression's model selection as one batch on the GPU
    (``b200aa_forest_regression_cross_validate``, DESIGN.md kernel 13, regression): StandardScaler().fit_transform of
    the whole matrix once, then per (train, test) split ``RandomForestRegressor(n_estimators[p]).fit`` on the training
    rows and predict of the test and training rows, bit for bit scikit-learn's.  The forests stay on the device.

    X: C-contiguous float64 [n, F] (host, or a CUDA tensor); y: n finite targets; splits: (train, test) row indices per
    problem; seeds: per problem the tree seeds fit would draw (``forests.tree_seeds(T, forests.REGRESSOR)``); n_estimators: the tree
    count per problem.  Returns CUDA float64 (test predictions [sum of the test counts], training predictions [sum of the
    training counts]), each problem's rows in its split's order.  Raises ``forests.Unsupported`` when one tree of the
    largest training set would exceed the trainer's 256 MB scratch bound."""
    from . import forests as FO
    X = _cv_X(X)
    n = X.shape[0]
    y = np.ascontiguousarray(y.cpu() if isinstance(y, torch.Tensor) else y, dtype=np.float64)
    if y.shape != (n,) or not np.isfinite(y).all():
        raise ValueError("y must hold one finite target per row of X")
    train, _, (train_off, train_idx), (test_off, test_idx) = _cv_splits(splits, seeds, n_estimators, "tree")
    n_trees = np.ascontiguousarray(n_estimators, dtype=np.int32)
    weights, rand_r = _forest_draws(seeds, n_trees, train, FO.REGRESSOR)
    with torch.cuda.device(X.device):
        pred_test = torch.empty(int(test_off[-1]), dtype=torch.float64, device=X.device)
        pred_train = torch.empty(int(train_off[-1]), dtype=torch.float64, device=X.device)
        status = lib().b200aa_forest_regression_cross_validate(
            ctypes.c_void_p(X.data_ptr()), n, X.shape[1], _ptr(y), len(splits), _ptr(train_off), _ptr(train_idx),
            _ptr(test_off), _ptr(test_idx), _ptr(n_trees), _ptr(weights), _ptr(rand_r),
            ctypes.c_void_p(pred_test.data_ptr()), ctypes.c_void_p(pred_train.data_ptr()), _stream())
    _scratch_refusal(status, "forest_regression_cross_validate", "%d training rows" % max(t.size for t in train),
                     X.shape[1])
    return pred_test, pred_train


def boosting_fit(X, y, n_estimators):
    """``GradientBoostingClassifier(n_estimators).fit(X, y)`` trained on the GPU (``b200aa_boosting_stage``, DESIGN.md
    kernel 13, gradient boosting), stage for stage scikit-learn 1.9's under the same NumPy global state, which it leaves
    as ``fit`` leaves it.  Each stage's negative gradient and train_score_ are computed on the host by scikit-learn's own
    loss; the trees, their Newton leaf values and the raw-prediction update run on the device.  Returns the fitted
    scikit-learn estimator.

    X: float64 / float32 [n, F] host array (or a CUDA tensor, which is read from the device); y: n labels.  Raises
    ValueError with ``boosting.unsupported``'s reason for what it does not reproduce, and ``forests.Unsupported`` (a
    ValueError), with NumPy's global state as before the call, when one tree's scratch would exceed the trainer's 256 MB
    bound; ``train_gradient_boosting`` hands those calls to scikit-learn."""
    from . import boosting as BO
    from . import forests as FO
    Xh = X.detach().cpu().numpy() if isinstance(X, torch.Tensor) else X
    why = BO.unsupported(Xh, y, n_estimators)
    if why is not None:
        raise ValueError("boosting_fit on the GPU: " + why)
    n, F = Xh.shape
    T = int(n_estimators)
    est, X32, y_enc, raw0 = BO.begin(Xh, y, T)
    K = est.n_trees_per_iteration_
    if isinstance(X, torch.Tensor) and X.is_cuda and X.dtype in (torch.float32, torch.float64):
        d_X = X.to(torch.float32).contiguous()     # fit's cast to float32, round to nearest
    else:
        d_X = torch.from_numpy(np.ascontiguousarray(X32)).to(X.device if isinstance(X, torch.Tensor) and X.is_cuda else "cuda")
    state = np.random.get_state()
    seeds = BO.draw_seeds(T * K)
    raw = np.ascontiguousarray(np.broadcast_to(raw0, (n, K)), dtype=np.float64)
    sw = np.ones(n)
    factor = BO.loss_factor(est._loss)
    train_off, test_off = np.array([0, n], np.int64), None
    rows = np.arange(n, dtype=np.int32)
    K_arr, active = np.array([K], np.int32), np.ones(1, np.int32)
    cap = K * (2 * n - 1)
    nodes = np.empty(cap, dtype=FO.NODE_DTYPE)
    values = np.empty(cap, dtype=np.float64)
    counts = np.empty(K, dtype=np.int64)
    depth = np.empty(K, dtype=np.int32)
    with torch.cuda.device(d_X.device):
        d_y = torch.from_numpy(y_enc.astype(np.int32)).to(d_X.device)
        d_raw = torch.from_numpy(raw).to(d_X.device)
        d_neg = torch.empty((n, K), dtype=torch.float64, device=d_X.device)
        for i in range(T):
            d_neg.copy_(torch.from_numpy(BO.neg_gradient(est._loss, y_enc, raw)))
            status = lib().b200aa_boosting_stage(
                ctypes.c_void_p(d_X.data_ptr()), n, F, 1, _ptr(train_off), _ptr(rows), None, None, _ptr(K_arr),
                _ptr(active), ctypes.c_void_p(d_y.data_ptr()), ctypes.c_void_p(d_neg.data_ptr()),
                ctypes.c_void_p(d_raw.data_ptr()), None, _ptr(seeds[i * K:(i + 1) * K]), float(est.learning_rate),
                _ptr(nodes), _ptr(values), cap, _ptr(counts), _ptr(depth), _stream())
            _scratch_refusal(status, "boosting_fit", "%d training rows" % n, F, state)
            raw = d_raw.cpu().numpy()
            est.train_score_[i] = factor * est._loss(y_true=y_enc, raw_prediction=raw, sample_weight=sw)
            for k, tree in enumerate(_tree_states(nodes, values, counts, depth, 1)):
                est.estimators_[i, k] = BO.make_tree(est, F, tree)
    est.n_estimators_ = T
    return est


def boosting_cross_validate(X, y, splits, seeds, n_estimators, n_classes=None):
    """The "gradientboosting" branch of evaluate_classifier's model selection (audioTrainTest.py:631-699) on the GPU:
    per (train, test) split, StandardScaler fit on the training rows (``b200aa_boosting_scale``),
    ``GradientBoostingClassifier(n_estimators[p]).fit`` on them stage for stage scikit-learn's, every problem's stage in
    one call (``b200aa_boosting_stage``; problems drop out once their stages are done), the test rows' raw scores updated
    with each stage's trees, and predict's class of every test row counted (``b200aa_boosting_count``).  The trees stay
    on the device; each stage's negative gradients are computed on the host with scikit-learn's loss.

    X: float64 [n, F] (host, or a CUDA tensor); y: the n class indices in [0, n_classes); splits: (train, test) row
    indices per problem, every training set holding at least two classes; seeds: per problem the n_estimators[p] * K_p
    splitter seeds its fit draws (``boosting.draw_seeds``; K_p from the classes in its training rows).  Returns CUDA (pred
    int32 [sum of the test counts], counts int64 [P, n_classes, n_classes]).  Raises ``forests.Unsupported`` when one tree
    of the largest training set would exceed the trainer's 256 MB scratch bound."""
    from . import boosting as BO
    X = _cv_X(X)
    n, F = X.shape
    y = np.asarray(y.cpu() if isinstance(y, torch.Tensor) else y)
    if y.shape != (n,) or not np.array_equal(y, np.floor(y)) or (n and y.min() < 0):
        raise ValueError("y must hold one class index >= 0 per row of X")
    n_classes = int(y.max()) + 1 if n_classes is None else int(n_classes)
    P = len(splits)
    train, test, (train_off, train_idx), (test_off, test_idx) = _cv_splits(splits, seeds, n_estimators, "stage")
    n_tr, n_te = int(train_off[-1]), int(test_off[-1])
    stages = np.asarray(n_estimators, dtype=np.int64)
    # each problem's fit preamble on the host: present classes, K, loss, encoded labels, initial raw prediction
    init = [BO.problem_init(y[tr].astype(np.float64)) for tr in train]
    K = np.array([k for _, k, _, _, _ in init], dtype=np.int32)
    if any(c.size < 2 for c, _, _, _, _ in init):
        raise ValueError("every training set needs two classes (fit raises otherwise)")
    if any(len(s) != t * k for s, t, k in zip(seeds, stages, K)):
        raise ValueError("every problem needs n_estimators * K seeds")
    seeds = [np.asarray(s, dtype=np.uint32) for s in seeds]
    g_off = np.concatenate([[0], np.cumsum([tr.size * k for tr, k in zip(train, K)])]).astype(np.int64)
    t_off = np.concatenate([[0], np.cumsum([te.size * k for te, k in zip(test, K)])]).astype(np.int64)
    raw_tr = np.concatenate([np.broadcast_to(r0, (tr.size, k)).ravel() for (_, k, _, _, r0), tr in zip(init, train)])
    raw_te = np.concatenate([np.broadcast_to(r0, (te.size, k)).ravel() for (_, k, _, _, r0), te in zip(init, test)] +
                            [np.zeros(0)])
    y_loc = np.ascontiguousarray(np.concatenate([ye for _, _, _, ye, _ in init]), dtype=np.int32)
    classes = np.zeros((P, 32), dtype=np.int32)
    for p, (c, _, _, _, _) in enumerate(init):
        classes[p, :c.size] = c.astype(np.int32)
    # the losses of the problems grouped by K: the gradient is row by row, so one call per group computes every problem's
    groups = {}
    for p, (_, k, loss, _, _) in enumerate(init):
        groups.setdefault(int(k), (loss, []))[1].append(p)
    rows_tr = np.arange(n_tr, dtype=np.int32)
    rows_te = np.arange(n_tr, n_tr + n_te, dtype=np.int32)
    lr = 0.1                                        # GradientBoostingClassifier's learning_rate
    with torch.cuda.device(X.device):
        d_Xs = torch.empty((n_tr + n_te, F), dtype=torch.float32, device=X.device)
        check(lib().b200aa_boosting_scale(ctypes.c_void_p(X.data_ptr()), n, F, P, _ptr(train_off), _ptr(train_idx),
                                          _ptr(test_off), _ptr(test_idx), ctypes.c_void_p(d_Xs.data_ptr()), _stream()))
        d_y = torch.from_numpy(y_loc).to(X.device)
        d_raw_tr = torch.from_numpy(np.ascontiguousarray(raw_tr, dtype=np.float64)).to(X.device)
        d_raw_te = torch.from_numpy(np.ascontiguousarray(raw_te, dtype=np.float64)).to(X.device)
        d_neg = torch.empty(max(int(g_off[-1]), 1), dtype=torch.float64, device=X.device)
        neg = np.zeros(max(int(g_off[-1]), 1))
        for s in range(int(stages.max())):
            active = (stages > s).astype(np.int32)
            raw = d_raw_tr.cpu().numpy()
            for k, (loss, probs) in groups.items():
                ps = [p for p in probs if active[p]]
                if not ps:
                    continue
                yk = np.concatenate([init[p][3] for p in ps])
                rk = np.concatenate([raw[g_off[p]:g_off[p + 1]].reshape(-1, k) for p in ps])
                gk = BO.neg_gradient(loss, yk, rk).ravel()
                o = 0
                for p in ps:
                    m = int(g_off[p + 1] - g_off[p])
                    neg[g_off[p]:g_off[p + 1]] = gk[o:o + m]
                    o += m
            d_neg.copy_(torch.from_numpy(neg))
            st_seeds = np.ascontiguousarray(np.concatenate([seeds[p][s * K[p]:(s + 1) * K[p]] for p in range(P) if active[p]]),
                                            dtype=np.uint32)
            status = lib().b200aa_boosting_stage(
                ctypes.c_void_p(d_Xs.data_ptr()), n_tr + n_te, F, P, _ptr(train_off), _ptr(rows_tr), _ptr(test_off),
                _ptr(rows_te), _ptr(K), _ptr(active), ctypes.c_void_p(d_y.data_ptr()), ctypes.c_void_p(d_neg.data_ptr()),
                ctypes.c_void_p(d_raw_tr.data_ptr()), ctypes.c_void_p(d_raw_te.data_ptr()), _ptr(st_seeds), lr,
                None, None, 0, None, None, _stream())
            _scratch_refusal(status, "boosting_cross_validate", "%d training rows" % max(t.size for t in train), F)
        pred = torch.empty(max(n_te, 1), dtype=torch.int32, device=X.device)
        counts = torch.empty((P, n_classes, n_classes), dtype=torch.int64, device=X.device)
        y_test = np.ascontiguousarray(y[test_idx] if n_te else np.zeros(1), dtype=np.int32)
        check(lib().b200aa_boosting_count(ctypes.c_void_p(d_raw_te.data_ptr()), P, _ptr(test_off), _ptr(K), _ptr(classes),
                                          _ptr(y_test), n_classes, ctypes.c_void_p(pred.data_ptr()),
                                          ctypes.c_void_p(counts.data_ptr()), _stream()))
    return pred[:n_te], counts


def tree_classify_batch(model, vectors):
    """predict / predict_proba of a tree ensemble for every row of a CUDA float32 / float64 [n, F] tensor, in one kernel on
    the current stream (DESIGN.md, kernel 8): CUDA (ids int64 [n], indices into the model's classes_; P float64 [n, C]),
    bit for bit scikit-learn's.  Gradient boosting's probabilities are its loss's link applied on the host to the raw
    scores the kernel adds.  A row scikit-learn refuses (inf, a float64 beyond float32, or NaN where the model takes none)
    raises scikit-learn's own ValueError.  `model`: a TreeEnsembleModel, or an estimator uploaded for this call."""
    _require_cuda(vectors, "vectors")
    if not isinstance(model, TreeEnsembleModel):
        model = TreeEnsembleModel(model, vectors.device)
    vectors, stride, dtype = _query_matrix(model, vectors)
    n = vectors.shape[0]
    with torch.cuda.device(vectors.device):
        ids = torch.empty(n, dtype=torch.int64, device=vectors.device)
        scores = torch.empty((n, model.n_classes), dtype=torch.float64, device=vectors.device)
        bad = torch.empty(n, dtype=torch.int32, device=vectors.device)
        if n:
            check(lib().b200aa_trees_classify(
                model.handle, ctypes.c_void_p(vectors.data_ptr()), dtype, n, model.n_feats, stride,
                ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(scores.data_ptr()), ctypes.c_void_p(bad.data_ptr()), _stream()))
            flagged = torch.nonzero(bad)
            if flagged.numel():
                row = vectors[int(flagged[0, 0])].reshape(1, -1).cpu().numpy()
                model.estimator.predict(row)                    # raises scikit-learn's ValueError for this row
                raise ValueError("row %d holds a value scikit-learn refuses" % int(flagged[0, 0]))
        if model.mode == TREE_FOREST:
            return ids, scores
        raw = scores.cpu().numpy()
        P = model.estimator._loss.predict_proba(raw[:, 0] if model.n_classes == 1 else raw)
        return ids, torch.from_numpy(np.ascontiguousarray(P, dtype=np.float64)).to(vectors.device)


def classify_vectors(classifier, model_type, vectors):
    """classifier_wrapper (audioTrainTest.py:52-93) over the rows of `vectors` [n x F]: (class ids [n], probabilities [n x classes]).
    A CUDA tensor goes to the kNN kernel (``knn_classify_batch``; `classifier` a KnnModel or a Knn-like object) or, for the
    three tree types, to the tree kernel when ``TreeEnsembleModel`` takes the model (``tree_classify_batch``), and only the
    results come back; other models and NumPy input run on the host.  A plain estimator is flattened and uploaded in every
    call (tens of ms for a 100-tree forest, DESIGN.md kernel 8); pass a TreeEnsembleModel to classify repeatedly."""
    if isinstance(vectors, torch.Tensor):
        if model_type == "knn" and vectors.is_cuda:
            ids, P = knn_classify_batch(classifier, vectors)
            return ids.cpu().numpy(), P.cpu().numpy()
        if model_type in _TREE_TYPES and vectors.is_cuda:
            model = classifier
            if not isinstance(model, TreeEnsembleModel):
                try:
                    model = TreeEnsembleModel(classifier, vectors.device)
                except ValueError:
                    model = None
            if model is not None:
                ids, P = tree_classify_batch(model, vectors)
                return model.classes[ids.cpu().numpy()], P.cpu().numpy()
        vectors = vectors.cpu().numpy()
    if isinstance(classifier, TreeEnsembleModel):
        classifier = classifier.estimator
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

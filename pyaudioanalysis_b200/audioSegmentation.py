"""HMM segmentation of the reference's audioSegmentation (audioSegmentation.py:102-193, :287-515, :606-678) without
hmmlearn: the training statistics and the diagonal-Gaussian Viterbi decode run on the GPU (kernel 7,
``consumers.hmm_statistics_batch`` / ``consumers.hmm_decode_batch``), bit for bit the reference's NumPy statistics and
GaussianHMM(C, "diag").predict restated in NumPy (DESIGN.md, kernel 7).

The reference's behaviour is kept where it is visible to a caller:
- the class order of ``segments_to_labels`` is ``list(set(labels))``, so it follows the process's string hash seed;
- a window in no segment takes the label of the last segment;
- ``train_hmm_from_directory`` takes the files in glob order, cuts each to min(windows, labels), uses each file's own
  class order as if it were global, counts transitions across file boundaries, and raises UnboundLocalError when the
  first file has no .segments file;
- ``hmm_segmentation`` and the trainers do not downmix: a stereo file raises the drop-in mid_feature_extraction's
  ValueError;
- the model files hold four pickles (model, class names, mid window, mid step).  The model is hmmlearn's GaussianHMM
  when hmmlearn imports, else ``DiagonalGaussianHMM`` with the same attribute names; loading accepts either.

``evaluate_segmentation_classification_dir`` decodes every file of the folder in one ragged batch and prints the
reference's text.  Its classifier methods need the reference's own function (``install.install_segmentation`` keeps
it); called here they raise ValueError.

Speaker diarization (:815-1091): ``diarize`` runs the steps after the mid-term features.  The SVM posteriors, k-means
and LDA stay on the host, as the reference makes them; the StandardScalers, the feature-outlier rule and the LDA branch's
pooling run on the GPU (kernel 11, ``consumers.standard_scale_batch`` / ``outlier_columns`` / ``pool_frames_batch``), the
silhouette's cluster distance means on kernel 9 (``consumers.cluster_distance_means``) and the HMM smoothing on kernel 7
(``hmm_statistics_batch`` and the float64 decode), all from one upload of the matrix.  The reference's visible quirks are
kept:
- the "outliers" dropped are feature columns (dist_all is the pdist of the columns of the normalised matrix);
- A[c] is the mean pdist over the transposed cluster, i.e. between its feature columns;
- the labels smoothed by the HMM and the median filter are those of the LAST candidate speaker count, not of the best;
- the speaker count reported (the class names, the plot) comes from the best silhouette.
"""
import csv
import glob
import os
import pickle
import warnings

import numpy as np

_CLASSIFIER_METHODS = ("svm", "svm_rbf", "knn", "randomforest", "gradientboosting", "extratrees")
_SHORT = 0.050                  # the trainers' and hmm_segmentation's short-term window and step (:374-375)


class DiagonalGaussianHMM:
    """A picklable diagonal GaussianHMM with hmmlearn's attribute names (startprob_ [C], transmat_ [C, C], means_ [C, F],
    covars_ [C, F] diagonal), written by the trainers when hmmlearn is not installed."""

    def __init__(self, n_components, covariance_type="diag"):
        self.n_components = n_components
        self.covariance_type = covariance_type


# ------------------------------------------------------------------ host helpers (:102-193, :495-515, :606-633)
def read_segmentation_gt(gt_file):
    """(start times, end times, labels) of the tab-separated rows of three fields in a segments file."""
    starts, ends, labels = [], [], []
    with open(gt_file, "rt") as f:
        for row in csv.reader(f, delimiter="\t"):
            if len(row) == 3:
                starts.append(float(row[0]))
                ends.append(float(row[1]))
                labels.append(row[2])
    return np.array(starts), np.array(ends), labels


def segments_to_labels(start_times, end_times, labels, window):
    """One class index per `window` seconds, probed at the window centres up to the last end time: (flags, class names),
    class names in ``list(set(labels))`` order.  A centre in no segment takes the last segment's label."""
    class_names = list(set(labels))
    flags = []
    t = window / 2.0
    while t < end_times[-1]:
        hit = len(start_times) - 1
        for i in range(len(start_times)):
            if start_times[i] < t <= end_times[i]:
                hit = i
                break
        flags.append(class_names.index(labels[hit]))
        t += window
    return np.array(flags), class_names


def compute_metrics(confusion_matrix, class_names):
    """(recall, precision, f1) per class of a confusion matrix."""
    recall, precision, f1 = [], [], []
    if len(class_names) != confusion_matrix.shape[0]:
        print("Error in computePreRec! Confusion matrix and class_names list must be of the same size!")
        return recall, precision, f1
    for i in range(len(class_names)):
        precision.append(confusion_matrix[i, i] / np.sum(confusion_matrix[:, i]))
        recall.append(confusion_matrix[i, i] / np.sum(confusion_matrix[i, :]))
        f1.append(2 * precision[-1] * recall[-1] / (precision[-1] + recall[-1]))
    return recall, precision, f1


def load_ground_truth_segments(gt_file, mt_step):
    seg_start, seg_end, seg_labels = read_segmentation_gt(gt_file)
    labels, class_names = segments_to_labels(seg_start, seg_end, seg_labels, mt_step)
    return np.array([class_names.index(class_names[k]) for k in labels]), class_names


def calculate_confusion_matrix(predictions, ground_truth, classes):
    """cm[truth, prediction] counts over the common length (a -1 prediction counts in the last column, as NumPy indexes)."""
    cm = np.zeros((len(classes), len(classes)))
    n = min(predictions.shape[0], ground_truth.shape[0])
    np.add.at(cm, (np.asarray(ground_truth[:n]).astype(np.int64), np.asarray(predictions[:n]).astype(np.int64)), 1)
    return cm


def segmentation_accuracy(flags_ind, flags_ind_gt):
    """The share of equal labels over the common length, -1 when it is empty (:187-192)."""
    n = min(flags_ind.shape[0], flags_ind_gt.shape[0])
    return np.sum(flags_ind[:n] == flags_ind_gt[:n]) / float(n) if n > 0 else -1


def _plot_segmentation(flags_ind, flags_ind_gt, class_names, mt_step, accuracy):
    """The per-class duration statistics and plots of plot_segmentation_results (:194-247): needs matplotlib."""
    try:
        import matplotlib.pyplot as plt
    except ImportError as exc:
        raise ImportError("plot_results=True needs matplotlib") from exc
    from .consumers import labels_to_segments
    segments, classes = labels_to_segments([class_names[int(f)] for f in flags_ind], mt_step)
    segments = np.asarray(segments, dtype=np.float64).reshape(-1, 2)
    duration = segments[-1, 1]
    totals = np.zeros(len(class_names))
    for (a, b), c in zip(segments, classes):
        totals[class_names.index(c)] += b - a
    percentages = 100.0 * totals / duration
    counts = np.array([sum(1 for c in classes if c == name) for name in class_names])
    av_durations = np.where(counts > 0, totals / np.maximum(counts, 1), 0.0)
    for i in range(len(class_names)):
        print(class_names[i], percentages[i], av_durations[i])
    fig = plt.figure()
    ax1 = fig.add_subplot(211)
    ax1.set_yticks(np.arange(len(class_names)))
    ax1.set_yticklabels(class_names)
    ax1.plot(np.arange(len(flags_ind)) * mt_step + mt_step / 2.0, flags_ind)
    if flags_ind_gt.shape[0] > 0:
        ax1.plot(np.arange(len(flags_ind_gt)) * mt_step + mt_step / 2.0, flags_ind_gt + 0.05, "--r")
    plt.xlabel("time (seconds)")
    if accuracy >= 0:
        plt.title("Accuracy = {0:.1f}%".format(100.0 * accuracy))
    print(np.arange(len(class_names)), percentages)
    fig.add_subplot(223).bar(np.arange(len(class_names)) + 0.5, percentages)
    fig.add_subplot(224).bar(np.arange(len(class_names)) + 0.5, av_durations)
    fig.tight_layout()
    plt.show()


def load_ground_truth(gt_file, labels, class_names, mid_step, plot_results):
    """(ground-truth labels, the model's class names, accuracy, confusion matrix) of predicted labels against a segments
    file; prints "Overall Accuracy".  Without the file: (empty, class names, 0, empty)."""
    accuracy, cm, labels_gt = 0, np.array([]), np.array([])
    if os.path.isfile(gt_file):
        labels_gt, class_names_gt = load_ground_truth_segments(gt_file, mid_step)
        mapped = np.array([class_names_gt.index(class_names[int(v)]) if class_names[int(v)] in class_names_gt else -1
                           for v in labels])
        cm = calculate_confusion_matrix(mapped, labels_gt, class_names_gt)
        accuracy = segmentation_accuracy(mapped, labels_gt)
        if plot_results:
            _plot_segmentation(mapped, labels_gt, class_names_gt, mid_step, accuracy)
        if accuracy >= 0:
            print("Overall Accuracy: {0:.2f}".format(accuracy))
    return labels_gt, class_names, accuracy, cm


# ------------------------------------------------------------------ training statistics (:287-344)
def _transitions(labels, C):
    """Transition counts indexed by int(label), row-normalised (a row without transitions is NaN)."""
    T = np.zeros((C, C))
    n = labels.shape[0]
    if n > 1:
        ints = [int(v) for v in labels]
        a = np.array(ints, dtype=np.int64)
        if a.min() < -C or a.max() >= C:
            for i in range(n - 1):                      # raises the reference's IndexError at the first bad label
                T[ints[i], ints[i + 1]] += 1
        np.add.at(T, (a[:-1], a[1:]), 1)
    for i in range(C):
        T[i, :] /= T[i, :].sum()
    return T


def _statistics(labels, n_columns, device_stats):
    """train_hmm_compute_statistics around a device call: device_stats(class windows) -> CUDA [4, C, F]."""
    labels = np.asarray(labels)
    unique = np.unique(labels)
    C = len(unique)
    if n_columns < labels.shape[0]:
        print("trainHMM warning: number of short-term feature vectors must be greater or equal to the labels length!")
        labels = labels[0:n_columns]
    priors = np.zeros((C,))
    for i, u in enumerate(unique):
        priors[i] = np.count_nonzero(labels == u)
    priors = priors / priors.sum()
    trans = _transitions(labels, C)
    if C == 0:
        return priors, trans, np.zeros((0, 0)), np.zeros((0, 0))
    out = device_stats([np.nonzero(labels == u)[0] for u in unique]).cpu().numpy()
    return priors, trans, out[1], out[3]


def train_hmm_compute_statistics(features, labels):
    """(class priors [C], transition matrix [C, C], means [C, F], std [C, F]) of a feature matrix [F x n] and its window
    labels, bit for bit the reference's; the means and standard deviations are computed on the GPU."""
    import torch
    from .consumers import hmm_statistics_batch
    features = np.asarray(features)
    mid = torch.from_numpy(np.ascontiguousarray(features, dtype=np.float64)).cuda().unsqueeze(0)
    return _statistics(labels, features.shape[1], lambda windows: hmm_statistics_batch(mid, windows))


def _new_model(priors, trans, means, cov):
    try:
        import hmmlearn.hmm
        hmm = hmmlearn.hmm.GaussianHMM(priors.shape[0], "diag")
    except ImportError:
        hmm = DiagonalGaussianHMM(priors.shape[0], "diag")
    hmm.covars_ = cov
    hmm.means_ = means
    hmm.startprob_ = priors
    hmm.transmat_ = trans
    return hmm


def save_hmm(hmm_model_name, model, classes, mid_window, mid_step):
    """The reference's model file: four pickles (model, class names, mid window, mid step)."""
    with open(hmm_model_name, "wb") as f:
        for obj in (model, classes, mid_window, mid_step):
            pickle.dump(obj, f, protocol=pickle.HIGHEST_PROTOCOL)


def _load_hmm(hmm_model_name):
    with open(hmm_model_name, "rb") as f:
        return tuple(pickle.load(f) for _ in range(4))


# ------------------------------------------------------------------ mid-term features on the device
def _mid_batch(paths, mid_window, mid_step):
    """The mid-term matrices of files as the trainers and hmm_segmentation compute them (mid_feature_extraction with
    short window = step = round(fs * 0.050), no downmix), on the device, in ragged batches of one (rate, format).
    Returns (mid CUDA float32 [n, 136, M], the n files that mid_feature_extraction accepts in order, zero past each
    one's windows; their window counts [n]; errors {file index: exception} for the files it would refuse (stereo, no
    frames, a zero step); slot [len(paths)], each file's row of mid or None).  Each batch's features are copied into mid
    and released before the next batch runs."""
    import torch
    from . import _lib, audioio
    from .MidTermFeatures import _Clip, _plan_chunks
    from .ShortTermFeatures import _as_clip, _fs_int, _raise_no_frames
    from .batch import mid_feature_extraction_batch, mid_ratios
    L = _lib.lib()
    clips, counts, slot, errors = [], [], [None] * len(paths), {}
    for i, path in enumerate(paths):
        try:
            fs, x = audioio.read_audio_file(path)
            data, code = _as_clip(x)
            fs = _fs_int(fs)
            w = round(fs * _SHORT)
            T = L.b200aa_num_frames(data.shape[0], w, w)
            if T <= 0:
                _raise_no_frames(fs, w)
            stepr = mid_ratios(mid_window * fs, mid_step * fs, w, w)[1]
            if stepr < 1:
                raise ValueError("mid-term step shorter than half a short-term step")
        except Exception as exc:        # raised again at the file's turn, after the output of the files before it
            errors[i] = exc
            continue
        slot[i] = len(clips)
        clips.append(_Clip(path, fs, data.shape[0], data, code))
        counts.append(int(L.b200aa_mid_windows(T, stepr)))
    out = torch.zeros((len(clips), 136, max(counts, default=1)), dtype=torch.float32, device="cuda")
    for part in _plan_chunks(clips):
        chunk = [clips[k] for k in part]
        fs = chunk[0].fs
        w = round(fs * _SHORT)
        dev, lengths = audioio.stage(chunk)
        mid, _ = mid_feature_extraction_batch(dev, fs, mid_window * fs, mid_step * fs, w, w, lengths=lengths)
        for j, k in enumerate(part):
            out[k, :, :counts[k]] = mid[j, :, :counts[k]]
        del dev, mid
    return out, counts, errors, slot


def _decode_mids(mid, hmm, n_windows=None):
    """Labels (int64 [n]) of each clip of a CUDA float32 [B, F, M] batch; ValueError for non-finite features."""
    from .consumers import HmmModel, hmm_decode_batch
    model = HmmModel(hmm, mid.device)
    ids, bad = hmm_decode_batch(mid, model, n_windows)
    ids, bad = ids.cpu().numpy(), bad.cpu().numpy()
    counts = [mid.shape[2]] * mid.shape[0] if n_windows is None else list(n_windows)
    return [None if bad[b] else ids[b, :counts[b]].astype(np.int64) for b in range(mid.shape[0])]


def _nonfinite():
    return ValueError("Input X contains NaN, infinity or a value too large for dtype('float64').")


# ------------------------------------------------------------------ trainers and decode (:347-492)
def train_hmm_from_file(wav_file, gt_file, hmm_model_name, mid_window, mid_step):
    """Train an HMM from one annotated file and save it; returns (hmm, class names)."""
    from .consumers import hmm_statistics_batch
    seg_start, seg_end, seg_labs = read_segmentation_gt(gt_file)
    flags, class_names = segments_to_labels(seg_start, seg_end, seg_labs, mid_step)
    mid, counts, errors, _ = _mid_batch([wav_file], mid_window, mid_step)
    if errors:
        raise errors[0]
    priors, trans, means, cov = _statistics(flags, counts[0],
                                            lambda windows: hmm_statistics_batch(mid, windows, n_windows=counts))
    hmm = _new_model(priors, trans, means, cov)
    save_hmm(hmm_model_name, hmm, class_names, mid_window, mid_step)
    return hmm, class_names


def _unbound_f_all():
    return UnboundLocalError("cannot access local variable 'f_all' where it is not associated with a value")


def train_hmm_from_directory(folder_path, hmm_model_name, mid_window, mid_step):
    """Train an HMM from the .wav / .segments pairs of a folder and save it; returns (hmm, class names of all files).
    Every file's features are computed in shared ragged launches and the statistics in one call.  As in the reference,
    the first file in glob order must have a .segments file: otherwise the next annotated file (after its features), or
    the statistics when there is none, raise UnboundLocalError."""
    from .consumers import hmm_statistics_batch
    files = glob.glob(folder_path + os.sep + "*.wav")
    labelled, flag_lists, class_names_all = [], [], []
    for f in files:
        gt_file = f.replace(".wav", ".segments")
        if os.path.isfile(gt_file):
            flags, class_names = segments_to_labels(*read_segmentation_gt(gt_file), mid_step)
            for c in class_names:
                if c not in class_names_all:
                    class_names_all.append(c)
            labelled.append(f)
            flag_lists.append(flags)
    mid, counts, errors, _ = _mid_batch(labelled, mid_window, mid_step)
    first_labelled = bool(files) and bool(labelled) and labelled[0] == files[0]
    for k in range(len(labelled)):
        if k in errors:
            raise errors[k]
        if not first_labelled:
            raise _unbound_f_all()
    if not labelled:
        raise _unbound_f_all()
    used = [min(n, len(fl)) for n, fl in zip(counts, flag_lists)]
    flags_all = np.array([])
    for fl, n in zip(flag_lists, used):
        flags_all = np.append(flags_all, np.array([int(v) for v in fl[:n]]))
    priors, trans, means, cov = _statistics(flags_all, sum(used),
                                            lambda windows: hmm_statistics_batch(mid, windows, n_windows=used))
    hmm = _new_model(priors, trans, means, cov)
    save_hmm(hmm_model_name, hmm, class_names_all, mid_window, mid_step)
    return hmm, class_names_all


def hmm_segmentation(audio_file, hmm_model_name, plot_results=False, gt_file=""):
    """Decode a file with a saved HMM: (labels [M], class names, accuracy, confusion matrix), the accuracy and matrix
    against gt_file when it exists."""
    hmm, class_names, mid_window, mid_step = _load_hmm(hmm_model_name)
    mid, counts, errors, _ = _mid_batch([audio_file], mid_window, mid_step)
    if errors:
        raise errors[0]
    labels = _decode_mids(mid, hmm, counts)[0]
    if labels is None:
        raise _nonfinite()
    _, class_names, accuracy, cm = load_ground_truth(gt_file, labels, class_names, mid_step, plot_results)
    return labels, class_names, accuracy, cm


def evaluate_segmentation_classification_dir(dir_name, model_name, method_name):
    """Decode every .wav file of a folder with an HMM model file and print the reference's per-file and summary text.
    All files are decoded in one ragged batch before the first line is printed."""
    if method_name.lower() in _CLASSIFIER_METHODS:
        raise ValueError("method %r: only HMM segmentation runs here (install.install_segmentation keeps the "
                         "reference's function for the classifier methods)" % (method_name,))
    files = glob.glob(dir_name + os.sep + "*.wav")
    labels_of = {}
    if files:
        hmm, model_classes, mid_window, mid_step = _load_hmm(model_name)
        mid, counts, errors, slot = _mid_batch(files, mid_window, mid_step)
        decoded = _decode_mids(mid, hmm, counts) if mid.shape[0] else []
        for i in range(len(files)):
            labels_of[i] = errors[i] if i in errors else (decoded[slot[i]] if decoded[slot[i]] is not None else _nonfinite())
    accuracies, class_names, cm_total = [], [], np.array([])
    for index, wav_file in enumerate(files):
        print(wav_file)
        if isinstance(labels_of[index], Exception):
            raise labels_of[index]
        gt_file = wav_file.replace(".wav", ".segments")
        _, class_names, accuracy, cm_temp = load_ground_truth(gt_file, labels_of[index], model_classes, mid_step, False)
        if accuracy > 0:
            cm_total = np.copy(cm_temp) if not index else cm_total + cm_temp
            accuracies.append(accuracy)
            print(cm_temp, class_names)
            print(cm_total)
    if len(cm_total.shape) > 1:
        cm_total = cm_total / np.sum(cm_total)
        rec, pre, f1 = compute_metrics(cm_total, class_names)
        print(" - - - - - - - - - - - - - - - - - - - - - - - - - - - - - - ")
        print("Average Accuracy: {0:.1f}".format(100.0 * np.array(accuracies).mean()))
        print("Average recall: {0:.1f}".format(100.0 * np.array(rec).mean()))
        print("Average precision: {0:.1f}".format(100.0 * np.array(pre).mean()))
        print("Average f1: {0:.1f}".format(100.0 * np.array(f1).mean()))
        print("Median Accuracy: {0:.1f}".format(100.0 * np.median(np.array(accuracies))))
        print("Min Accuracy: {0:.1f}".format(100.0 * np.array(accuracies).min()))
        print("Max Accuracy: {0:.1f}".format(100.0 * np.array(accuracies).max()))
    else:
        print("Confusion matrix was empty, accuracy for every file was 0")


def dispatcher(original):
    """An evaluate_segmentation_classification_dir that runs the HMM method here and the classifier methods through
    `original`."""
    def evaluate_segmentation_classification_dir_dispatch(dir_name, model_name, method_name):
        run = original if method_name.lower() in _CLASSIFIER_METHODS else evaluate_segmentation_classification_dir
        return run(dir_name, model_name, method_name)
    evaluate_segmentation_classification_dir_dispatch.original = original
    return evaluate_segmentation_classification_dir_dispatch


# ------------------------------------------------------------------ speaker diarization (:251-284, :815-1091)
_DIARIZATION_MODELS = ("svm_rbf_speaker_10", "svm_rbf_speaker_male_female")


def evaluate_speaker_diarization(labels, labels_gt):
    """(cluster purity, speaker purity) of window labels against ground-truth labels over their common length."""
    n = min(labels.shape[0], labels_gt.shape[0])
    labels, labels_gt = labels[0:n], labels_gt[0:n]
    flags, flags_gt = np.unique(labels), np.unique(labels_gt)
    table = np.zeros((flags.shape[0], flags_gt.shape[0]))
    np.add.at(table, (np.searchsorted(flags, labels), np.searchsorted(flags_gt, labels_gt)), 1.0)
    row_sum, column_sum, total = np.sum(table, axis=0), np.sum(table, axis=1), np.sum(table)
    purity_clust = np.array([np.max(table[i, :]) / column_sum[i] for i in range(table.shape[0])])
    purity_speak = np.array([np.max(table[:, j]) / row_sum[j] for j in range(table.shape[1])])
    return np.sum(purity_clust * column_sum) / total, np.sum(purity_speak * row_sum) / total


def _posteriors(vectors, model):
    """predict_proba of an SVM (classifier, mean, std) for the rows of `vectors`, normalised as the reference does per
    window: one batched call, row-wise as the per-window loop."""
    classifier, mean, std = model
    return np.asarray(classifier.predict_proba((vectors - mean) / std))


def _with_posteriors(feats, posteriors):
    """[feats; p1 + 1e-4; p2 + 1e-4] (rows: features, columns: windows) as float64."""
    return np.concatenate([np.asarray(feats, dtype=np.float64)] + [np.asarray(p, dtype=np.float64).T + 1e-4
                                                                    for p in posteriors])


def pool_frames(st, ratio):
    """The LDA branch's pooling (:884-906): for every short-term frame i, the mean and population std of each feature row
    over frames [i, min(i + ratio, T)), as [2F, T] float64 (means, then stds).  Each row's statistics are NumPy's of the
    contiguous slice, as the reference's per-row loop takes them (np.mean / np.std along a row reduce it in the same
    order as the 1-D slice)."""
    st = np.ascontiguousarray(st, dtype=np.float64)
    F, T = st.shape
    out = np.zeros((2 * F, T))
    for i in range(T):
        w = st[:, i:min(i + ratio, T)]
        out[:F, i] = np.mean(w, axis=1)
        out[F:, i] = np.std(w, axis=1)
    return out


def _kmeans(x, k):
    import sklearn.cluster
    k_means = sklearn.cluster.KMeans(n_clusters=k)
    k_means.fit(x)
    return k_means.labels_


def _silhouette(cls, k, A, B):
    """The average silhouette of :949-985 from the cluster distance means (A [k], B [k, k], NumPy arrays)."""
    sil_1, sil_2 = [], []
    for c in range(k):
        share = np.nonzero(cls == c)[0].shape[0] / float(len(cls))
        if share < 0.020:
            sil_1.append(0.0)
            sil_2.append(0.0)
        else:
            sil_1.append(A[c] * share)
            sil_temp = []
            for c2 in range(k):
                if c2 != c:
                    share_2 = np.nonzero(cls == c2)[0].shape[0] / float(len(cls))
                    sil_temp.append(B[c, c2] * (share + share_2) / 2.0)
            sil_2.append(min(np.array(sil_temp)))
    sil_1, sil_2 = np.array(sil_1), np.array(sil_2)
    sil = [(sil_2[c] - sil_1[c]) / (max(sil_2[c], sil_1[c]) + 1e-5) for c in range(k)]
    return np.mean(sil)


def cluster_means_gpu(x, cls, k, rows):
    """(A, B) of kernel 9 for one clustering, as NumPy arrays.  x: a CUDA float64 tensor (or host data, uploaded for this
    call).  Every mean of no terms (pdist of fewer than two columns, cdist against an empty cluster) warns as np.mean of
    an empty array does, in the reference's order, under the caller's np.errstate."""
    import torch
    from .consumers import cluster_distance_means
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()
    A, B = cluster_distance_means(t, cls, k, rows)
    A, B = A.cpu().numpy(), B.cpu().numpy()
    counts = np.bincount(np.asarray(cls, dtype=np.int64), minlength=k)
    for c in sorted(rows):
        if t.shape[1] < 2:
            np.mean(np.empty(0))
        for c2 in range(k):
            if c2 != c and counts[c] * counts[c2] == 0:
                np.mean(np.empty(0))
    return A, B


def _hmm_smooth(x, cls):
    """The HMM post-processing of :1001-1010 for the normalised matrix x [M, D] (a CUDA float64 tensor, or host data,
    uploaded here): statistics of x.T per label, then predict(x) of the C-contiguous x on the GPU (kernel 7, float64
    windows)."""
    import torch
    from .consumers import HmmModel, hmm_decode_batch, hmm_statistics_batch
    if not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()
    features = x.t().contiguous().unsqueeze(0)
    start_prob, transmat, means, cov = _statistics(cls, x.shape[0], lambda windows: hmm_statistics_batch(features, windows))
    hmm = DiagonalGaussianHMM(start_prob.shape[0], "diag")
    hmm.startprob_, hmm.transmat_, hmm.means_, hmm.covars_ = start_prob, transmat, means, cov
    t = x.contiguous()
    ids, bad = hmm_decode_batch(t.unsqueeze(0).transpose(1, 2), HmmModel(hmm, t.device))
    if bool(bad[0]):
        raise _nonfinite()
    return ids[0].cpu().numpy().astype(np.int64)


def diarize(mid, models, n_speakers, mid_step, short_window, lda_dim, st=None, mid_window=None, posteriors=None,
            cluster=None, means=None, details=False):
    """The steps of speaker_diarization after the mid-term features (:848-1012) for a mid-term matrix mid [F, M]:
    returns cls [M] (float64, the median-filtered labels), or with ``details`` (cls, a dict of the intermediate arrays:
    posteriors, i_non_outliers, labels per candidate count, sil_all, num_speakers).

    models: the two (classifier, mean, std) SVM triples (svm_rbf_speaker_10, svm_rbf_speaker_male_female); posteriors:
    their predict_proba matrices [M, C] instead.  lda_dim > 0 needs models (even with posteriors given: the posteriors of
    the pooled short-term frames are computed here), st (the short-term features [68, T]) and mid_window: every
    short-term frame is pooled as the reference pools it (``pool_frames``) and projected by LDA, and there is no HMM.  cluster(x, k) -> labels
    (default: sklearn.cluster.KMeans(n_clusters=k), seeded by the global NumPy state as in the reference); means(x, cls,
    k, rows) -> (A, B) (default: kernel 9)."""
    import torch
    from scipy.signal import medfilt
    from .consumers import outlier_columns, pool_frames_batch, standard_scale_batch
    cluster = _kmeans if cluster is None else cluster
    means = cluster_means_gpu if means is None else means
    mid = np.asarray(mid, dtype=np.float64)
    if lda_dim > 0 and (models is None or st is None or mid_window is None):
        raise ValueError("lda_dim > 0 needs models (the posteriors of every short-term frame are computed here), st "
                         "and mid_window")
    if posteriors is None:
        posteriors = [_posteriors(mid.T, m) for m in models]
    feats = _with_posteriors(mid, posteriors)
    on_device = means is cluster_means_gpu          # a caller's own host means keeps the matrix on the host
    if on_device:
        # StandardScaler().fit_transform(feats.T) of the C-contiguous [D, M] feats: a column-major [M, D] on the device
        norm_dev = standard_scale_batch(torch.from_numpy(feats).cuda().t())[0]
        i_non_outliers = outlier_columns(norm_dev)[0]
        mt_feats_norm_or = norm_dev.t().cpu().numpy().T
    else:
        from scipy.spatial import distance
        from sklearn.preprocessing import StandardScaler
        mt_feats_norm_or = StandardScaler().fit_transform(feats.T)
        dist_all = np.sum(distance.squareform(distance.pdist(mt_feats_norm_or.T)), axis=0)
        i_non_outliers = np.nonzero(dist_all < 1.1 * np.mean(dist_all))[0]
        norm_dev = None
    mid_feats_norm = mt_feats_norm_or[:, i_non_outliers]
    if lda_dim > 0:
        import sklearn.discriminant_analysis
        ratio = int(round(mid_window / short_window))
        if on_device:
            st = np.asarray(st)
            st_dev = torch.from_numpy(np.ascontiguousarray(st, dtype=np.float32 if st.dtype == np.float32 else np.float64))
            pooled_dev = pool_frames_batch(st_dev.cuda(), ratio)
            pooled = pooled_dev.cpu().numpy()
            post = _with_posteriors(np.zeros((0, pooled.shape[1])), [_posteriors(pooled.T, m) for m in models])
            red_dev = torch.cat([pooled_dev, torch.from_numpy(post).to(pooled_dev.device)])
            red = standard_scale_batch(red_dev.t())[0].t().cpu().numpy()
        else:
            from sklearn.preprocessing import StandardScaler
            pooled = pool_frames(st, ratio)
            red = _with_posteriors(pooled, [_posteriors(pooled.T, m) for m in models])
            red = StandardScaler().fit_transform(red.T).T
        labels = np.zeros((red.shape[1],))
        lda_step_ratio = 1.0 / short_window
        for index in range(labels.shape[0]):
            labels[index] = int(index * short_window / lda_step_ratio)
        clf = sklearn.discriminant_analysis.LinearDiscriminantAnalysis(n_components=lda_dim)
        mid_feats_norm = clf.fit_transform(red.T, labels)
    s_range = range(2, 10) if n_speakers <= 0 else [n_speakers]
    x = mid_feats_norm
    if on_device and lda_dim <= 0:                  # the device copy, for every candidate count
        x = norm_dev[:, torch.from_numpy(i_non_outliers).to(norm_dev.device)].contiguous()
    elif on_device:
        x = torch.from_numpy(np.ascontiguousarray(mid_feats_norm, dtype=np.float64)).cuda()
    cluster_labels, sil_all = [], []
    cls = None
    for speakers in s_range:
        cls = cluster(mid_feats_norm, speakers)
        cluster_labels.append(cls)
        shares = np.bincount(np.asarray(cls, dtype=np.int64), minlength=speakers) / float(len(cls))
        rows = [c for c in range(speakers) if not shares[c] < 0.020]
        A, B = means(x, cls, speakers, rows)
        sil_all.append(_silhouette(cls, speakers, A, B))
    imax = int(np.argmax(sil_all))
    num_speakers = s_range[imax]
    if lda_dim <= 0:
        cls = _hmm_smooth(mt_feats_norm_or if norm_dev is None else norm_dev, cls)
    cls = medfilt(cls, 5)
    if not details:
        return cls
    return cls, {"posteriors": posteriors, "i_non_outliers": i_non_outliers, "labels": cluster_labels,
                 "sil_all": np.array(sil_all), "num_speakers": num_speakers}


def _load_svm(path):
    """(classifier, mean, std, class names) of a model file pair written by the reference's trainer."""
    with open(path + "MEANS", "rb") as fo:
        mean, std, class_names = pickle.load(fo), pickle.load(fo), pickle.load(fo)
    with open(path, "rb") as fid:
        classifier = pickle.load(fid)
    return classifier, np.array(mean), np.array(std), class_names


def _models_dir(models_dir):
    if models_dir is None:
        try:
            import pyAudioAnalysis
            models_dir = os.path.join(os.path.dirname(os.path.realpath(pyAudioAnalysis.__file__)), "data", "models")
        except ImportError:
            models_dir = None
    paths = None if models_dir is None else [os.path.join(models_dir, m) for m in _DIARIZATION_MODELS]
    if paths is None or not all(os.path.isfile(p) and os.path.isfile(p + "MEANS") for p in paths):
        raise FileNotFoundError("speaker_diarization needs the SVM models %s and %s (with their MEANS files) in "
                                "pyAudioAnalysis/data/models or models_dir" % _DIARIZATION_MODELS)
    return paths


def _diarization_features(filename, mid_window, mid_step):
    """(mid [136, M], st [68, T], duration) of a file as speaker_diarization computes them (:828-846): the file read,
    downmixed, and its mid-term features on the GPU (the drop-in mid_feature_extraction) at a 50 ms short-term window
    and step."""
    from . import audioio
    from .MidTermFeatures import mid_feature_extraction
    sampling_rate, signal = audioio.read_audio_file(filename)
    signal = audioio.stereo_to_mono(signal)
    duration = len(signal) / sampling_rate
    mid, st, _ = mid_feature_extraction(signal, sampling_rate, mid_window * sampling_rate, mid_step * sampling_rate,
                                        round(sampling_rate * 0.05), round(sampling_rate * 0.05))
    return mid, st, duration


def speaker_diarization(filename, n_speakers, mid_window=1.0, mid_step=0.1, short_window=0.1, lda_dim=0, plot_res=False,
                        models_dir=None):
    """The reference's speaker_diarization: (cls, cluster purity, speaker purity), the purities -1 without a .segments
    file next to the WAV; prints them as the reference does.  Mid-term features on the GPU (the drop-in
    mid_feature_extraction), then ``diarize``."""
    paths = _models_dir(models_dir)
    loaded = [_load_svm(p) for p in paths]
    mid_feats, st_feats, duration = _diarization_features(filename, mid_window, mid_step)
    return _diarize_file(filename, [m[:3] for m in loaded], mid_feats, st_feats, duration, n_speakers, mid_window,
                         mid_step, short_window, lda_dim, plot_res)


def _diarize_file(filename, models, mid_feats, st_feats, duration, n_speakers, mid_window, mid_step, short_window, lda_dim,
                  plot_res):
    """speaker_diarization after the features: diarize, the ground-truth lookup, the printed purities and the plot."""
    cls, info = diarize(mid_feats, models, n_speakers, mid_step, short_window, lda_dim, st=st_feats,
                        mid_window=mid_window, details=True)
    num_speakers = info["num_speakers"]
    class_names = ["speaker{0:d}".format(c) for c in range(num_speakers)]
    gt_file = filename.replace(".wav", ".segments")
    flags_gt = None
    if os.path.isfile(gt_file):
        seg_start, seg_end, seg_labs = read_segmentation_gt(gt_file)
        flags_gt, _ = segments_to_labels(seg_start, seg_end, seg_labs, mid_step)
    plt = None
    if plot_res:
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            plt = None
    if plt is not None:
        fig = plt.figure()
        ax1 = fig.add_subplot(111) if n_speakers > 0 else fig.add_subplot(211)
        ax1.set_yticks(np.array(range(len(class_names))))
        ax1.axis((0, duration, -1, len(class_names)))
        ax1.set_yticklabels(class_names)
        ax1.plot(np.array(range(len(cls))) * mid_step + mid_step / 2.0, cls)
    purity_cluster_m, purity_speaker_m = -1, -1
    if flags_gt is not None:
        if plt is not None:
            ax1.plot(np.array(range(len(flags_gt))) * mid_step + mid_step / 2.0, flags_gt, "r")
        purity_cluster_m, purity_speaker_m = evaluate_speaker_diarization(cls, flags_gt)
        print("{0:.1f}\t{1:.1f}".format(100 * purity_cluster_m, 100 * purity_speaker_m))
        if plt is not None:
            plt.title("Cluster purity: {0:.1f}% - Speaker purity: {1:.1f}%".format(100 * purity_cluster_m,
                                                                                   100 * purity_speaker_m))
    if plt is not None:
        plt.xlabel("time (seconds)")
        if n_speakers <= 0:
            plt.subplot(212)
            plt.plot(list(range(2, 10)), info["sil_all"])
            plt.xlabel("number of clusters")
            plt.ylabel("average clustering's sillouette")
        plt.show()
    return cls, purity_cluster_m, purity_speaker_m


def speaker_diarization_evaluation(folder_name, lda_dimensions, models_dir=None):
    """Print the cluster and speaker purity of every WAV file of a folder with a .segments file, for each LDA dimension,
    as the reference does by calling speaker_diarization(wav, n, 2.0, 0.2, 0.05, dim) per file; the speaker count of each
    file comes from its ground truth (-1 without one).  Each file is read, downmixed and its features computed once, at
    its first turn, and reused for every LDA dimension."""
    wav_files = sorted(glob.glob(os.path.join(folder_name, "*.wav")))
    num_speakers = []
    for wav_file in wav_files:
        gt_file = wav_file.replace(".wav", ".segments")
        if os.path.isfile(gt_file):
            _, _, seg_labs = read_segmentation_gt(gt_file)
            num_speakers.append(len(list(set(seg_labs))))
        else:
            num_speakers.append(-1)
    models, features = None, {}
    for dim in lda_dimensions:
        print("LDA = {0:d}".format(dim))
        for i, wav_file in enumerate(wav_files):
            if models is None:
                models = [_load_svm(p)[:3] for p in _models_dir(models_dir)]
            if i not in features:
                features[i] = _diarization_features(wav_file, 2.0, 0.2)
            mid, st, duration = features[i]
            _diarize_file(wav_file, models, mid, st, duration, num_speakers[i], 2.0, 0.2, 0.05, dim, False)


def standardise(st_feats):
    """StandardScaler().fit_transform(st_feats.T) (audioSegmentation.py:51-52) on the host, as a C-contiguous float64
    [T, F] matrix of one frame per row: the rows self_similarity_matrix compares."""
    from sklearn.preprocessing import StandardScaler
    return np.ascontiguousarray(StandardScaler().fit_transform(np.asarray(st_feats).T), dtype=np.float64)


def _standardise_device(st_feats):
    """``standardise`` on the GPU (kernel 11): StandardScaler().fit_transform(st_feats.T) of the float64 features,
    as a CUDA C-contiguous float64 [T, F] matrix, bit for bit."""
    import torch
    from .consumers import standard_scale_batch
    st = torch.from_numpy(np.ascontiguousarray(st_feats, dtype=np.float64)).cuda()
    return standard_scale_batch(st.t())[0].contiguous()


def self_similarity_matrix(feature_vectors):
    """The reference's self_similarity_matrix (:40-55): the scaler and the cosine similarities on the GPU (kernels 11 and
    10, ``consumers.standard_scale_batch`` and ``consumers.self_similarity_batch``), bit for bit.  Returns a NumPy float64
    [n_vectors, n_vectors]."""
    from .consumers import self_similarity_batch
    X = _standardise_device(feature_vectors)
    return self_similarity_batch(X, [X.shape[0]])[0].cpu().numpy()


def music_thumbnailing(signal, sampling_rate, short_window=1.0, short_step=0.5, thumb_size=10.0, limit_1=0, limit_2=1):
    """The reference's music_thumbnailing (:1093-1180): (A1, A2, B1, B2, the masked filtered matrix), the times NumPy
    float64 as the reference returns them.  The signal is downmixed, its short-term features come from the drop-in
    feature_extraction, the scaler runs on the GPU (kernel 11), and the similarity matrix, diagonal filter, masks, argmax
    and walk on kernel 10 (``consumers.thumbnail_batch``), bit for bit the reference's steps on the same features."""
    from .audioio import stereo_to_mono
    from .consumers import thumbnail_batch
    from .ShortTermFeatures import feature_extraction
    signal = stereo_to_mono(signal)
    st_feats, _ = feature_extraction(signal, sampling_rate, sampling_rate * short_window, sampling_rate * short_step)
    X = _standardise_device(st_feats)
    idx, C = thumbnail_batch(X, [X.shape[0]], int(round(thumb_size / short_step)),
                             5.0 / short_step, limit_1, limit_2)
    i1, i2, j1, j2 = idx[0]
    return short_step * i1, short_step * i2, short_step * j1, short_step * j2, C[0].cpu().numpy()

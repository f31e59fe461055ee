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
"""
import csv
import glob
import os
import pickle

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

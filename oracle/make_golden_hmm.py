"""Golden HMM-segmentation results of the UNMODIFIED reference (run where the reference tree exists):

    python -m oracle.make_golden_hmm

The reference's audioSegmentation imports hmmlearn and matplotlib at module level, so its functions are executed from
its source text (as in make_golden_knn.py) with:
- hmmlearn replaced by a recorder: the trainers only construct GaussianHMM and assign attributes to it;
- `set` replaced by an insertion-ordered set, so that the class order, which follows the string hash seed in the
  reference, is the same in every run (the tests put the same ordered set into the port);
- glob returning sorted paths, and, for the directory trainer and the folder evaluation, mid_feature_extraction and
  hmm_segmentation replaced by stubs that return stored matrices and stored predicted labels.

Writes tests/golden/hmm.npz:
- seg_cases: for each, <c>_text (a .segments file), <c>_step, and the reference's read_segmentation_gt
  (<c>_start / _end / _labels), segments_to_labels as class names per window (<c>_flags), and
  load_ground_truth_segments as class names (<c>_gt);
- stat_cases: <c>_features [F, M] float64, <c>_labels, and train_hmm_compute_statistics' <c>_priors / _trans / _means /
  _cov, its stdout (<c>_stdout) and the name of the exception it raised ('' for none: <c>_error).  scottish and
  diarizationExample use the reference's own mid_feature_extraction at a 1.0 s mid step;
- dir_cases: <c>_names (file names), <c>_texts (their .segments, '' for none), <c>_matrices (the stub's float32-valued
  matrices, concatenated along the windows, <c>_cols per file), and train_hmm_from_directory's class names, statistics
  and exception name;
- eval_cases: <c>_names, <c>_texts, <c>_pred (predicted labels, concatenated, <c>_lens per file), <c>_classes (the
  model's class names), <c>_step, and the stdout of evaluate_segmentation_classification_dir(..., "hmm") with the folder
  written as "<dir>".
"""
import contextlib
import csv
import io
import os
import pickle
import tempfile
import types
import warnings

import numpy as np
from scipy.io import wavfile

from oracle.ref_import import REFERENCE_ROOT, load_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "hmm.npz")
REF = os.path.join(REFERENCE_ROOT, "pyAudioAnalysis")


def ordered_set(items):
    """An insertion-ordered stand-in for set(): list() of it gives the items in first-appearance order."""
    return dict.fromkeys(items).keys()


class Recorder:
    """hmmlearn.hmm.GaussianHMM as the trainers use it: constructed, then assigned attributes."""

    def __init__(self, n_components, covariance_type):
        self.n_components, self.covariance_type = n_components, covariance_type


def _exec_between(path, start, stop, env):
    src = open(path).read()
    a = src.index(start)
    b = src.index(stop, a)
    exec(src[a:b], env)
    return env


def reference_env():
    import glob as glob_mod
    env = {"np": np, "os": os, "csv": csv, "cpickle": pickle, "set": ordered_set, "plt": None,
           "glob": types.SimpleNamespace(glob=lambda p: sorted(glob_mod.glob(p))),
           "hmmlearn": types.SimpleNamespace(hmm=types.SimpleNamespace(GaussianHMM=Recorder))}
    path = os.path.join(REF, "audioSegmentation.py")
    for start, stop in (("def labels_to_segments", "def evaluate_speaker_diarization"),
                        ("def train_hmm_compute_statistics", "def train_hmm_from_file"),
                        ("def train_hmm_from_directory", "def hmm_segmentation"),
                        ("def load_ground_truth_segments", "def mid_term_file_classification"),
                        ("def load_ground_truth(", "def silence_removal")):
        _exec_between(path, start, stop, env)
    return env


def run(fn, *args):
    """(result, stdout, exception class name or '')."""
    out = io.StringIO()
    with contextlib.redirect_stdout(out), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return fn(*args), out.getvalue(), ""
        except Exception as exc:
            return None, out.getvalue(), type(exc).__name__


def main():
    _, M, _ = load_reference()
    R = reference_env()
    rng = np.random.default_rng(20261017)
    g = {}
    tmp = tempfile.mkdtemp()

    def write(name, text):
        path = os.path.join(tmp, name)
        with open(path, "w") as f:
            f.write(text)
        return path

    # ---- segments files: the reference's two, and gaps / overlaps / a bad row
    seg_cases = []
    texts = {"scottish": open(os.path.join(REF, "data", "scottish.segments")).read(),
             "diarization": open(os.path.join(REF, "data", "diarizationExample.segments")).read(),
             "gaps": "0.0\t2.0\tspeech\n2.5\t4.0\tmusic\nnot a row\n3.5\t6.2\tspeech\n7.0\t9.0\tnoise\n"}
    for name, text in texts.items():
        path = write(name + ".segments", text)
        for step in (1.0, 0.3):
            c = "%s_%g" % (name, step)
            start, end, labels = R["read_segmentation_gt"](path)
            flags, names = R["segments_to_labels"](start, end, labels, step)
            gt, gt_names = R["load_ground_truth_segments"](path, step)
            g.update({c + "_text": text, c + "_step": step, c + "_start": start, c + "_end": end, c + "_labels": np.array(labels),
                      c + "_flags": np.array([names[k] for k in flags]), c + "_gt": np.array([gt_names[k] for k in gt])})
            seg_cases.append(c)
    g["seg_cases"] = np.array(seg_cases)

    # ---- statistics: the reference's own matrices of its two files, and seeded edge cases
    stat_cases = []

    def stats(c, feats, labels):
        res, out, err = run(R["train_hmm_compute_statistics"], feats, labels)
        g.update({c + "_features": feats, c + "_labels": np.asarray(labels, dtype=np.float64), c + "_stdout": out,
                  c + "_error": err})
        if res is not None:
            g.update({c + "_priors": res[0], c + "_trans": res[1], c + "_means": res[2], c + "_cov": res[3]})
        stat_cases.append(c)
        print(c, feats.shape, err or "ok")

    for name, wav in (("scottish", "scottish.wav"), ("diarization", "diarizationExample.wav")):
        fs, x = wavfile.read(os.path.join(REF, "data", wav))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            feats = np.asarray(M.mid_feature_extraction(x, fs, 1.0 * fs, 1.0 * fs, round(fs * 0.050), round(fs * 0.050))[0],
                               dtype=np.float64)
        start, end, labels = R["read_segmentation_gt"](os.path.join(REF, "data", wav.replace(".wav", ".segments")))
        flags, _ = R["segments_to_labels"](start, end, labels, 1.0)
        stats("real_" + name, feats, flags)
    # seeded cases: 136 rows once, 12 rows for the rest (the golden file stays small)
    F = 136
    wide = rng.normal(size=(F, 60)) * rng.choice([1e-3, 1.0, 1e3], size=(F, 1))
    wide[5] = 2.75                                       # a constant feature: std 0
    stats("constant_row", wide, rng.integers(0, 3, size=60).astype(np.float64))
    base = rng.normal(size=(12, 300)) * rng.choice([1e-3, 1.0, 1e3], size=(12, 1))
    lab = rng.integers(0, 3, size=300).astype(np.float64)
    one = lab.copy()
    one[17] = 3.0
    stats("one_window", base, one)
    nan = lab.copy()
    nan[-1] = 3.0                                        # class 3 has no outgoing transition: a NaN row
    stats("nan_row", base, nan)
    stats("label_ge_c", base[:, :40], np.where(lab == 1, 2.0, lab)[:40])
    stats("truncated", base[:, :250], lab)
    stats("one_feature", base[:1], lab)
    g["stat_cases"] = np.array(stat_cases)

    # ---- the directory trainer, features stubbed
    dir_cases = []

    def directory(c, files):
        d = tempfile.mkdtemp(dir=tmp)
        mats = {}
        for fname, text, cols in files:
            open(os.path.join(d, fname), "wb").close()
            if text:
                with open(os.path.join(d, fname.replace(".wav", ".segments")), "w") as f:
                    f.write(text)
            mats[fname] = (rng.normal(size=(F, cols)) * 10).astype(np.float32).astype(np.float64)
        R["audioBasicIO"] = types.SimpleNamespace(read_audio_file=lambda p: (16000, os.path.basename(p)))
        R["mtf"] = types.SimpleNamespace(mid_feature_extraction=lambda sig, *a: (mats[sig], None, None))
        res, out, err = run(R["train_hmm_from_directory"], d, os.path.join(d, "model"), 1.0, 1.0)
        names = [f[0] for f in files]
        g.update({c + "_names": np.array(names), c + "_texts": np.array([f[1] for f in files]),
                  c + "_cols": np.array([f[2] for f in files]),
                  c + "_matrices": np.concatenate([mats[n] for n in names], axis=1), c + "_error": err})
        if res is not None:
            hmm, classes = res
            g.update({c + "_classes": np.array(classes), c + "_priors": hmm.startprob_, c + "_trans": hmm.transmat_,
                      c + "_means": hmm.means_, c + "_cov": hmm.covars_})
        dir_cases.append(c)
        print(c, err or "ok")

    t1 = "0\t5\tspeech\n5\t9\tmusic\n9\t14\tspeech\n"
    t2 = "0\t3\tnoise\n3\t8\tspeech\n"
    t3 = "0\t4\tmusic\n4\t6\tnoise\n6\t12\tmusic\n"
    directory("dir_mixed", [("a.wav", t1, 12), ("b.wav", t2, 10), ("c.wav", "", 7), ("d.wav", t3, 14)])
    directory("dir_first_unlabelled", [("a.wav", "", 5), ("b.wav", t1, 12)])
    g["dir_cases"] = np.array(dir_cases)

    # ---- the folder evaluation, hmm_segmentation stubbed with stored predictions
    eval_cases = []

    def evaluation(c, files, classes, step):
        d = tempfile.mkdtemp(dir=tmp)
        pred = {}
        for fname, text, p in files:
            open(os.path.join(d, fname), "wb").close()
            if text:
                with open(os.path.join(d, fname.replace(".wav", ".segments")), "w") as f:
                    f.write(text)
            pred[os.path.join(d, fname)] = np.asarray(p, dtype=np.int64)

        def hmm_segmentation(wav, model, plot, gt):
            labels = pred[wav]
            _, names, acc, cm = R["load_ground_truth"](gt, labels, classes, step, plot)
            return labels, names, acc, cm
        R["hmm_segmentation"] = hmm_segmentation
        _, out, err = run(R["evaluate_segmentation_classification_dir"], d, "model", "hmm")
        assert not err, err
        g.update({c + "_names": np.array([f[0] for f in files]), c + "_texts": np.array([f[1] for f in files]),
                  c + "_pred": np.concatenate([np.asarray(f[2], dtype=np.int64) for f in files]),
                  c + "_lens": np.array([len(f[2]) for f in files]), c + "_classes": np.array(classes), c + "_step": step,
                  c + "_stdout": out.replace(d, "<dir>")})
        eval_cases.append(c)
        print(c, len(out.splitlines()), "lines")

    classes = ["speech", "music", "noise", "silence"]
    tA = "0\t5\tspeech\n5\t9\tmusic\n9\t14\tnoise\n"
    tB = "0\t3\tnoise\n3\t8\tspeech\n8\t11\tmusic\n"
    evaluation("eval_mixed", [("a.wav", tA, rng.integers(0, 3, size=14)), ("b.wav", tB, rng.integers(0, 4, size=9)),
                              ("c.wav", "", rng.integers(0, 3, size=6)), ("d.wav", tA, [0] * 5 + [1] * 4 + [2] * 6)],
               classes, 1.0)
    evaluation("eval_empty", [("a.wav", "0\t4\tspeech\n", [3] * 4), ("b.wav", "", [0, 1])], classes, 1.0)
    g["eval_cases"] = np.array(eval_cases)

    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()

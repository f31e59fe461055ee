"""CPU: the host side of audioSegmentation against the reference's own code (tests/golden/hmm.npz,
oracle/make_golden_hmm.py): the segments helpers, the priors / transitions / printed warnings / exceptions of
train_hmm_compute_statistics, the directory trainer's UnboundLocalError, the whole stdout of
evaluate_segmentation_classification_dir with the predictions given, and install_segmentation / uninstall.  The class
order of ``list(set(...))`` follows the hash seed, so the golden was made, and these tests run, with an insertion-ordered
set in its place."""
import contextlib
import glob as glob_mod
import io
import types

import numpy as np
import pytest
import torch

from tests.conftest import load_golden
from pyaudioanalysis_b200 import audioSegmentation as S


def _ordered_set(items):
    return dict.fromkeys(items).keys()


@pytest.fixture
def ordered(monkeypatch):
    monkeypatch.setattr(S, "set", _ordered_set, raising=False)
    monkeypatch.setattr(S, "glob", types.SimpleNamespace(glob=lambda p: sorted(glob_mod.glob(p))))


def test_segments_helpers(tmp_path):
    g = load_golden("hmm.npz")
    for c in g["seg_cases"]:
        path = tmp_path / (c + ".segments")
        path.write_text(str(g[c + "_text"]))
        step = float(g[c + "_step"])
        start, end, labels = S.read_segmentation_gt(str(path))
        assert np.array_equal(start, g[c + "_start"]) and np.array_equal(end, g[c + "_end"]), c
        assert labels == [str(x) for x in g[c + "_labels"]], c
        flags, names = S.segments_to_labels(start, end, labels, step)
        assert [names[k] for k in flags] == [str(x) for x in g[c + "_flags"]], c
        gt, gt_names = S.load_ground_truth_segments(str(path), step)
        assert [gt_names[k] for k in gt] == [str(x) for x in g[c + "_gt"]], c


def test_statistics_host_side():
    """Priors, transitions, the truncation warning and the exceptions; the means / std come from the GPU (tested there)."""
    g = load_golden("hmm.npz")
    for c in g["stat_cases"]:
        feats = g[c + "_features"]
        out, err = io.StringIO(), ""
        with contextlib.redirect_stdout(out), np.errstate(all="ignore"):
            try:
                res = S._statistics(g[c + "_labels"], feats.shape[1],
                                    lambda windows: torch.zeros((4, len(windows), feats.shape[0]), dtype=torch.float64))
            except Exception as exc:
                err = type(exc).__name__
        assert err == str(g[c + "_error"]), c
        assert out.getvalue() == str(g[c + "_stdout"]), c
        if not err:
            assert np.array_equal(res[0], g[c + "_priors"]), c
            assert np.array_equal(res[1], g[c + "_trans"], equal_nan=True), c


def test_directory_first_file_unlabelled(tmp_path, monkeypatch, ordered):
    g = load_golden("hmm.npz")
    c = "dir_first_unlabelled"
    assert str(g[c + "_error"]) == "UnboundLocalError"
    for name, text in zip(g[c + "_names"], g[c + "_texts"]):
        (tmp_path / str(name)).write_bytes(b"")
        if str(text):
            (tmp_path / str(name).replace(".wav", ".segments")).write_text(str(text))
    monkeypatch.setattr(S, "_mid_batch", lambda paths, mw, ms: (None, [10] * len(paths), {}, list(range(len(paths)))))
    with pytest.raises(UnboundLocalError):
        S.train_hmm_from_directory(str(tmp_path), str(tmp_path / "model"), 1.0, 1.0)


def test_evaluation_stdout(tmp_path, monkeypatch, ordered):
    """Every line the reference prints, the summary and the "Confusion matrix was empty" branch included."""
    g = load_golden("hmm.npz")
    for c in g["eval_cases"]:
        d = tmp_path / c
        d.mkdir()
        names = [str(n) for n in g[c + "_names"]]
        for name, text in zip(names, g[c + "_texts"]):
            (d / name).write_bytes(b"")
            if str(text):
                (d / name.replace(".wav", ".segments")).write_text(str(text))
        cuts = np.concatenate([[0], np.cumsum(g[c + "_lens"])])
        preds = [g[c + "_pred"][cuts[k]:cuts[k + 1]] for k in range(len(names))]
        classes = [str(x) for x in g[c + "_classes"]]
        step = float(g[c + "_step"])
        monkeypatch.setattr(S, "_load_hmm", lambda name: (None, classes, 1.0, step))
        monkeypatch.setattr(S, "_mid_batch", lambda paths, mw, ms: (np.zeros((len(paths), 1, 1)), [len(p) for p in preds], {},
                                                                    list(range(len(paths)))))
        monkeypatch.setattr(S, "_decode_mids", lambda mid, hmm, counts: [p.copy() for p in preds])
        out = io.StringIO()
        with contextlib.redirect_stdout(out), np.errstate(all="ignore"):
            S.evaluate_segmentation_classification_dir(str(d), "model", "hmm")
        assert out.getvalue().replace(str(d), "<dir>") == str(g[c + "_stdout"]), c


def test_install_segmentation_and_uninstall():
    import importlib
    install = importlib.import_module("pyaudioanalysis_b200.install")
    names = ("train_hmm_compute_statistics", "train_hmm_from_file", "train_hmm_from_directory", "hmm_segmentation",
             "evaluate_segmentation_classification_dir")
    calls = []
    originals = {n: (lambda n: lambda *a: calls.append((n, a)))(n) for n in names}
    mod = types.ModuleType("pyAudioAnalysis.audioSegmentation")
    for n, f in originals.items():
        setattr(mod, n, f)
    try:
        done = install.install_segmentation(mod)
        assert sorted(done) == sorted("pyAudioAnalysis.audioSegmentation." + n for n in names)
        for n in names[:4]:
            assert getattr(mod, n) is getattr(S, n)
        mod.evaluate_segmentation_classification_dir("dir", "model", "SVM_rbf")      # a classifier method: the original
        assert calls == [("evaluate_segmentation_classification_dir", ("dir", "model", "SVM_rbf"))]
        assert mod.evaluate_segmentation_classification_dir.original is originals[names[4]]
    finally:
        install.uninstall()
    for n in names:
        assert getattr(mod, n) is originals[n]

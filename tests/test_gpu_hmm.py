"""GPU: kernel 7 (b200aa_hmm_statistics / b200aa_hmm_decode, consumers.hmm_statistics_batch / hmm_decode_batch) bit for bit
against NumPy's statistics and tests/hmm_oracle.py's decode, over ragged batches, scratch slices, streams and threads; and
the drop-in audioSegmentation end to end on generated WAV + .segments folders against the restated reference pipeline fed
by the drop-in's own mid-term matrices."""
import contextlib
import io
import os
import threading
import types

import numpy as np
import pytest

from tests import hmm_oracle as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import consumers
    return consumers


def _hmm(rng, n_states, F, zeros=False):
    start = rng.random(n_states) + 0.05
    trans = rng.random((n_states, n_states)) + 0.05
    if zeros and n_states > 1:
        start[0] = 0.0
        trans[rng.random((n_states, n_states)) < 0.3] = 0.0
        trans[np.arange(n_states), np.arange(n_states)] = 1.0
    return types.SimpleNamespace(startprob_=start / start.sum(), transmat_=trans / trans.sum(axis=1, keepdims=True),
                                 means_=rng.normal(size=(n_states, F)), covars_=rng.random((n_states, F)) + 0.3)


def _batch(rng, counts, F, M, poison=True):
    import torch
    x = rng.normal(size=(len(counts), F, M)).astype(np.float32)
    if poison:
        for b, n in enumerate(counts):
            x[b, :, n:] = np.nan
    return x, torch.from_numpy(x).cuda()


def _oracle(x, n, hmm, chunk=None):
    """The restated predict of a clip's first n windows; asserts that no exact tie decided the path."""
    path, ties = H.predict(x[:, :n].astype(np.float64), hmm.startprob_, hmm.transmat_, hmm.means_, hmm.covars_, ties=True,
                           chunk=chunk)
    assert ties == 0, "an exact tie decided the path: draw another seed"
    return path


def _decode(C, t, hmm, counts):
    import torch
    ids, bad = C.hmm_decode_batch(t, hmm, counts)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), bad.cpu().numpy()


@pytest.mark.parametrize("n_states", [1, 2, 3, 10, 31, 32, 33, 64])
def test_decode_matches_oracle(C, n_states):
    rng = np.random.default_rng(100 + n_states)
    F = 136
    counts = [1, 2, 33, 4097]
    x, t = _batch(rng, counts, F, 4097)
    for zeros in (False, True):
        hmm = _hmm(rng, n_states, F, zeros)
        ids, bad = _decode(C, t, hmm, counts)
        assert not bad.any()
        for b, n in enumerate(counts):
            assert np.array_equal(ids[b, :n], _oracle(x[b], n, hmm)), (n_states, n, zeros)
            assert not ids[b, n:].any()


@pytest.mark.parametrize("n_states", [1, 2, 3, 10, 31, 32, 33, 64])
def test_decode_one_hour(C, n_states):
    """36 000 windows (an hour at a 0.1 s step), every state count."""
    rng = np.random.default_rng(700 + n_states)
    x, t = _batch(rng, [36000], 136, 36000)
    hmm = _hmm(rng, n_states, 136, zeros=True)
    ids, _ = _decode(C, t, hmm, None)
    assert np.array_equal(ids[0], _oracle(x[0], 36000, hmm, chunk=4000))


def test_decode_across_scratch_slices(C):
    """64 states x 12 B per (window, state): 9 clips of 40 000 windows need 276 MB of scratch, so two slices."""
    rng = np.random.default_rng(8)
    counts = [40000, 39000, 40000, 1, 40000, 12345, 40000, 40000, 39999]
    x, t = _batch(rng, counts, 8, 40000)
    hmm = _hmm(rng, 64, 8)
    ids, bad = _decode(C, t, hmm, counts)
    assert not bad.any()
    for b, n in enumerate(counts):
        assert np.array_equal(ids[b, :n], _oracle(x[b], n, hmm)), b
        assert not ids[b, n:].any()


def test_nonfinite_clip_refused(C):
    rng = np.random.default_rng(9)
    counts = [50, 40, 30]
    x, t = _batch(rng, counts, 6, 50)
    t[1, 2, 17] = float("inf")
    hmm = _hmm(rng, 4, 6)
    model = C.HmmModel(hmm)
    got, bad = C.hmm_decode_batch(t, model, counts)
    assert bad.cpu().numpy().tolist() == [False, True, False]
    ids = got.cpu().numpy()
    assert not ids[1].any()                                          # nothing written for the refused clip
    for b in (0, 2):
        assert np.array_equal(ids[b, :counts[b]], _oracle(x[b], counts[b], hmm))


def test_model_checks(C):
    rng = np.random.default_rng(10)
    base = _hmm(rng, 3, 4)
    for attr, value, text in (("startprob_", np.array([0.5, 0.2, 0.2]), "startprob_"),
                              ("transmat_", np.array([[0.5, 0.5, 0.0], [0.0, 0.0, 0.0], [0.2, 0.3, 0.5]]), "transmat_"),
                              ("covars_", np.where(np.arange(12).reshape(3, 4) == 5, 0.0, 1.0), "covars")):
        hmm = types.SimpleNamespace(**vars(base))
        setattr(hmm, attr, value)
        with pytest.raises(ValueError, match=text):
            C.HmmModel(hmm)


def test_statistics_match_numpy(C):
    import torch
    rng = np.random.default_rng(11)
    counts = [300, 0, 77, 512]
    F, M = 136, 512
    x = rng.normal(size=(4, F, M)).astype(np.float32) * rng.choice([1e-3, 1.0, 1e3], size=(1, F, 1)).astype(np.float32)
    cat = np.concatenate([x[b, :, :n] for b, n in enumerate(counts)], axis=1).astype(np.float64)
    labels = rng.integers(0, 5, size=cat.shape[1])
    labels[7] = 4
    windows = [np.nonzero(labels == u)[0] for u in range(5)]
    windows.append(np.array([3]))                                    # a one-window class: std 0
    for dt in (torch.float32, torch.float64):
        t = torch.from_numpy(x).cuda().to(dt)
        out = C.hmm_statistics_batch(t, windows, counts).cpu().numpy()
        for c, idx in enumerate(windows):
            assert np.array_equal(out[1, c], cat[:, idx].mean(axis=1)), (dt, c)
            assert np.array_equal(out[3, c], np.std(cat[:, idx], axis=1)), (dt, c)


def test_train_hmm_compute_statistics_matches_numpy():
    from pyaudioanalysis_b200 import audioSegmentation as S
    rng = np.random.default_rng(12)
    for F in (136, 1):
        feats = rng.normal(size=(F, 900))
        labels = rng.integers(0, 4, size=905).astype(np.float64)     # longer than the matrix: truncated, with the warning
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            pri, tr, mu, sd = S.train_hmm_compute_statistics(feats, labels)
        assert "trainHMM warning" in buf.getvalue()
        lab = labels[:900]
        for i, u in enumerate(np.unique(labels)):
            idx = np.nonzero(lab == u)[0]
            assert np.array_equal(mu[i], feats[:, idx].mean(axis=1))
            assert np.array_equal(sd[i], np.std(feats[:, idx], axis=1))
            assert pri[i] == np.count_nonzero(lab == u) / 900.0


def test_side_stream_and_threads(C):
    import torch
    rng = np.random.default_rng(13)
    counts = [700, 650, 20]
    x, t = _batch(rng, counts, 136, 700)
    hmm = _hmm(rng, 7, 136)
    model = C.HmmModel(hmm)
    want = [_oracle(x[b], n, hmm) for b, n in enumerate(counts)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ids, _ = C.hmm_decode_batch(t, model, counts)
    s.synchronize()
    for b, n in enumerate(counts):
        assert np.array_equal(ids[b, :n].cpu().numpy(), want[b])
    errors = []

    def work():
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(3):
                    got, _ = C.hmm_decode_batch(t, model, counts)
                    torch.cuda.current_stream().synchronize()
                    for b, n in enumerate(counts):
                        assert np.array_equal(got[b, :n].cpu().numpy(), want[b])
        except Exception as exc:                                     # reported by the main thread
            errors.append(exc)
    th = [threading.Thread(target=work) for _ in range(2)]
    for h in th:
        h.start()
    for h in th:
        h.join()
    assert not errors, errors


# ------------------------------------------------------------------ end to end
def _write_folder(root, n_files, seed, fs=16000, unannotated=True):
    """WAV files with .segments files: tones per class in seconds-long segments, every class in every annotated file (the
    reference adds the files' confusion matrices, so their class sets must agree).  With `unannotated`, one file that is
    not the first in glob order has no .segments file (the reference's trainer needs the first one annotated)."""
    import glob
    from tests import wavgen
    rng = np.random.default_rng(seed)
    names = ["speech", "music", "noise"]
    os.makedirs(root, exist_ok=True)
    for k in range(n_files):
        dur = int(rng.integers(12, 20))
        t = np.arange(dur * fs) / fs
        x = np.zeros(dur * fs)
        rows, a = [], 0.0
        order = rng.permutation(3)
        while a < dur:
            b = min(dur, a + float(rng.integers(2, 5)))
            c = int(order[len(rows) % 3])
            sl = (t >= a) & (t < b)
            x[sl] = [np.sin(2 * np.pi * 220 * t[sl]), np.sign(np.sin(2 * np.pi * 1000 * t[sl])) * 0.5,
                     rng.normal(scale=0.3, size=sl.sum())][c]
            rows.append("%.1f\t%.1f\t%s" % (a, b, names[c]))
            a = b
        x = np.clip(np.round(x * 12000 + rng.normal(scale=200, size=x.size)), -32768, 32767).astype(np.int64)
        wavgen.write(os.path.join(root, "f%02d.wav" % k), fs, x, "s16")
        with open(os.path.join(root, "f%02d.segments" % k), "w") as f:
            f.write("\n".join(rows) + "\n")
    if unannotated:
        os.remove(glob.glob(root + os.sep + "*.wav")[-1].replace(".wav", ".segments"))


def _restated_labels(S, path, hmm, mid_window, mid_step):
    from pyaudioanalysis_b200 import MidTermFeatures, audioio
    fs, x = audioio.read_audio_file(path)
    feats = MidTermFeatures.mid_feature_extraction(x, fs, mid_window * fs, mid_step * fs, round(fs * 0.05), round(fs * 0.05))[0]
    return feats, H.predict(feats, hmm.startprob_, hmm.transmat_, hmm.means_, hmm.covars_)


def test_folder_end_to_end(tmp_path):
    import glob
    from pyaudioanalysis_b200 import MidTermFeatures, audioio
    from pyaudioanalysis_b200 import audioSegmentation as S
    root = str(tmp_path / "data")
    _write_folder(root, 6, 21)
    model = str(tmp_path / "hmm")
    hmm, names = S.train_hmm_from_directory(root, model, 1.0, 0.5)
    # restated trainer fed by the drop-in's own matrices
    f_all, flags_all, names_all = None, np.array([]), []
    for i, f in enumerate(glob.glob(root + os.sep + "*.wav")):
        gt = f.replace(".wav", ".segments")
        if not os.path.isfile(gt):
            continue
        flags, cn = S.segments_to_labels(*S.read_segmentation_gt(gt), 0.5)
        names_all += [c for c in cn if c not in names_all]
        fs, x = audioio.read_audio_file(f)
        fv = MidTermFeatures.mid_feature_extraction(x, fs, 1.0 * fs, 0.5 * fs, round(fs * 0.05), round(fs * 0.05))[0]
        m = min(fv.shape[1], len(flags))
        flags_all = np.append(flags_all, np.array(flags[:m]))
        f_all = fv[:, :m] if f_all is None else np.concatenate((f_all, fv[:, :m]), axis=1)
    assert names == names_all
    lab = flags_all
    for i, u in enumerate(np.unique(lab)):
        idx = np.nonzero(lab == u)[0]
        assert np.array_equal(hmm.means_[i], f_all[:, idx].mean(axis=1))
        assert np.array_equal(hmm.covars_[i], np.std(f_all[:, idx], axis=1))
    files = glob.glob(root + os.sep + "*.wav")
    labels, cn, acc, cm = S.hmm_segmentation(files[0], model, gt_file=files[0].replace(".wav", ".segments"))
    feats, want = _restated_labels(S, files[0], hmm, 1.0, 0.5)
    assert np.array_equal(labels, want)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        S.evaluate_segmentation_classification_dir(root, model, "hmm")
    ref = io.StringIO()
    with contextlib.redirect_stdout(ref):                                # the loop of :636-678, file by file
        accs, cm_total = [], np.array([])
        for index, f in enumerate(files):
            print(f)
            _, want = _restated_labels(S, f, hmm, 1.0, 0.5)
            _, cn, a, c = S.load_ground_truth(f.replace(".wav", ".segments"), want, names, 0.5, False)
            if a > 0:
                cm_total = np.copy(c) if not index else cm_total + c
                accs.append(a)
                print(c, cn)
                print(cm_total)
        print("Average Accuracy: {0:.1f}".format(100.0 * np.array(accs).mean()))
    got = buf.getvalue()
    assert got.startswith(ref.getvalue().rsplit("Average Accuracy", 1)[0])
    assert ref.getvalue().splitlines()[-1] in got


def test_stereo_and_other_methods(tmp_path):
    from tests import wavgen
    from pyaudioanalysis_b200 import audioSegmentation as S
    root = str(tmp_path / "d")
    _write_folder(root, 2, 5, unannotated=False)
    model = str(tmp_path / "m")
    S.train_hmm_from_directory(root, model, 1.0, 1.0)
    st = str(tmp_path / "stereo.wav")
    wavgen.write(st, 16000, wavgen.signal("s16", 2, 32000, 1), "s16")
    with pytest.raises(ValueError, match="one-dimensional"):
        S.hmm_segmentation(st, model)
    with pytest.raises(ValueError):
        S.evaluate_segmentation_classification_dir(root, model, "svm")
    empty = tmp_path / "e"
    empty.mkdir()
    (empty / "a.wav").write_bytes(open(os.path.join(root, "f00.wav"), "rb").read())
    with pytest.raises(UnboundLocalError):
        S.train_hmm_from_directory(str(empty), model, 1.0, 1.0)


# ------------------------------------------------------------------ against the reference's own results (tests/golden/hmm.npz)
def test_golden_statistics():
    """train_hmm_compute_statistics on the reference's matrices of scottish.wav / diarizationExample.wav and the seeded
    edge cases: priors, transitions, means, std, stdout and exceptions equal the reference's."""
    from tests.conftest import load_golden
    from pyaudioanalysis_b200 import audioSegmentation as S
    g = load_golden("hmm.npz")
    for c in g["stat_cases"]:
        out = io.StringIO()
        err = ""
        with contextlib.redirect_stdout(out), np.errstate(all="ignore"):
            try:
                res = S.train_hmm_compute_statistics(g[c + "_features"], g[c + "_labels"])
            except Exception as exc:
                err = type(exc).__name__
        assert err == str(g[c + "_error"]), c
        assert out.getvalue() == str(g[c + "_stdout"]), c
        if not err:
            for got, key in zip(res, ("_priors", "_trans", "_means", "_cov")):
                assert np.array_equal(got, g[c + key], equal_nan=True), (c, key)


def test_golden_directory_trainer(tmp_path, monkeypatch):
    """train_hmm_from_directory on the reference's stubbed folder: the stored matrices stand in for the features."""
    import glob as glob_mod
    import torch
    from tests.conftest import load_golden
    from pyaudioanalysis_b200 import audioSegmentation as S
    g = load_golden("hmm.npz")
    c = "dir_mixed"
    names, texts, cols = [str(n) for n in g[c + "_names"]], [str(t) for t in g[c + "_texts"]], list(g[c + "_cols"])
    for name, text in zip(names, texts):
        (tmp_path / name).write_bytes(b"")
        if text:
            (tmp_path / name.replace(".wav", ".segments")).write_text(text)
    starts = np.concatenate([[0], np.cumsum(cols)])
    mats = {n: g[c + "_matrices"][:, starts[k]:starts[k + 1]] for k, n in enumerate(names)}

    def mid_batch(paths, mid_window, mid_step):
        m = [mats[os.path.basename(p)] for p in paths]
        out = np.zeros((len(m), 136, max(x.shape[1] for x in m)), dtype=np.float32)
        for k, x in enumerate(m):
            out[k, :, :x.shape[1]] = x
        return torch.from_numpy(out).cuda(), [x.shape[1] for x in m], {}, list(range(len(m)))
    monkeypatch.setattr(S, "set", lambda items: dict.fromkeys(items).keys(), raising=False)
    monkeypatch.setattr(S, "glob", types.SimpleNamespace(glob=lambda p: sorted(glob_mod.glob(p))))
    monkeypatch.setattr(S, "_mid_batch", mid_batch)
    hmm, classes = S.train_hmm_from_directory(str(tmp_path), str(tmp_path / "model"), 1.0, 1.0)
    assert classes == [str(n) for n in g[c + "_classes"]]
    for attr, key in (("startprob_", "_priors"), ("transmat_", "_trans"), ("means_", "_means"), ("covars_", "_cov")):
        assert np.array_equal(getattr(hmm, attr), g[c + key], equal_nan=True), key

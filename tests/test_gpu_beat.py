"""GPU: beat extraction (kernel 4, batch.beat_extraction_batch) equals the host MidTermFeatures.beat_extraction bit for bit
on the same float32 values, NaN matching NaN -- golden matrices, ragged feature batches, pulse clips, poisoned padding,
0 / 1 / 2 frames, 40 000 clips, one hour of frames, every histogram size from 1 bin to more bins than frames -- and the
directory and file-classification paths that use it."""
import ctypes
import os
import types
import warnings
import wave

import numpy as np
import pytest

from oracle.make_golden_r2 import pulse_clip
from tests.conftest import load_golden
from tests.signals import bank

pytestmark = pytest.mark.gpu

WINDOWS = (0.05, 0.025, 0.1, 0.8, 1.5, 0.0005)      # 0.8: round(2.5) ties to 2; 1.5: one bin; 0.0005: 4000 bins


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


def _host(st, frames, window):
    """Host beat_extraction of every clip of a float32 [B, F, T] array on its first frames[b] columns."""
    from pyaudioanalysis_b200.MidTermFeatures import beat_extraction
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                 # mean of an empty slice, 0 / 0 for a clip of no frames
        return np.array([beat_extraction(st[b, :, :frames[b]].astype(np.float64), window) for b in range(st.shape[0])])


def _assert_same(got, ref, what):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, what
    same = (got.view(np.int64) == ref.view(np.int64)) | (np.isnan(got) & np.isnan(ref))
    bad = np.argwhere(~same)
    assert bad.size == 0, "%s: %d mismatches, first %s: got %r want %r" % (what, len(bad), bad[0], got[tuple(bad[0])], ref[tuple(bad[0])])


def _device_beat(P, st, window, frames=None):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(st, dtype=np.float32)).cuda()
    fr = None if frames is None else torch.as_tensor(np.asarray(frames, dtype=np.int64)).cuda()
    out = P.beat_extraction_batch(d, window, fr)
    assert out.dtype == torch.float64 and tuple(out.shape) == (st.shape[0], 2)
    return out.cpu().numpy()


def _check(P, st, windows, frames=None, what=""):
    st = np.asarray(st, dtype=np.float32)
    fr = [st.shape[2]] * st.shape[0] if frames is None else list(frames)
    for w in windows:
        _assert_same(_device_beat(P, st, w, frames), _host(st, fr, w), "%s window %g" % (what, w))


def test_golden_matrices(P):
    g = load_golden("beat.npz")
    for i in range(int(g["n"])):
        st = np.asarray(g["st_%d" % i], dtype=np.float32)[None]
        _check(P, st, (float(g["win_%d" % i]),) + WINDOWS, what="golden %d" % i)


def test_signal_bank_ragged(P):
    """Features of the adversarial bank as one ragged batch; columns past each clip's frame count are whatever the padded
    batch left there, and n_frames keeps the kernel off them."""
    from tests.kernels import ragged
    lib = P._lib.lib()
    clips = list(bank(16000, 800, 400).values())
    for deltas in (True, False):
        d, lens = ragged(clips, np.int16)
        st = P.feature_extraction_batch(d, 16000, 800, 400, deltas=deltas, lengths=lens).cpu().numpy()
        frames = [lib.b200aa_num_frames(x.size, 800, 400) for x in clips]
        assert st.shape[1] == (68 if deltas else 34)
        _check(P, st, WINDOWS, frames, "bank F=%d" % st.shape[1])


def test_pulse_clips(P):
    import torch
    fs = 16000
    x = np.stack([pulse_clip(50 + i, 10 * fs, fs, bpm) for i, bpm in enumerate((120, 90, 140, 75))])
    st = P.feature_extraction_batch(torch.from_numpy(x).cuda(), fs, 800, 400).cpu().numpy()
    _check(P, st, WINDOWS, what="pulse")
    st = P.feature_extraction_batch(torch.from_numpy(x).cuda(), fs, 400, 200).cpu().numpy()
    _check(P, st, (0.0125,), what="pulse 25/12.5 ms")


def test_stride_past_frames_is_never_read(P):
    """t_stride > T: the padding is NaN and +-inf; the result equals the unpadded clip's."""
    import torch
    from pyaudioanalysis_b200._lib import check, lib
    rng = np.random.default_rng(4)
    T = 300
    base = np.cumsum(rng.standard_normal((3, 68, T)), axis=2).astype(np.float32)
    pad = np.full((3, 68, T + 37), np.nan, dtype=np.float32)
    pad[..., T + 1::2] = np.inf
    pad[..., :T] = base
    frames = [T, 211, 2]
    for b, n in enumerate(frames):
        pad[b, :, n:] = np.nan
    _check(P, pad, WINDOWS, frames, "NaN padding")
    # the C ABI's own n_frames < t_stride (no per-clip counts)
    out = torch.empty((3, 2), dtype=torch.float64, device="cuda")
    pad[...] = np.nan
    pad[..., :T] = base
    d = torch.from_numpy(pad).cuda()
    check(lib().b200aa_beat_extraction(ctypes.c_void_p(d.data_ptr()), 3, 68, T, T + 37, None, 0.025,
                                       ctypes.c_void_p(out.data_ptr()), None))
    _assert_same(out.cpu().numpy(), _host(base, [T] * 3, 0.025), "C ABI t_stride > n_frames")


def test_tiny_clips_constant_rows_and_nan(P):
    rng = np.random.default_rng(5)
    st = np.cumsum(rng.standard_normal((8, 19, 40)), axis=2).astype(np.float32)
    st[3] = 1.5                                   # every row constant: thr 0 -> 1e-16, no peaks
    st[4, 5] = 7.0                                # one constant row among walks
    st[5, 0, 17] = np.nan                         # a single NaN
    st[6, :, 20] = np.nan                         # a NaN in every row
    st[7, 2, :] = np.nan
    frames = [0, 1, 2, 40, 40, 40, 40, 40]
    _check(P, st, WINDOWS, frames, "tiny / constant / NaN")
    _check(P, st[:1, :, :0], (0.05,), [0], "T = 0 tensor")
    _check(P, st[:1, :, :1], (0.05,), [1], "T = 1 tensor")


def test_multi_chunk_rows_ragged(P):
    """Rows of several 1024-frame chunks, frame counts on and next to chunk boundaries."""
    rng = np.random.default_rng(6)
    T = 5000
    st = np.cumsum(rng.standard_normal((5, 34, T)), axis=2).astype(np.float32)
    st[2] = np.round(st[2])                       # integer-valued: exact ties against mx - delta
    st[3] = np.sin(np.arange(T) * 0.37)[None, :] + 0.01 * st[3]
    _check(P, st, (0.025, 0.0005), [T, 2049, 1025, 1024, 4097], "multi-chunk")


def test_forty_thousand_clips(P):
    rng = np.random.default_rng(7)
    B, T = 40000, 40
    st = np.cumsum(rng.standard_normal((B, 19, T)), axis=2).astype(np.float32)
    frames = rng.integers(0, T + 1, B)
    got = _device_beat(P, st, 0.025, frames)
    idx = np.r_[np.arange(0, B, 53), np.arange(B - 64, B)]
    _assert_same(got[idx], _host(st[idx], frames[idx], 0.025), "40000 clips")


def test_one_hour_row(P):
    """143 999 frames, the size of one hour at 50 / 25 ms: 141 chunks on 256 threads."""
    rng = np.random.default_rng(8)
    st = np.cumsum(rng.standard_normal((1, 19, 143999)), axis=2).astype(np.float32)
    _check(P, st, (0.025, 0.0005), what="one hour")


def test_errors(P):
    import torch
    st = torch.zeros((2, 68, 50), device="cuda")
    with pytest.raises(TypeError):
        P.beat_extraction_batch(st.cpu(), 0.05)
    with pytest.raises(ValueError):
        P.beat_extraction_batch(st[:, :18].contiguous(), 0.05)
    with pytest.raises(ValueError):
        P.beat_extraction_batch(st.double(), 0.05)
    with pytest.raises(ValueError):
        P.beat_extraction_batch(st[0], 0.05)
    with pytest.raises(ValueError):
        P.beat_extraction_batch(st, 0.05, torch.zeros(2, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        P.beat_extraction_batch(st, 0.05, torch.zeros(3, dtype=torch.int64, device="cuda"))
    with pytest.raises(TypeError):
        P.beat_extraction_batch(st, 0.05, torch.zeros(2, dtype=torch.int64))
    for w in (5.0, -1.0):                         # round(2 / w) = 0, -2: the host raises ValueError too
        with pytest.raises(ValueError):
            P.beat_extraction_batch(st, w)
        with pytest.raises(ValueError):
            P.MidTermFeatures.beat_extraction(np.zeros((68, 50)), w)


def _write_wav(path, x, fs):
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(fs)
        w.writeframes(x.astype("<i2").tobytes())


def test_directory_feature_extraction_beat(P, tmp_path):
    import torch
    from pyaudioanalysis_b200 import MidTermFeatures as M
    from pyaudioanalysis_b200.batch import mid_feature_extraction_batch
    fs = 16000
    clips = [pulse_clip(60 + i, 10 * fs, fs, bpm) for i, bpm in enumerate((120, 90, 140, 75, 100, 128))]
    for i, x in enumerate(clips):
        _write_wav(str(tmp_path / ("c%02d.wav" % i)), x, fs)
    M.VERBOSE = False
    feats, files, names = M.directory_feature_extraction(str(tmp_path), 1.0, 1.0, 0.05, 0.025, compute_beat=True)
    assert feats.shape == (6, 138) and names[-2:] == ["bpm", "ratio"]
    # the path this replaces: the same batch's st copied to the host, beat_extraction per file
    _, st = mid_feature_extraction_batch(torch.from_numpy(np.stack(clips)).cuda(), fs, 16000, 16000, 800, 400)
    ref = _host(st.cpu().numpy(), [st.shape[2]] * 6, 0.025)
    _assert_same(feats[:, -2:], ref, "directory_feature_extraction")
    plain, _, names2 = M.directory_feature_extraction(str(tmp_path), 1.0, 1.0, 0.05, 0.025, compute_beat=False)
    _assert_same(plain, feats[:, :-2], "features without the beat")
    assert names2 == names[:-2]


def test_file_classification_vector_beat(P):
    import torch
    from pyaudioanalysis_b200 import consumers as C
    from pyaudioanalysis_b200.batch import long_term_mean_batch, mid_feature_extraction_batch
    fs = 16000
    x = pulse_clip(70, 8 * fs, fs, 110)
    mt, st_w = 1.0, 0.05
    mid, st = mid_feature_extraction_batch(torch.from_numpy(x).cuda().reshape(1, -1), fs, mt * fs, mt * fs, round(fs * st_w),
                                           round(fs * st_w))
    lt = long_term_mean_batch(mid)[0].double().cpu().numpy()
    beat = _host(st.cpu().numpy(), [st.shape[2]], st_w)[0]
    vec = np.append(lt, beat)
    rng = np.random.default_rng(9)
    mean, std = vec + rng.normal(0, 0.1, vec.size), np.full(vec.size, 0.5)
    train = rng.normal(0, 1, (12, vec.size))
    knn = types.SimpleNamespace(features=train, labels=np.arange(12) % 3, neighbors=5)
    cid, prob = C.file_classification_vector(x, fs, knn, "knn", mean, std, mt, mt, st_w, st_w, compute_beat=True)
    ref_id, ref_p = C.knn_classify_matrix(knn, ((vec - mean) / std).reshape(1, -1))
    assert cid == ref_id[0]
    np.testing.assert_array_equal(prob, ref_p[0])
    # the beat entries are what moved the vector: the same call without them sees 136 values
    knn136 = types.SimpleNamespace(features=train[:, :136], labels=knn.labels, neighbors=5)
    cid2, _ = C.file_classification_vector(x, fs, knn136, "knn", mean[:136], std[:136], mt, mt, st_w, st_w)
    assert cid2 == C.knn_classify_matrix(knn136, ((lt - mean[:136]) / std[:136]).reshape(1, -1))[0][0]

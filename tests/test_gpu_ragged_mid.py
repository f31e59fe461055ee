"""GPU: ragged mid-term pooling, long-term mean and per-clip counts, and the directory wrappers that batch a folder of
files of different lengths through them.

Kernel level: a clip of a ragged batch (frame / window counts given per clip, NaN past them) gives bit for bit what it
gives alone, for frame counts around the step and the window ratio, zero, negative and beyond the row stride, and window
ratios 39, 1, 0, -1 and longer than the clip; through the C ABI only the columns below a clip's own window count are
written.  Path level: the adversarial bank as one ragged batch through mid_feature_extraction_batch(lengths=).
Wrapper level: a generated folder of 16 kHz files of distinct lengths, a 44.1 kHz group, a stereo and a float file,
against the same wrappers run on one-file folders and against the oracle; and one launch chain for a folder of 40
files of nearly equal length.
"""
import ctypes
import os

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import ragged
from tests.parity import check_close, check_mid_propagated, exception_bounds
from tests.test_gpu_mid import oracle_st, rows

pytestmark = pytest.mark.gpu

T_STRIDE = 150


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    pkg.ShortTermFeatures.PRINT_SPECTROGRAM_SHAPE = False
    pkg.MidTermFeatures.VERBOSE = False
    return pkg


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def clamp(v, hi):
    return min(max(int(v), 0), hi)


def padded(F, counts, stride, seed):
    """float32 [B, F, stride] host array: clip b has rows() values in its first clamp(counts[b]) columns, NaN after."""
    rng = np.random.default_rng(seed)
    x = np.full((len(counts), F, stride), np.nan, dtype=np.float32)
    for b, n in enumerate(counts):
        n = clamp(n, stride)
        if n:
            x[b, :, :n] = rows(rng, F, n, b)
    return x


@pytest.mark.parametrize("ratio,stepr", [(39, 40), (39, 5), (1, 1), (1, 3), (0, 3), (-1, 2), (T_STRIDE + 7, 4)])
def test_mid_pool_ragged_equals_alone(P, ratio, stepr):
    import torch
    from pyaudioanalysis_b200._lib import lib
    counts = [0, 1, stepr - 1, stepr, stepr + 1, ratio, ratio + 1, T_STRIDE, -3, T_STRIDE + 5]
    F = 68
    host = padded(F, counts, T_STRIDE, 100 + stepr)
    st = torch.from_numpy(host).cuda()
    fr = torch.tensor(counts, dtype=torch.int64, device="cuda")
    got = P.mid_pool_batch(st, ratio, stepr, n_frames=fr).cpu().numpy()
    M = lib().b200aa_mid_windows(T_STRIDE, stepr)
    assert got.shape == (len(counts), 2 * F, M)
    # through the C ABI into a NaN-filled output: exactly the columns below each clip's window count are written
    raw = torch.full((len(counts), 2 * F, M), float("nan"), device="cuda")
    assert lib().b200aa_mid_pool_ragged(ctypes.c_void_p(st.data_ptr()), len(counts), F, T_STRIDE,
                                        ctypes.c_void_p(fr.data_ptr()), ratio, stepr, ctypes.c_void_p(raw.data_ptr()),
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    raw = raw.cpu().numpy()
    for b, n in enumerate(counts):
        T = clamp(n, T_STRIDE)
        Mb = lib().b200aa_mid_windows(T, stepr)
        what = "ratio %d step %d, clip %d of %d frames" % (ratio, stepr, b, T)
        assert not got[b, :, Mb:].any(), what + ": columns past the clip's windows"
        assert not np.isnan(raw[b, :, :Mb]).any() and np.isnan(raw[b, :, Mb:]).all(), what + ": columns written"
        assert np.array_equal(bits(raw[b, :, :Mb]), bits(got[b, :, :Mb])), what
        if T == 0:
            continue
        alone = P.mid_pool_batch(torch.from_numpy(np.ascontiguousarray(host[b:b + 1, :, :T])).cuda(), ratio, stepr,
                                 n_frames=T).cpu().numpy()
        assert alone.shape == (1, 2 * F, Mb), what
        assert np.array_equal(bits(alone[0]), bits(got[b, :, :Mb])), what + ": differs from the clip alone"


def test_long_term_mean_ragged_equals_alone(P):
    import torch
    stride = 70
    counts = [0, 1, 31, 32, 33, stride, stride + 3, -1, 5]
    x = padded(136, counts, stride, 7)
    got = P.long_term_mean_batch(torch.from_numpy(x).cuda(),
                                 n_windows=torch.tensor(counts, dtype=torch.int64, device="cuda")).cpu().numpy()
    for b, n in enumerate(counts):
        Mb = clamp(n, stride)
        if Mb == 0:
            assert np.isnan(got[b]).all(), "a clip of no windows averages to NaN (np.mean of an empty axis)"
            continue
        alone = P.long_term_mean_batch(torch.from_numpy(np.ascontiguousarray(x[b:b + 1, :, :Mb])).cuda()).cpu().numpy()
        assert np.array_equal(bits(alone[0]), bits(got[b])), "clip %d of %d windows differs from the clip alone" % (b, Mb)
    empty = P.long_term_mean_batch(torch.zeros((2, 136, 0), device="cuda"),
                                   n_windows=torch.tensor([0, 4], dtype=torch.int64, device="cuda")).cpu().numpy()
    assert np.isnan(empty).all()


@pytest.mark.parametrize("fs,w,s", [(16000, 800, 400), (44100, 882, 441), (16000, 400, 160)])
def test_frame_counts(P, fs, w, s):
    import torch
    from pyaudioanalysis_b200._lib import lib
    lengths = [0, w - 1, w, w + s - 1, 10 * fs, 60 * fs, 1]
    d = torch.tensor(lengths, dtype=torch.int64, device="cuda")
    frames = P.frame_counts(d, w, s).cpu().tolist()
    assert frames == [lib().b200aa_num_frames(n, w, s) for n in lengths]
    for stepr in (1, 39, 40):
        fr, win = P.frame_counts(d, w, s, stepr)
        assert fr.cpu().tolist() == frames
        assert win.cpu().tolist() == [lib().b200aa_mid_windows(t, stepr) for t in frames]
    with pytest.raises(ValueError):
        P.frame_counts(d, w, s, 0)
    assert P.frame_counts(d[:0], w, s).numel() == 0


@pytest.mark.parametrize("fs,w,s,mw,ms", [(16000, 800, 400, 3200, 1600), (44100, 882, 441, 8820, 4410),
                                          (16000, 800, 400, 32000, 16000)])
def test_mid_path_ragged_bank(P, fs, w, s, mw, ms):
    """The adversarial bank as ONE ragged batch (int16 and float32): every int16 clip bit for bit the clip alone, every
    clip within the propagated tolerance of the oracle, zero past its own counts."""
    import torch
    from pyaudioanalysis_b200._lib import get_plan, lib
    ratio, stepr = O.mid_ratios(mw, ms, w, s)
    kind = get_plan(fs, w, s).kernel_kind()
    for bank, dtype in ((SG.bank(fs, w, s), np.int16), (SG.float_bank(fs, w, s), np.float32)):
        names, clips = list(bank), list(bank.values())
        d, lens = ragged(clips, dtype)
        mid, st = P.mid_feature_extraction_batch(d, fs, mw, ms, w, s, lengths=lens)
        mid, st = mid.cpu().numpy(), st.cpu().numpy()
        for i, (name, x) in enumerate(zip(names, clips)):
            T = lib().b200aa_num_frames(x.size, w, s)
            M = lib().b200aa_mid_windows(T, stepr)
            what = "fs=%d %d/%d mid %d/%d: %s" % (fs, w, s, mw, ms, name)
            assert not st[i, :, T:].any() and not mid[i, :, M:].any(), what + ": columns past the clip's counts"
            if dtype == np.int16:
                amid, ast = P.mid_feature_extraction_batch(torch.from_numpy(x).cuda()[None], fs, mw, ms, w, s)
                assert np.array_equal(bits(ast[0].cpu().numpy()), bits(st[i, :, :T])), what + ": st differs from alone"
                assert np.array_equal(bits(amid[0].cpu().numpy()), bits(mid[i, :, :M])), what + ": mid differs from alone"
            ref = oracle_st(x.astype(np.float64) if dtype == np.float32 else x, fs, w, s)
            check_mid_propagated(mid[i, :, :M], st[i, :, :T], ref, ratio, stepr, w // 2, what,
                                 allow=exception_bounds(name, kind))


# ----------------------------------------------------------------------------------------------------- directory wrappers
FS = 16000
WIN = (1.0, 1.0, 0.05, 0.05)          # mid window, mid step, short window, short step (seconds)


def write_folder(d):
    """40 16 kHz mono PCM16 files of distinct lengths (two one sample apart, one of exactly fs / 5 samples), three
    44.1 kHz files, a stereo file and a float WAV.  Returns {file name: (fs, mono signal as analysed, int16 coded)}."""
    from scipy.io import wavfile
    d.mkdir()
    rng = np.random.default_rng(77)
    lens = sorted(set(rng.integers(FS // 5 + 1, 3 * FS, size=60).tolist()))[:37]
    lens += [lens[-1] + 1, FS // 5, 2 * FS + 123]
    out = {}
    for i, n in enumerate(lens):
        x = O.synth_clip(500 + i, n, FS)
        wavfile.write(str(d / ("a%02d.wav" % i)), FS, x)
        out["a%02d.wav" % i] = (FS, x, True)
    for i, n in enumerate((44100, 44100 + 17, 70000)):
        x = O.synth_clip(600 + i, n, 44100)
        wavfile.write(str(d / ("b%d.wav" % i)), 44100, x)
        out["b%d.wav" % i] = (44100, x, True)
    x = O.synth_clip(700, 30001, FS)
    stereo = np.stack([x, O.synth_clip(701, 30001, FS)], axis=1)
    wavfile.write(str(d / "c_stereo.wav"), FS, stereo)
    out["c_stereo.wav"] = (FS, (stereo[:, 1] / 2) + (stereo[:, 0] / 2), False)
    f = (O.synth_clip(702, 27777, FS) / 32768.0).astype(np.float32)
    wavfile.write(str(d / "d_float.wav"), FS, f)
    out["d_float.wav"] = (FS, f, False)
    return out


def one_file_folder(tmp, src, name):
    import shutil
    d = tmp / ("one_" + name.replace(".", "_"))
    if not d.exists():
        d.mkdir()
        shutil.copy(str(src / name), str(d / name))
    return str(d)


def same_rows(got, ref, int_coded, what):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if int_coded:
        assert np.array_equal(got.view(np.int64), ref.view(np.int64)), what + ": differs from the file alone"
    else:
        check_close(got, ref, what + " (float32-coded file)")


def test_directory_wrappers(P, tmp_path):
    M = P.MidTermFeatures
    src = tmp_path / "mix"
    info = write_folder(src)
    names = sorted(info)
    for beat in (True, False):
        feats, files, fnames = M.directory_feature_extraction(str(src), *WIN, compute_beat=beat)
        assert [os.path.basename(f) for f in files] == names
        assert feats.shape == (len(names), 138 if beat else 136) and len(fnames) == feats.shape[1]
        for k, name in enumerate(names):
            fs, x, int_coded = info[name]
            alone, afiles, anames = M.directory_feature_extraction(one_file_folder(tmp_path, src, name), *WIN,
                                                                   compute_beat=beat)
            assert anames == fnames
            same_rows(feats[k], alone, int_coded, "%s (beat %s)" % (name, beat))
            if not beat:
                ref = O.mid_feature_extraction(x, fs, fs, fs, round(fs * 0.05), round(fs * 0.05))[0].mean(axis=1)
                check_close(feats[k], ref, "%s against the oracle" % name, rtol=2e-4, atol=2e-5)
    # no averaging: every mid-term vector of every file
    X, idx, files = M.directory_feature_extraction_no_avg(str(src), 1.0, 0.5, 0.05, 0.025)
    a = 0
    for k, name in enumerate(names):
        Xa, _, _ = M.directory_feature_extraction_no_avg(one_file_folder(tmp_path, src, name), 1.0, 0.5, 0.05, 0.025)
        same_rows(X[a:a + Xa.shape[0]], Xa, info[name][2], "no_avg " + name)
        assert (idx[a:a + Xa.shape[0]] == k).all()
        a += Xa.shape[0]
    assert a == X.shape[0]
    # three class folders in one pass: each folder's matrix is that folder's own directory_feature_extraction
    from scipy.io import wavfile
    other = tmp_path / "other"
    other.mkdir()
    for i, n in enumerate((20000, 20001, 33333, 47000, 9000)):
        wavfile.write(str(other / ("o%d.wav" % i)), FS, O.synth_clip(800 + i, n, FS))
    (tmp_path / "empty").mkdir()
    dirs = [str(src), str(tmp_path / "empty"), str(other) + os.sep]
    for beat in (False, True):
        f3, classes, fn3 = M.multiple_directory_feature_extraction(dirs, *WIN, compute_beat=beat)
        assert classes == ["mix", "other"] and len(f3) == 2 and len(fn3) == 2
        for f, fn, d in zip(f3, fn3, (dirs[0], dirs[2])):
            ref, rfiles, _ = M.directory_feature_extraction(d, *WIN, compute_beat=beat)
            assert fn == rfiles and f.shape == ref.shape
            for k, path in enumerate(fn):
                int_coded = info[os.path.basename(path)][2] if d == dirs[0] else True
                same_rows(f[k], ref[k], int_coded, "multiple_directory " + path)


def test_file_dir_writer(P, tmp_path):
    import shutil
    M = P.MidTermFeatures
    src = tmp_path / "mix"
    info = write_folder(src)
    d = tmp_path / "few"
    d.mkdir()
    keep = ["a00.wav", "a37.wav", "a38.wav", "a39.wav", "b1.wav", "c_stereo.wav", "d_float.wav"]
    for name in keep:
        shutil.copy(str(src / name), str(d / name))
    M.mid_feature_extraction_file_dir(str(d), *WIN, store_short_features=True, store_csv=True)
    ref_dir = tmp_path / "ref"
    ref_dir.mkdir()
    for name in keep:
        out = str(ref_dir / name)
        M.mid_feature_extraction_to_file(str(d / name), *WIN, out, store_short_features=True, store_csv=True)
        for suffix in ("_mt.npy", "_st.npy"):
            same_rows(np.load(str(d / name) + suffix), np.load(out + suffix), info[name][2], name + suffix)
        for suffix in ("_mt.csv", "_st.csv"):
            got, ref = np.loadtxt(str(d / name) + suffix, delimiter=","), np.loadtxt(out + suffix, delimiter=",")
            if info[name][2]:
                assert np.array_equal(got, ref), name + suffix
            else:
                check_close(got, ref, name + suffix)
    M.mid_feature_extraction_file_dir(str(d), *WIN)           # no short-term features: only _mt.npy, same values
    assert np.array_equal(np.load(str(d / "a00.wav_mt.npy")), np.load(str(ref_dir / "a00.wav_mt.npy")))


def test_file_shorter_than_a_window_raises(P, tmp_path):
    from scipy.io import wavfile
    d = tmp_path / "short"
    d.mkdir()
    wavfile.write(str(d / "a.wav"), FS, O.synth_clip(1, 2 * FS, FS))
    wavfile.write(str(d / "b.wav"), FS, O.synth_clip(2, int(0.3 * FS), FS))      # above fs / 5, below one 0.5 s window
    with pytest.raises(ValueError, match="need at least one array to concatenate"):
        P.MidTermFeatures.directory_feature_extraction(str(d), 1.0, 1.0, 0.5, 0.5)
    with pytest.raises(ValueError, match="need at least one array to concatenate"):
        P.MidTermFeatures.directory_feature_extraction_no_avg(str(d), 1.0, 1.0, 0.5, 0.5)


def test_folder_is_one_launch_chain(P, tmp_path):
    """40 files of 10 s +- up to 100 samples launch as many kernels as one file."""
    from scipy.io import wavfile
    from pyaudioanalysis_b200._lib import lib
    rng = np.random.default_rng(5)
    many, one = tmp_path / "many", tmp_path / "one"
    many.mkdir()
    one.mkdir()
    base = O.synth_clip(9, 10 * FS + 100, FS)
    for i, dn in enumerate(rng.integers(-100, 101, size=40)):
        wavfile.write(str(many / ("f%02d.wav" % i)), FS, base[:10 * FS + int(dn)])
    wavfile.write(str(one / "f.wav"), FS, base[:10 * FS])
    M = P.MidTermFeatures
    M.directory_feature_extraction(str(one), 1.0, 1.0, 0.05, 0.05, compute_beat=True)         # plans, first launches
    c0 = lib().b200aa_launch_count()
    M.directory_feature_extraction(str(one), 1.0, 1.0, 0.05, 0.05, compute_beat=True)
    c1 = lib().b200aa_launch_count()
    feats, _, _ = M.directory_feature_extraction(str(many), 1.0, 1.0, 0.05, 0.05, compute_beat=True)
    c2 = lib().b200aa_launch_count()
    assert feats.shape == (40, 138)
    assert c2 - c1 == c1 - c0, "one-file folder: %d launches, 40 files: %d" % (c1 - c0, c2 - c1)

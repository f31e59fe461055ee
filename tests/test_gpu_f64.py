"""GPU: the float64 feature path (kernel family 12) against the float64 oracle and the reference's goldens.

Held to the tolerances the oracle itself is held to against the reference (tests/test_oracle_golden.py: rtol 1e-9,
atol 1e-11), with the exceptions documented there (digitally silent frames, whose non-DC bins are float64 round-off).
Bit for bit: the normalisation records and rows 0-1 against NumPy, the mid-term pooling and the long-term mean against
NumPy on the kernel's own rows, every clip of a ragged batch against the clip alone, concurrent calls against the same
calls alone, and the float32 path's bits before and after float64 calls.

These tolerances are the path's published contract.  Beside them, tests/test_gpu_f64_feature_bounds.py holds rows 2-67
of every frame, constant frames and the deltas after them included, to a per-entry float64 error bound, and the feature
stage bit for bit to its NumPy statement on the kernel's own spectra."""
import threading

import numpy as np
import pytest
import torch

from oracle import st_oracle as O
from pyaudioanalysis_b200 import batch as BT
from tests import signals as SG
from tests.host_exe import bits

pytestmark = pytest.mark.gpu

RT, AT = 1e-9, 1e-11
F64 = torch.float64


def close(a, b, rt=RT, at=AT, what=""):
    np.testing.assert_allclose(a, b, rtol=rt, atol=at, err_msg=what)


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def st64(x, fs, w, s, deltas=True):
    return BT.feature_extraction_batch(dev(x), fs, w, s, deltas=deltas, dtype=F64)[0].cpu().numpy()


def clip(seed, n, fs, kind):
    x = O.synth_clip(seed, n, fs)
    if kind == "f32":
        return (x.astype(np.float32) * np.float32(0.37) + np.float32(11.5)).astype(np.float32)
    if kind == "f64":
        return x.astype(np.float64) * 1.000123e-3 + 0.25
    return x


# ---------------------------------------------------------------------------------------------------------------------
# normalisation and rows 0-1, bit for bit
@pytest.mark.parametrize("kind", ["i16", "f32", "f64"])
@pytest.mark.parametrize("n", [1, 7, 129, 4097, (1 << 17) + 333])
def test_clip_records_bit_for_bit(kind, n):
    x = clip(n, n, 16000, kind)
    rec = BT.clip_stats_f64(dev(x)).view(torch.float64).cpu().numpy()[0]
    y = np.asarray(x, dtype=np.float64) / 32768.0
    mean = y.mean()
    assert bits(rec[0]) == bits(mean)
    assert bits(rec[1]) == bits(np.abs(y - mean).max() + 1e-10)


@pytest.mark.parametrize("kind", ["i16", "f32", "f64"])
def test_rows_0_1_bit_for_bit(kind):
    fs, w, s = 16000, 800, 400
    x = clip(3, 3 * fs + 77, fs, kind)
    F = st64(x, fs, w, s)
    y = O.normalize_clip(x)
    T = O.frame_count(len(y), w, s)
    z = np.array([O._zcr(y[t * s:t * s + w]) for t in range(T)])
    e = np.array([O._energy(y[t * s:t * s + w]) for t in range(T)])
    np.testing.assert_array_equal(bits(F[0]), bits(z))
    np.testing.assert_array_equal(bits(F[1]), bits(e))


def test_signal_bank_rows_0_1_and_features():
    fs, w, s = 16000, 800, 400
    for name, x in SG.bank(fs, w, s).items():
        F = st64(x, fs, w, s)
        y = O.normalize_clip(x)
        T = O.frame_count(len(y), w, s)
        np.testing.assert_array_equal(bits(F[0]), bits([O._zcr(y[t * s:t * s + w]) for t in range(T)]), err_msg=name)
        np.testing.assert_array_equal(bits(F[1]), bits([O._energy(y[t * s:t * s + w]) for t in range(T)]), err_msg=name)
        ref, _ = O.feature_extraction(x, fs, w, s)
        bad = SG.noise_defined_frames(x, w, s)                   # frames defined by the float64 round-off of a transform
        ok = ~bad & ~np.concatenate([[False], bad[:-1]])         # and the deltas of the frame after one
        close(F[:, ok], ref[:, ok], what=name)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's goldens (doremi.npz: the fixture tests/test_oracle_golden.py holds the oracle to)
def test_doremi_golden(golden_doremi):
    g = golden_doremi
    F = st64(g["x"], 16000, 800, 400)
    assert F.shape == (68, 319)
    close(F[:, 5:], g["st"][:, 5:])
    np.testing.assert_allclose(F[:, :5], g["st"][:, :5], rtol=0, atol=1e-7)   # frames 0-3: digital silence
    sp = BT.spectrogram_batch(dev(g["x"]), 16000, 800, 400, dtype=F64)[0].cpu().numpy()
    np.testing.assert_allclose(sp, g["spectrogram"], rtol=2e-6, atol=1e-9)      # fixture stored as f32
    ch = BT.chromagram_batch(dev(g["x"]), 16000, 800, 400, dtype=F64)[0].cpu().numpy()
    close(ch, g["chromagram"])
    mid, st = BT.mid_feature_extraction_batch(dev(g["x"]), 16000, 16000, 16000, 800, 400, dtype=F64)
    close(mid[0].cpu().numpy(), g["mid"], 1e-6, 1e-9)       # window 0 pools the noise-defined silent frames


# ---------------------------------------------------------------------------------------------------------------------
# every window class: pair windows, 882 / 400 / 600, odd windows, and 1 s at 44.1 kHz (global-memory arrays)
@pytest.mark.parametrize("fs,w,s", [(16000, 800, 400), (16000, 512, 256), (44100, 882, 441), (16000, 400, 160),
                                    (16000, 600, 240), (16000, 801, 333), (8000, 257, 100), (44100, 44100, 22050)])
def test_windows_against_oracle(fs, w, s):
    x = clip(w, 6 * w + 3 * s + 5, fs, "i16")
    F = st64(x, fs, w, s)
    ref, _ = O.feature_extraction_loop(x, fs, w, s, tables_per_frame=False)
    close(F, ref, what="features %d/%d" % (w, s))
    sp = BT.spectrogram_batch(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy()
    close(sp, O.spectrogram(x, fs, w, s)[0], what="spectrogram")
    try:
        ref_ch = O.chromagram(x, fs, w, s)[0]
    except ValueError:              # a clipped last frame shorter than K: the reference's scatter raises, so does the path
        with pytest.raises(ValueError):
            BT.chromagram_batch(dev(x), fs, w, s, dtype=F64)
        return
    close(BT.chromagram_batch(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy(), ref_ch, what="chromagram")


@pytest.mark.parametrize("fs,w,s,n", [(16000, 800, 300, 2 * 16000 + 123), (16000, 800, 400, 16000 + 650),
                                      (44100, 882, 441, 44100 + 700), (16000, 801, 333, 12000 + 401)])
def test_chromagram_with_clipped_frames(fs, w, s, n):
    x = clip(n, n, fs, "f32")
    ch = BT.chromagram_batch(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy()
    close(ch, O.chromagram(x, fs, w, s)[0])


# ---------------------------------------------------------------------------------------------------------------------
# mid-term pooling and the long-term mean, bit for bit NumPy on the kernel's own rows
@pytest.mark.parametrize("ratio,stepr", [(-3, 2), (0, 1), (1, 1), (5, 3), (40, 40), (41, 20), (1000, 7)])
def test_mid_pool_bit_for_bit(ratio, stepr):
    fs, w, s = 16000, 800, 400
    x = clip(9, 4 * fs, fs, "i16")
    st = BT.feature_extraction_batch(dev(x), fs, w, s, dtype=F64)
    mid = BT.mid_pool_batch(st, ratio, stepr, dtype=F64)
    ref = O.mid_pool(st[0].cpu().numpy(), ratio, stepr)
    np.testing.assert_array_equal(bits(mid[0].cpu().numpy()), bits(ref))
    lt = BT.long_term_mean_batch(mid)[0].cpu().numpy()
    np.testing.assert_array_equal(bits(lt), bits(mid[0].cpu().numpy().T.mean(axis=0)))


# ---------------------------------------------------------------------------------------------------------------------
# ragged batches: each clip as alone, poisoned padding left unwritten
def test_ragged_batch_equals_each_clip_alone():
    fs, w, s = 16000, 800, 400
    lens = [fs * 2 + 17, w - 1, fs, w, 3 * fs]
    N = max(lens)
    xs = [clip(20 + i, n, fs, "f32") for i, n in enumerate(lens)]
    batch = np.zeros((len(lens), N), np.float32)
    for i, x in enumerate(xs):
        batch[i, :len(x)] = x
    L = dev(np.array(lens, np.int64))
    T = O.frame_count(N, w, s)
    poison = torch.empty((len(lens), 68, T), dtype=torch.int64, device="cuda").fill_(0x7ff4dead0000beef).view(F64)
    out = BT.feature_extraction_batch(dev(batch), fs, w, s, lengths=L, out=poison, dtype=F64).cpu().numpy()
    for i, x in enumerate(xs):
        Tb = O.frame_count(len(x), w, s)
        if Tb:
            np.testing.assert_array_equal(bits(out[i, :, :Tb]), bits(st64(x, fs, w, s)), err_msg="clip %d" % i)
        assert (out[i, :, Tb:].view(np.int64) == 0x7ff4dead0000beef).all(), "clip %d padding written" % i
    for which, fn in ((0, BT.spectrogram_batch), (1, BT.chromagram_batch)):
        rows = BT.row_counts(L, w, s, which).cpu().numpy()
        got = fn(dev(batch), fs, w, s, lengths=L, dtype=F64).cpu().numpy()
        for i, x in enumerate(xs):
            if rows[i]:
                alone = fn(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy()
                np.testing.assert_array_equal(bits(got[i, :rows[i]]), bits(alone), err_msg="rows %d clip %d" % (which, i))
    frames = BT.frame_counts(L, w, s)
    mid = BT.mid_pool_batch(torch.as_tensor(out).cuda(), 40, 40, n_frames=frames, dtype=F64).cpu().numpy()
    for i, x in enumerate(xs):
        Tb = O.frame_count(len(x), w, s)
        if Tb:
            np.testing.assert_array_equal(bits(mid[i, :, :-(-Tb // 40)]), bits(O.mid_pool(out[i, :, :Tb], 40, 40)))


# ---------------------------------------------------------------------------------------------------------------------
def test_concurrent_streams_and_threads_equal_alone():
    fs, w, s = 16000, 800, 400
    xs = [dev(clip(40 + i, 2 * fs + 100 * i, fs, "i16")) for i in range(6)]
    alone = [BT.feature_extraction_batch(x, fs, w, s, dtype=F64).cpu().numpy() for x in xs]
    got = [None] * len(xs)

    def work(i):
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            r = BT.feature_extraction_batch(xs[i], fs, w, s, dtype=F64)
        st.synchronize()
        got[i] = r.cpu().numpy()

    ts = [threading.Thread(target=work, args=(i,)) for i in range(len(xs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for a, b in zip(got, alone):
        np.testing.assert_array_equal(bits(a), bits(b))


def test_float32_path_unchanged_by_float64_calls():
    fs, w, s = 16000, 800, 400
    x = dev(clip(5, 2 * fs, fs, "i16"))
    before = BT.feature_extraction_batch(x, fs, w, s).cpu().numpy()
    BT.feature_extraction_batch(x, fs, w, s, dtype=F64)
    after = BT.feature_extraction_batch(x, fs, w, s).cpu().numpy()
    assert before.dtype == np.float32
    np.testing.assert_array_equal(before.view(np.int32), after.view(np.int32))


def test_float64_signals_need_the_float64_path_and_cpu_tensors_raise():
    x = torch.zeros(16000, dtype=F64, device="cuda")
    with pytest.raises(TypeError):
        BT.feature_extraction_batch(x, 16000, 800, 400)
    with pytest.raises(TypeError):
        BT.feature_extraction_batch(torch.zeros(16000, dtype=F64), 16000, 800, 400, dtype=F64)


def test_long_term_mean_ragged_bit_for_bit():
    rng = np.random.default_rng(7)
    mid = rng.normal(size=(4, 136, 23)) * 10 ** rng.uniform(-3, 3, size=(4, 136, 1))
    nw = np.array([23, 1, 0, 17], np.int64)
    got = BT.long_term_mean_batch(dev(mid), n_windows=dev(nw)).cpu().numpy()
    for b in range(4):
        with np.errstate(invalid="ignore", divide="ignore"):
            ref = mid[b, :, :nw[b]].T.mean(axis=0)
        np.testing.assert_array_equal(bits(got[b]), bits(ref), err_msg="clip %d" % b)


def test_beat_on_float64_rows_bit_for_bit():
    from pyaudioanalysis_b200 import MidTermFeatures as MT
    fs, w, s = 16000, 800, 400
    lens = [5 * fs + 3, 2 * fs, 9 * fs + 100]
    batch = np.zeros((3, max(lens)), np.int16)
    for i, n in enumerate(lens):
        batch[i, :n] = clip(60 + i, n, fs, "i16")
    L = dev(np.array(lens, np.int64))
    st = BT.feature_extraction_batch(dev(batch), fs, w, s, lengths=L, dtype=F64)
    frames = BT.frame_counts(L, w, s)
    got = BT.beat_extraction_batch(st, s / fs, n_frames=frames, dtype=F64).cpu().numpy()
    host = st.cpu().numpy()
    for i, n in enumerate(lens):
        T = O.frame_count(n, w, s)
        bpm, ratio = MT.beat_extraction(host[i, :, :T], s / fs)
        np.testing.assert_array_equal(bits(got[i]), bits([bpm, ratio]), err_msg="clip %d" % i)


# ---------------------------------------------------------------------------------------------------------------------
# the drop-ins under set_precision("float64"), and the float32 default around it
def test_drop_ins_follow_set_precision():
    import pyaudioanalysis_b200 as pkg
    from pyaudioanalysis_b200 import MidTermFeatures as MT
    from pyaudioanalysis_b200 import ShortTermFeatures as ST
    fs, w, s = 16000, 800, 400
    x = clip(77, 3 * fs + 11, fs, "f64")
    ST.PRINT_SPECTROGRAM_SHAPE, shape_flag = False, ST.PRINT_SPECTROGRAM_SHAPE
    try:
        before = ST.feature_extraction(x, fs, w, s)[0]
        mid32 = MT.mid_feature_extraction(x, fs, fs, fs, w, s)[0]
        pkg.set_precision("float64")
        assert pkg.get_precision() == "float64"
        F = ST.feature_extraction(x, fs, w, s)[0]
        np.testing.assert_array_equal(bits(F), bits(st64(x, fs, w, s)))
        close(F, O.feature_extraction(x, fs, w, s)[0])
        close(ST.spectrogram(x, fs, w, s)[0], O.spectrogram(x, fs, w, s)[0])
        close(ST.chromagram(x, fs, w, s)[0], O.chromagram(x, fs, w, s)[0])
        mid, st, names = MT.mid_feature_extraction(x, fs, fs, fs, w, s)
        np.testing.assert_array_equal(bits(st), bits(F))
        np.testing.assert_array_equal(bits(mid), bits(O.mid_pool(F, *O.mid_ratios(fs, fs, w, s))))
        assert len(names) == 136
        bpm = MT.beat_extraction(st, s / fs)
        assert bpm == MT.beat_extraction(F, s / fs)
        f32_in_f64_mode = BT.feature_extraction_batch(dev(x.astype(np.float32)), fs, w, s).cpu().numpy()[0]
    finally:
        pkg.set_precision("float32")
        ST.PRINT_SPECTROGRAM_SHAPE = shape_flag
    after = ST.feature_extraction(x, fs, w, s)[0]
    np.testing.assert_array_equal(bits(before), bits(after))
    np.testing.assert_array_equal(bits(mid32), bits(MT.mid_feature_extraction(x, fs, fs, fs, w, s)[0]))
    np.testing.assert_array_equal(f32_in_f64_mode.view(np.int32), ST.feature_extraction(x, fs, w, s)[0].astype(np.float32).view(np.int32))


def test_directory_wrapper_float64_decode(tmp_path):
    import pyaudioanalysis_b200 as pkg
    from pyaudioanalysis_b200 import MidTermFeatures as MT
    from pyaudioanalysis_b200 import audioio
    from pyaudioanalysis_b200._lib import DTYPE_F64
    from tests import wavgen
    fs = 16000
    flavours = [("s24", 2), ("s32", 1), ("s32", 2), ("f64", 1), ("f64", 2), ("s24", 1), ("s16", 2), ("f32", 1)]
    host64 = {("s24", 2), ("s32", 1), ("s32", 2), ("f64", 1), ("f64", 2)}
    for k, (name, ch) in enumerate(flavours):
        wavgen.write(str(tmp_path / ("%02d_%s_%d.wav" % (k, name, ch))), fs, wavgen.signal(name, ch, 30000 + 977 * k, 300 + k),
                     name)
    verbose, MT.VERBOSE = MT.VERBOSE, False
    pkg.set_precision("float64")
    try:
        clips = MT._folder_clips(str(tmp_path))
        for c, fl in zip(clips, flavours):
            assert (c.code == DTYPE_F64) == (fl in host64), (c.path, c.code)
        feats, files, _ = MT.directory_feature_extraction(str(tmp_path), 1.0, 1.0, 0.05, 0.05, compute_beat=False)
        with_beat, _, names = MT.directory_feature_extraction(str(tmp_path), 1.0, 1.0, 0.05, 0.05, compute_beat=True)
    finally:
        pkg.set_precision("float32")
        MT.VERBOSE = verbose
    assert len(files) == len(flavours) and names[-2:] == ["bpm", "ratio"]
    np.testing.assert_array_equal(bits(with_beat[:, :136]), bits(feats))      # the beat of float64 rows on kernel 4
    assert np.isfinite(with_beat[:, 136:]).all()
    for v, path in zip(feats, files):
        rate, x = audioio.read_audio_file(path)
        x = audioio.stereo_to_mono(x)
        mid, _, _ = O.mid_feature_extraction(x, rate, fs, fs, 800, 800)
        close(v, mid.mean(axis=1), what=path)

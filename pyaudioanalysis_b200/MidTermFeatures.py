"""Drop-in for ``pyAudioAnalysis.MidTermFeatures.mid_feature_extraction`` (MidTermFeatures.py:87-127), ``beat_extraction``
(:18-84) and the directory wrappers around them (``directory_feature_extraction`` :140-221,
``multiple_directory_feature_extraction`` :224-260, ``directory_feature_extraction_no_avg`` :263-309): files are decoded on
the GPU (PCM / float WAV, mono or stereo: ``audioio.wav_pcm_layout``, ``audioio.stage``) or on the host (other WAV
files, .aif / .aiff, and .mp3 / .au / .ogg when pydub is installed, as in the reference); files of equal sampling rate and
sample format, whatever their lengths, are staged in page-locked memory and batched into ragged GPU launches."""
import ctypes
import glob
import os

import numpy as np

from . import _lib, precision
from ._lib import lib, check, get_plan
from . import ShortTermFeatures
from .ShortTermFeatures import _as_clip, _as_clip64, _device64, _fs_int, _ptr
from .batch import mid_ratios


def mid_feature_extraction(signal, sampling_rate, mid_window, mid_step, short_window, short_step):
    """Mid-term feature extraction: (mid float64 [136 x M], short float64 [68 x T], 136 names).

    Short-term features with deltas (MidTermFeatures.py:93-95), then the mean and population
    standard deviation of every row over runs of ``ratio`` frames every ``step_ratio`` frames
    (:100-124), ``np.nan_to_num`` (:126).  All window arguments are in samples.  As in the reference, a mid-term
    window shorter than one short-term step gives ``ratio <= 0``: windows are Python slices, an empty one pools to 0.
    A mid-term step that rounds to 0 short-term steps raises ValueError (the reference's window loop never ends).
    """
    w, s = int(short_window), int(short_step)
    x, code = _as_clip(signal)
    plan = get_plan(_fs_int(sampling_rate), w, s)
    T = lib().b200aa_num_frames(x.shape[0], w, s)
    if T <= 0:
        ShortTermFeatures._raise_no_frames(plan.fs, w)
    ratio, stepr = mid_ratios(mid_window, mid_step, short_window, short_step)
    if stepr < 1:
        raise ValueError("mid-term step shorter than half a short-term step")
    st_names = ShortTermFeatures.feature_names(True)
    names = [n + "_mean" for n in st_names] + [n + "_std" for n in st_names]
    if precision.wide():
        import torch
        from .batch import mid_feature_extraction_batch
        mid, st = mid_feature_extraction_batch(_device64(signal), plan.fs, mid_window, mid_step, short_window, short_step,
                                               dtype=torch.float64)
        return mid[0].cpu().numpy(), st[0].cpu().numpy(), names
    M = lib().b200aa_mid_windows(T, stepr)
    mid = np.empty((136, M), dtype=np.float32)
    st = np.empty((68, T), dtype=np.float32)
    _lib.refuse_capture("b200aa_mid_features_host", _lib.HOST_BUFFER_WHY)
    check(lib().b200aa_mid_features_host(plan.handle, _ptr(x), code, x.shape[0], ratio, stepr, _ptr(mid), _ptr(st)))
    return mid.astype(np.float64), st.astype(np.float64), names


VERBOSE = True      # the reference prints one "Analyzing file ..." line per file


_BEAT_ROWS = (0, 1, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18)     # MidTermFeatures.py:31-32
_BEAT_EPS = 0.00000001                                                               # MidTermFeatures.py:13


def _peak_positions(v, delta):
    """Indices of the local maxima of ``v`` in the sense of the reference's ``utilities.peakdet`` (:33-103): a running
    maximum becomes a peak once the signal has dropped more than ``delta`` below it; the search for the next maximum
    starts after the signal has risen more than ``delta`` above the running minimum."""
    peaks = []
    mx, mn = -np.inf, np.inf
    mxpos = 0
    look_for_max = True
    for i, x in enumerate(v.tolist()):
        if x > mx:
            mx, mxpos = x, i
        if x < mn:
            mn = x
        if look_for_max:
            if x < mx - delta:
                peaks.append(mxpos)
                mn = x
                look_for_max = False
        elif x > mn + delta:
            mx, mxpos = x, i
            look_for_max = True
    return peaks


def beat_extraction(short_features, window_size, plot=False):
    """Beat-rate estimate from short-term features (reference MidTermFeatures.py:18-84): for 18 feature rows, local
    maxima with a threshold of twice the mean absolute first difference, histogram of the distances between successive
    maxima (in frames, 1 .. round(2 / window_size)), summed over the rows; returns (bpm of the tallest bin, its share).
    Host code (a serial scan per row over a few hundred frames); the short-term rows come from the GPU path."""
    st = np.asarray(short_features, dtype=np.float64)
    n_frames = st.shape[1]
    max_beat_time = int(round(2.0 / window_size))
    hist_all = np.zeros((max_beat_time,))
    for i in _BEAT_ROWS:
        row = st[i]
        thr = 2.0 * np.abs(row[:-1] - row[1:]).mean()
        if thr <= 0:
            thr = 0.0000000000000001
        pos = np.asarray(_peak_positions(row, thr), dtype=np.int64)
        d = pos[1:] - pos[:-1]
        d = d[(d >= 1) & (d <= max_beat_time)]
        hist_all += np.bincount(d - 1, minlength=max_beat_time).astype(float) / n_frames
    centers = np.arange(1, max_beat_time + 1, dtype=np.float64)
    k = int(np.argmax(hist_all))
    bpm = (60 / (centers * window_size))[k]
    ratio = hist_all[k] / (hist_all.sum() + _BEAT_EPS)
    if plot:
        ShortTermFeatures._plot(hist_all[None, :])
    return bpm, ratio


_MAX_CHUNK_BYTES = 1 << 30       # padded staging bytes of one chunk; a single larger clip gets a chunk of its own
_MAX_PADDING = 0.25              # padding samples of a chunk per sample of its clips (DESIGN §7, rank 1)


class _Clip:
    """One audio file of a folder: either still on disk as a WAV file whose data chunk the device decodes (``layout`` =
    (data_offset, format, channels) of ``audioio.wav_pcm_layout``; read later straight into page-locked staging memory)
    or already decoded to a 1-D array."""
    __slots__ = ("path", "fs", "n", "data", "code", "layout")

    def __init__(self, path, fs, n, data, code, layout=None):
        self.path, self.fs, self.n, self.data, self.code, self.layout = path, int(fs), int(n), data, code, layout


def _staged_exactly(fmt, ch):
    """Whether the device decode's int16 / float32 staging of a WAV data chunk is the host decode's signal exactly
    (DESIGN §7's table): not for stereo 24 / 32-bit PCM, mono 32-bit PCM and float64, which the float64 path reads on
    the host as float64."""
    from . import audioio
    if fmt == audioio.PCM_F64:
        return False
    if fmt == audioio.PCM_S32:
        return False
    return not (fmt == audioio.PCM_S24 and ch == 2)


def _open_clip(path):
    """audioBasicIO.read_audio_file + stereo_to_mono for one file, lazily for every WAV flavour audioio.wav_pcm_layout
    accepts: mono 8 / 16-bit PCM stages as int16, everything else as float32, the code _as_clip gives.  Under
    set_precision("float64") a file whose staged form would not be exact is decoded on the host and staged as float64
    (_as_clip64)."""
    from . import audioio
    from ._lib import DTYPE_I16, DTYPE_F32
    wide = precision.wide()
    if os.path.splitext(path)[1].lower() == ".wav":
        lay = audioio.wav_pcm_layout(path)
        if lay is not None and (not wide or _staged_exactly(lay[4], lay[1])):
            fs, ch, n, off, fmt = lay
            code = DTYPE_I16 if ch == 1 and fmt in (audioio.PCM_U8, audioio.PCM_S16) else DTYPE_F32
            return _Clip(path, fs, n, None, code, layout=(off, fmt, ch))
    fs, x = audioio.read_audio_file(path)
    clip, code = (_as_clip64 if wide else _as_clip)(audioio.stereo_to_mono(x))
    return _Clip(path, fs, clip.shape[0], clip, code)


def _plan_chunks(clips, max_bytes=None, max_padding=None):
    """Cut a list of _Clip into batches: [[index into clips, ...], ...], every index exactly once.  A chunk holds clips
    of one (rate, format), longest first; it is staged as [len(chunk), n_max] with n_max its first clip's length, so
    its padding is len(chunk) * n_max - (its clips' samples).  Clips of a (rate, format) are taken longest first and a
    chunk is closed when the next clip would bring its padded bytes above ``max_bytes`` or its padding above
    ``max_padding`` times its clips' samples; a clip larger than ``max_bytes`` on its own is a chunk of its own.  The
    bounds default to _MAX_CHUNK_BYTES and _MAX_PADDING."""
    from ._lib import DTYPE_I16, DTYPE_F64
    max_bytes = _MAX_CHUNK_BYTES if max_bytes is None else max_bytes
    max_padding = _MAX_PADDING if max_padding is None else max_padding
    groups = {}
    for idx, c in enumerate(clips):
        groups.setdefault((c.fs, c.code), []).append(idx)
    chunks = []
    for (_, code), idxs in groups.items():
        item = 2 if code == DTYPE_I16 else (8 if code == DTYPE_F64 else 4)
        cur, n_max, payload = [], 0, 0
        for i in sorted(idxs, key=lambda i: (-clips[i].n, i)):
            n, k = clips[i].n, len(cur) + 1
            if cur and (k * n_max * item > max_bytes or k * n_max - (payload + n) > max_padding * (payload + n)):
                chunks.append(cur)
                cur = []
            if not cur:
                n_max, payload = n, 0
            cur.append(i)
            payload += n
        if cur:
            chunks.append(cur)
    return chunks


def _mid_per_clip(clips, mid_window, mid_step, short_window, short_step, want_short=False, want_long_term=False,
                  want_beat=False):
    """Mid-term results of a list of _Clip, in input order: (mid float64 [136 x M] or its long-term mean [136],
    st float64 [68 x T] | None, (bpm, ratio) of beat_extraction(st, short_step) | None).  Clips of one (rate, format)
    share launches as ragged batches (_plan_chunks); every clip's results are bit for bit those of the clip alone.  The
    long-term mean and the beat are computed on the GPU from the resident features."""
    import torch
    from .batch import mid_feature_extraction_batch, long_term_mean_batch, beat_extraction_batch, frame_counts
    from . import audioio
    from ._lib import DTYPE_F64
    L = lib()
    dtype = precision.torch_dtype()
    results = [None] * len(clips)
    for part in _plan_chunks(clips):
        chunk = [clips[i] for i in part]
        fs = chunk[0].fs
        w, s = round(fs * short_window), round(fs * short_step)
        mw, ms = round(mid_window * fs), round(mid_step * fs)
        if L.b200aa_num_frames(chunk[-1].n, w, s) <= 0:
            check(_lib.ERR_TOO_SHORT)       # alone, the shortest clip has no frames: a ragged batch would give it none
        if chunk[0].code == DTYPE_F64:                 # decoded on the host in float64: one H2D copy of the padded batch
            host = np.zeros((len(chunk), chunk[0].n), dtype=np.float64)
            for k, c in enumerate(chunk):
                host[k, :c.n] = c.data
            dev, lengths = torch.from_numpy(host).cuda(), torch.tensor([c.n for c in chunk], dtype=torch.int64).cuda()
        else:
            dev, lengths = audioio.stage(chunk)        # one arena, one H2D copy, one decode launch
        mid, st = mid_feature_extraction_batch(dev, fs, mw, ms, w, s, lengths=lengths, dtype=dtype)
        stepr = mid_ratios(mw, ms, w, s)[1]
        if want_long_term or want_beat:
            n_frames, n_windows = frame_counts(lengths, w, s, stepr)
        first = (long_term_mean_batch(mid, n_windows=n_windows) if want_long_term else mid).cpu().numpy().astype(np.float64)
        st_h = st.cpu().numpy().astype(np.float64) if want_short else None
        beat = beat_extraction_batch(st, short_step, n_frames=n_frames, dtype=dtype).cpu().numpy() if want_beat else None
        for k, (i, c) in enumerate(zip(part, chunk)):
            T = L.b200aa_num_frames(c.n, w, s)
            results[i] = (first[k] if want_long_term else first[k][:, :L.b200aa_mid_windows(T, stepr)],
                          st_h[k][:, :T] if want_short else None, tuple(beat[k]) if want_beat else None)
    return results


def directory_feature_extraction(folder_path, mid_window, mid_step, short_window, short_step, compute_beat=True):
    """One long-term averaged 136-vector per audio file of a folder (reference MidTermFeatures.py:140-221).

    Window arguments are in seconds.  Returns (features [n_files x 136] -- a 1-D vector for a single file and an
    empty array for none, exactly like the reference's np.vstack logic --, file list, feature names).  Files are
    decoded by ``audioio`` (.wav, .aif / .aiff, and .mp3 / .au / .ogg when pydub is installed, as in the reference; a
    file that cannot be decoded raises instead of silently changing the file list).  ``compute_beat=True`` appends
    ``bpm`` and ``ratio`` of the GPU short-term features, computed on the GPU (``batch.beat_extraction_batch``, bit for bit
    this module's ``beat_extraction``, reference :18-84); only those two numbers per file are copied back.  Files of
    any length share launches (ragged batches per sampling rate and sample format).
    """
    clips = _folder_clips(folder_path)
    res = _mid_per_clip(clips, mid_window, mid_step, short_window, short_step, want_long_term=True, want_beat=compute_beat)
    return _folder_features(clips, res, compute_beat)


def _folder_clips(folder_path):
    """The files of a folder that directory_feature_extraction analyses, as _Clip, with the reference's prints
    (MidTermFeatures.py:155-190)."""
    types = ('*.wav', '*.aif', '*.aiff', '*.mp3', '*.au', '*.ogg')
    files = []
    for t in types:
        files.extend(glob.glob(os.path.join(folder_path, t)))
    files = sorted(files)
    clips = []
    for i, path in enumerate(files):
        if VERBOSE:
            print("Analyzing file {0:d} of {1:d}: {2:s}".format(i + 1, len(files), path))
        if os.stat(path).st_size == 0:
            if VERBOSE:
                print("   (EMPTY FILE -- SKIPPING)")
            continue
        c = _open_clip(path)
        if c.fs == 0:
            continue
        if c.n < float(c.fs) / 5:
            if VERBOSE:
                print("  (AUDIO FILE TOO SMALL - SKIPPING)")
            continue
        clips.append(c)
    return clips


def _folder_features(clips, res, compute_beat):
    """directory_feature_extraction's return value from its clips and their _mid_per_clip results (reference :191-221)."""
    names = []
    if not clips:
        return np.array([]), [], names
    st_names = ShortTermFeatures.feature_names(True)
    names = [n + "_mean" for n in st_names] + [n + "_std" for n in st_names]
    out, out_files = np.array([]), []
    appended = False
    for c, (v, _, beat) in zip(clips, res):
        out_files.append(c.path)
        if (not np.isnan(v).any()) and (not np.isinf(v).any()):      # reference :203-204
            if compute_beat:                                         # beat: reference :191, computed by kernel 4
                v = np.append(np.append(v, beat[0]), beat[1])        # :205-208
                if not appended:
                    names = names + ["bpm", "ratio"]
                    appended = True
            out = v if len(out) == 0 else np.vstack((out, v))
    return out, out_files, names


def multiple_directory_feature_extraction(path_list, mid_window, mid_step, short_window, short_step, compute_beat=False):
    """Reference MidTermFeatures.py:224-260: one feature matrix per class folder.  Every folder is decoded first (its
    "Analyzing file" lines print folder by folder), then the files of all folders share launches."""
    per_dir = [_folder_clips(d) for d in path_list]
    res = _mid_per_clip([c for clips in per_dir for c in clips], mid_window, mid_step, short_window, short_step,
                        want_long_term=True, want_beat=compute_beat)
    features, class_names, file_names = [], [], []
    a = 0
    for d, clips in zip(path_list, per_dir):
        f, fn, _ = _folder_features(clips, res[a:a + len(clips)], compute_beat)
        a += len(clips)
        if f.shape[0] > 0:
            features.append(f)
            file_names.append(fn)
            class_names.append(d.split(os.sep)[-2] if d[-1] == os.sep else d.split(os.sep)[-1])
    return features, class_names, file_names


def directory_feature_extraction_no_avg(folder_path, mid_window, mid_step, short_window, short_step):
    """Reference MidTermFeatures.py:263-309: every mid-term vector of every file, no long-term averaging.
    Returns (X [sum of windows x 136], file index per row, file list)."""
    files = []
    for t in ('*.wav', '*.aif', '*.aiff', '*.ogg'):
        files.extend(glob.glob(os.path.join(folder_path, t)))
    files = sorted(files)
    idxs, clips = [], []
    for i, path in enumerate(files):
        c = _open_clip(path)
        if c.fs == 0:
            continue
        idxs.append(i)
        clips.append(c)
    mids = _mid_per_clip(clips, mid_window, mid_step, short_window, short_step)
    mid_features, signal_idx = np.array([]), np.array([])
    for i, (mid, _, _) in zip(idxs, mids):
        rows = np.transpose(mid)
        if len(mid_features) == 0:
            mid_features = rows
            signal_idx = np.zeros((rows.shape[0],))          # the reference labels the first block 0 (:301)
        else:
            mid_features = np.vstack((mid_features, rows))
            signal_idx = np.append(signal_idx, i * np.ones((rows.shape[0],)))
    return mid_features, signal_idx, files


def mid_feature_extraction_to_file(file_path, mid_window, mid_step, short_window, short_step, output_file,
                                   store_short_features=False, store_csv=False, plot=False):
    """Reference MidTermFeatures.py:324-362: <output>_mt.npy ([136 x M] float64), optional <output>_st.npy
    ([68 x T]) and transposed CSV copies -- the on-disk formats the reference's CLI consumers read."""
    (mid, st, _), = _mid_per_clip([_open_clip(file_path)], mid_window, mid_step, short_window, short_step,
                                  want_short=store_short_features)
    _save_features(output_file, mid, st, store_short_features, store_csv, plot)


def _save_features(output_file, mid, st, store_short_features, store_csv, plot):
    if store_short_features:
        np.save(output_file + "_st", st)
        if plot:
            print("Short-term np file: " + output_file + "_st.npy saved")
        if store_csv:
            np.savetxt(output_file + "_st.csv", st.T, delimiter=",")
            if plot:
                print("Short-term CSV file: " + output_file + "_st.csv saved")
    np.save(output_file + "_mt", mid)
    if plot:
        print("Mid-term np file: " + output_file + "_mt.npy saved")
    if store_csv:
        np.savetxt(output_file + "_mt.csv", mid.T, delimiter=",")
        if plot:
            print("Mid-term CSV file: " + output_file + "_mt.csv saved")


def mid_feature_extraction_file_dir(folder_path, mid_window, mid_step, short_window, short_step,
                                    store_short_features=False, store_csv=False, plot=False):
    """Reference MidTermFeatures.py:365-377: mid_feature_extraction_to_file(f, ..., output_file=f) for every .wav file
    of the folder, the files computed in shared launches and written in the reference's order."""
    files = glob.glob(folder_path + os.sep + '*.wav')
    res = _mid_per_clip([_open_clip(f) for f in files], mid_window, mid_step, short_window, short_step,
                        want_short=store_short_features)
    for f, (mid, st, _) in zip(files, res):
        _save_features(f, mid, st, store_short_features, store_csv, plot)

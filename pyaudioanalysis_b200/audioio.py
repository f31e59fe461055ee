"""File decode in front of the GPU path (SURVEY 8f rank 2): the reference's ``audioBasicIO.read_audio_file`` (:86-110) and
``stereo_to_mono`` (:156-168), plus a decoder that reads 16-bit PCM WAV data STRAIGHT INTO page-locked staging memory
(``read_wav_into`` / ``PinnedBatch``) so a folder of files goes file -> pinned buffer -> H2D copy with no intermediate
host copy.  Formats: .wav (own RIFF walk for PCM16, scipy for everything else wavfile.read understands), .aif / .aiff
(stdlib ``aifc``, big-endian 16-bit like the reference), .mp3 / .au / .ogg through pydub when it is installed (as in the
reference); undecodable files raise instead of being skipped silently.
"""
import os
import struct

import numpy as np


class DecodeError(IOError):
    pass


def stereo_to_mono(signal):
    """audioBasicIO.py:156-168: (L / 2) + (R / 2) in float64 for two channels, flatten a single column."""
    if signal.ndim == 2:
        if signal.shape[1] == 1:
            signal = signal.flatten()
        elif signal.shape[1] == 2:
            signal = (signal[:, 1] / 2) + (signal[:, 0] / 2)
    return signal


def wav_pcm16_layout(path):
    """(sampling_rate, channels, n_frames, data_offset) of a plain 16-bit PCM RIFF/WAVE file, or None for anything else
    (float / 24-bit / extensible sub-formats other than PCM / RF64 ...: left to scipy)."""
    try:
        with open(path, "rb") as f:
            head = f.read(12)
            if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
                return None
            fmt = None
            while True:
                ck = f.read(8)
                if len(ck) < 8:
                    return None
                cid, size = ck[:4], struct.unpack("<I", ck[4:])[0]
                if cid == b"fmt ":
                    body = f.read(size + (size & 1))
                    tag, ch, fs, _, _, bits = struct.unpack("<HHIIHH", body[:16])
                    if tag == 0xFFFE and size >= 26:                      # WAVE_FORMAT_EXTENSIBLE: sub-format GUID starts with the tag
                        tag = struct.unpack("<H", body[24:26])[0]
                    fmt = (tag, ch, fs, bits)
                elif cid == b"data":
                    if fmt is None or fmt[0] != 1 or fmt[3] != 16 or fmt[1] < 1:
                        return None
                    tag, ch, fs, bits = fmt
                    off = f.tell()
                    avail = os.fstat(f.fileno()).st_size - off
                    size = min(size, avail)
                    return fs, ch, size // (2 * ch), off
                else:
                    f.seek(size + (size & 1), 1)
    except (OSError, struct.error):
        return None


def read_wav_into(path, dst):
    """Decode a mono 16-bit PCM WAV file straight into ``dst`` (a C-contiguous int16 array, e.g. one row of a pinned
    staging buffer).  Returns the sampling rate, or None when the file is not mono PCM16 of exactly ``dst.size`` frames."""
    lay = wav_pcm16_layout(path)
    if lay is None or lay[1] != 1 or lay[2] != dst.size or dst.dtype != np.int16 or not dst.flags["C_CONTIGUOUS"]:
        return None
    with open(path, "rb", buffering=0) as f:
        f.seek(lay[3])
        got = f.readinto(memoryview(dst).cast("B"))
    if got != 2 * dst.size:
        raise DecodeError("short read in " + path)
    return lay[0]


def read_aif(path):
    """.aif / .aiff: big-endian 16-bit frames (audioBasicIO.py:113-127; the reference's np.fromstring call no longer
    exists in NumPy 2, np.frombuffer is the same decode)."""
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import aifc
    try:
        with aifc.open(path, "r") as s:
            n, ch, fs = s.getnframes(), s.getnchannels(), s.getframerate()
            raw = s.readframes(n)
    except Exception as exc:
        raise DecodeError("cannot decode %s: %s" % (path, exc)) from exc
    sig = np.frombuffer(raw, dtype=">i2").astype(np.int16)
    # the reference leaves multi-channel AIFF data interleaved in one vector (:121); keep that
    return fs, sig


def read_audio_generic(path):
    """.mp3 / .au / .ogg through pydub (ffmpeg), like audioBasicIO.py:130-153; raises when pydub is missing."""
    try:
        from pydub import AudioSegment
    except Exception as exc:
        raise DecodeError("%s needs pydub + ffmpeg to decode (as in the reference); not installed here" % path) from exc
    try:
        a = AudioSegment.from_file(path)
    except Exception as exc:
        raise DecodeError("cannot decode %s: %s" % (path, exc)) from exc
    if a.sample_width == 2:
        data = np.frombuffer(a._data, np.int16)
    elif a.sample_width == 4:
        data = np.frombuffer(a._data, np.int32)
    else:
        raise DecodeError("unsupported sample width in " + path)
    return a.frame_rate, np.stack([data[c::a.channels] for c in range(a.channels)], axis=1)


def read_audio_file(path):
    """(sampling_rate, signal) like audioBasicIO.read_audio_file (:86-110)."""
    ext = os.path.splitext(path)[1].lower()
    if ext in (".aif", ".aiff"):
        fs, sig = read_aif(path)
    elif ext == ".wav":
        from scipy.io import wavfile
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            fs, sig = wavfile.read(path)
    elif ext in (".mp3", ".au", ".ogg"):
        fs, sig = read_audio_generic(path)
    else:
        raise DecodeError("unknown audio file type " + ext)
    if sig.ndim == 2 and sig.shape[1] == 1:
        sig = sig.flatten()
    return fs, sig


class PinnedBatch:
    """[n, n_samples] int16 page-locked staging buffer filled file by file (``read_wav_into`` when the file is mono PCM16
    of the right length, decode + copy otherwise) and uploaded with one H2D copy."""

    def __init__(self, n, n_samples):
        from .hostpipe import PinnedArray
        self._buf = PinnedArray((n, n_samples), np.int16)
        self.array = self._buf.array
        self.direct = 0                 # files decoded without an intermediate copy

    def fill(self, i, path, decoded=None, n=None):
        """Row ``i`` <- the file's samples.  ``n``: the file has that many samples (a ragged batch): they go to
        ``array[i, :n]`` and the rest of the row is zeroed."""
        row = self.array[i] if n is None else self.array[i, :n]
        if n is not None:
            self.array[i, n:] = 0
        if decoded is None and read_wav_into(path, row) is not None:
            self.direct += 1
            return
        if decoded is None:
            decoded = stereo_to_mono(read_audio_file(path)[1])
        row[...] = decoded

    def to_device(self):
        import torch
        return torch.from_numpy(self.array).cuda(non_blocking=True)

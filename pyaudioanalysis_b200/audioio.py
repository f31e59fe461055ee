"""File decode in front of the GPU path (SURVEY 8f rank 2): the reference's ``audioBasicIO.read_audio_file`` (:86-110) and
``stereo_to_mono`` (:156-168), plus the device decode: the data chunks of PCM 8 / 16 / 24 / 32-bit and float 32 / 64 WAV
files, mono or stereo (``wav_pcm_layout``), are read STRAIGHT INTO one page-locked byte arena, copied to the GPU once and
converted + downmixed there by ``b200aa_decode_pcm`` (``stage``, ``load_batch``), bit for bit what the host decode
stages; nothing decoded stays in host memory.  ``read_wav_into`` / ``PinnedBatch`` read mono PCM16 into an int16
staging buffer.  Formats: .wav (own RIFF walk for the flavours above, scipy for everything else wavfile.read
understands), .aif / .aiff (stdlib ``aifc``, big-endian 16-bit like the reference), .mp3 / .au / .ogg through pydub when
it is installed (as in the reference); undecodable files raise instead of being skipped silently.
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


class _Walk:
    """The chunks of a RIFF/WAVE file: (id, declared size, body offset, body bytes for 'fmt ' else None) in file order,
    the RIFF header's end (declared size + 8), the file's length, and how many bytes the first incomplete chunk header
    had (0: the walk ended exactly at the end of the file)."""
    __slots__ = ("chunks", "riff_end", "file_len", "tail")


def _riff_walk(path):
    """One walk over every chunk header of a RIFF/WAVE file (bodies other than 'fmt ' are seeked over, an odd-sized chunk
    is followed by its pad byte), or None when the file cannot be opened or is not RIFF/WAVE."""
    try:
        with open(path, "rb") as f:
            head = f.read(12)
            if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
                return None
            w = _Walk()
            w.chunks, w.riff_end, w.file_len = [], struct.unpack("<I", head[4:8])[0] + 8, os.fstat(f.fileno()).st_size
            while True:
                ck = f.read(8)
                if len(ck) < 8:
                    w.tail = len(ck)
                    return w
                cid, size = ck[:4], struct.unpack("<I", ck[4:])[0]
                if cid == b"fmt ":
                    w.chunks.append((cid, size, f.tell(), f.read(size + (size & 1))))
                else:
                    w.chunks.append((cid, size, f.tell(), None))
                    f.seek(size + (size & 1), 1)
    except OSError:
        return None


def _pcm16_of(w):
    """wav_pcm16_layout of a walk: the last 'fmt ' chunk before the first 'data' chunk decides."""
    fmt = None
    for cid, size, off, body in w.chunks:
        if cid == b"fmt ":
            tag, ch, fs, _, _, bits = struct.unpack("<HHIIHH", body[:16])
            if tag == 0xFFFE and size >= 26:                      # WAVE_FORMAT_EXTENSIBLE: sub-format GUID starts with the tag
                tag = struct.unpack("<H", body[24:26])[0]
            fmt = (tag, ch, fs, bits)
        elif cid == b"data":
            if fmt is None or fmt[0] != 1 or fmt[3] != 16 or fmt[1] < 1:
                return None
            tag, ch, fs, bits = fmt
            size = min(size, w.file_len - off)
            return fs, ch, size // (2 * ch), off
    return None


def wav_pcm16_layout(path):
    """(sampling_rate, channels, n_frames, data_offset) of a plain 16-bit PCM RIFF/WAVE file, or None for anything else
    (float / 24-bit / extensible sub-formats other than PCM / RF64 ...: left to scipy)."""
    w = _riff_walk(path)
    try:
        return None if w is None else _pcm16_of(w)
    except struct.error:
        return None


# data-chunk formats of the device decode (include/b200aa.h B200AA_PCM_*): (format tag, bits per sample) -> code
PCM_U8, PCM_S16, PCM_S24, PCM_S32, PCM_F32, PCM_F64 = range(6)
PCM_SAMPLE_BYTES = (1, 2, 3, 4, 4, 8)
_PCM_CODES = {(1, 8): PCM_U8, (1, 16): PCM_S16, (1, 24): PCM_S24, (1, 32): PCM_S32, (3, 32): PCM_F32, (3, 64): PCM_F64}
_GUID_TAIL = b"\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"      # {XXXXXXXX-0000-0010-8000-00AA00389B71}


def _pcm_of(w):
    """The strict rule of wav_pcm_layout for every flavour but mono PCM16: exactly one 'fmt ' and one 'data' chunk,
    both inside the RIFF header's size, every chunk header there complete, and a complete data chunk that scipy reads
    in full -- a file scipy would read differently or refuse is left to it."""
    seen = [(cid, size, off, body) for cid, size, off, body in w.chunks if off - 8 < w.riff_end]
    if w.tail and w.file_len - w.tail < w.riff_end:
        return None
    fmts = [k for k, c in enumerate(seen) if c[0] == b"fmt "]
    datas = [k for k, c in enumerate(seen) if c[0] == b"data"]
    if len(fmts) != 1 or len(datas) != 1 or fmts[0] > datas[0]:
        return None
    _, fsize, _, body = seen[fmts[0]]
    if fsize < 16 or len(body) < fsize:
        return None
    tag, ch, fs, bytes_per_s, block_align, bits = struct.unpack("<HHIIHH", body[:16])
    if tag == 0xFFFE:                                           # WAVE_FORMAT_EXTENSIBLE with a standard sub-format GUID
        if fsize < 40 or struct.unpack("<H", body[16:18])[0] < 22 or body[24:40][4:] != _GUID_TAIL:
            return None
        tag = struct.unpack("<I", body[24:28])[0]
    code = _PCM_CODES.get((tag, bits))
    if code is None or ch not in (1, 2) or block_align != ch * bits // 8 or (code == PCM_S16 and ch == 1):
        return None
    if tag == 1 and bytes_per_s != fs * block_align:            # scipy raises on this header
        return None
    _, size, off, _ = seen[datas[0]]
    if size % block_align or off + size > w.file_len:
        return None
    return fs, ch, size // block_align, off, code


def wav_pcm_layout(path):
    """(sampling_rate, channels, n_frames, data_offset, format) of a WAV file whose data chunk the device decode reads
    as it lies on disk (format: PCM_U8 .. PCM_F64), or None for anything else, which stays with scipy.

    Accepted: PCM 8 / 16 / 24 / 32-bit (format tag 1) and IEEE float 32 / 64-bit (tag 3), also as
    WAVE_FORMAT_EXTENSIBLE sub-formats, 1 or 2 channels, block_align == channels * bits / 8.  Mono PCM16 is accepted
    exactly when ``wav_pcm16_layout`` accepts it (a truncated data chunk is clamped to the file); every other flavour
    needs a complete data chunk whose size is a multiple of block_align and the header checks scipy makes.  n_frames is
    the length ``scipy.io.wavfile.read`` returns."""
    w = _riff_walk(path)
    if w is None:
        return None
    try:
        lay = _pcm16_of(w)
        if lay is not None and lay[1] == 1:
            return lay + (PCM_S16,)
        return _pcm_of(w)
    except struct.error:
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


# b200aa_pcm_clip (include/b200aa.h)
_PCM_CLIP = np.dtype([("offset", "<i8"), ("n_frames", "<i8"), ("format", "<i4"), ("channels", "<i4")])


def stage(clips):
    """Clips of one staged format -> ([B, N] CUDA tensor, int64 CUDA lengths [B]), N the longest clip; row b holds clip
    b's samples and zeros after them.  A clip is anything with ``path``, ``n``, ``data`` and ``layout``: with ``data``
    None its file's data chunk (``layout`` = (data_offset, format, channels) of ``wav_pcm_layout``) is read with
    ``readinto`` straight into a page-locked byte arena, else ``data`` (a decoded 1-D int16 / float32 array) is copied
    there.  One H2D copy of the arena and one ``b200aa_decode_pcm`` launch convert and downmix every clip on the device,
    bit for bit what ``_as_clip(stereo_to_mono(read_audio_file(path)[1]))`` gives on the host."""
    import torch
    from ._lib import lib, check, DTYPE_I16, DTYPE_F32
    from .hostpipe import PinnedArray
    desc = np.zeros(len(clips), dtype=_PCM_CLIP)
    nbytes = []
    off = 0
    for k, c in enumerate(clips):
        if c.data is None:
            fmt, ch = c.layout[1], c.layout[2]
        else:
            fmt, ch = (PCM_S16 if c.data.dtype == np.int16 else PCM_F32), 1
        nb = c.n * ch * PCM_SAMPLE_BYTES[fmt]
        desc[k] = (off, c.n, fmt, ch)
        nbytes.append(nb)
        off += (nb + 15) // 16 * 16
    int16 = all(ch == 1 and fmt in (PCM_U8, PCM_S16) for fmt, ch in zip(desc["format"], desc["channels"]))
    n_max = max((c.n for c in clips), default=0)
    arena = PinnedArray((max(off, 16),), np.uint8)
    buf = arena.array
    for k, c in enumerate(clips):
        o, nb = int(desc[k]["offset"]), nbytes[k]
        if c.data is None:
            with open(c.path, "rb", buffering=0) as f:
                f.seek(c.layout[0])
                got = f.readinto(memoryview(buf[o:o + nb]))
            if got != nb:
                raise DecodeError("short read in " + c.path)
        else:
            buf[o:o + nb] = np.ascontiguousarray(c.data).view(np.uint8)
        buf[o + nb:o + (nb + 15) // 16 * 16] = 0
    out = torch.empty((len(clips), n_max), dtype=torch.int16 if int16 else torch.float32, device="cuda")
    lengths = torch.tensor([c.n for c in clips], dtype=torch.int64).cuda()
    d_arena = torch.from_numpy(buf).cuda(non_blocking=True)
    stream = torch.cuda.current_stream()
    check(lib().b200aa_decode_pcm(d_arena.data_ptr(), buf.size, desc.ctypes.data, len(clips),
                                  DTYPE_I16 if int16 else DTYPE_F32, out.data_ptr(), n_max, n_max, stream.cuda_stream))
    stream.synchronize()                # the arena is released on return
    return out, lengths


def load_batch(paths):
    """Decode a list of audio files on the GPU: (sampling_rate, signals CUDA [B, N], lengths int64 CUDA [B]), row b the
    first lengths[b] samples of ``stereo_to_mono(read_audio_file(paths[b])[1])`` as the feature path stages it (int16 for
    mono 8 / 16-bit PCM, float32 otherwise), zeros after.  WAV files ``wav_pcm_layout`` accepts are read straight from
    disk and decoded on the device (``stage``); other files are decoded on the host first.  Files of different sampling
    rates or staged formats raise ValueError.  The result is what ``mid_feature_extraction_batch(..., lengths=)`` takes."""
    from .MidTermFeatures import _open_clip
    clips = [_open_clip(p) for p in paths]
    if not clips:
        raise ValueError("load_batch needs at least one file")
    kinds = {(c.fs, c.code) for c in clips}
    if len(kinds) > 1:
        raise ValueError("files of different sampling rates or sample formats: %s" % sorted(kinds))
    sig, lengths = stage(clips)
    return clips[0].fs, sig, lengths

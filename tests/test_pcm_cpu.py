"""CPU: the device decode of WAV data chunks without a device.

* The per-frame conversion of csrc/pcm.cuh, run on the host by tests/pcm_host.cu over the raw payload of every one of the
  12 (format, channels) flavours, equals ``_as_clip(stereo_to_mono(read_audio_file(path)[1]))`` bit for bit (NaN: only
  NaN-ness), on rails, 24-bit and 32-bit extremes, float32 subnormals and their halves, signed zeros, infinities, float64
  values beyond the float32 range, rounding ties and random payloads.
* ``audioio.wav_pcm_layout`` accepts exactly the files the device decode reads as they lie on disk, with scipy's length,
  and a lazily opened ``_Clip`` has the sampling rate, length and staged format of today's host decode.
* Every argument error of ``b200aa_decode_pcm`` returns B200AA_ERR_INVALID before any CUDA call.
"""
import subprocess

import numpy as np
import pytest

from pyaudioanalysis_b200 import audioio
from pyaudioanalysis_b200.MidTermFeatures import _open_clip
from pyaudioanalysis_b200.ShortTermFeatures import _as_clip
from tests import host_exe
from tests import wavgen

INVALID = -1


def host_staged(path):
    """What the wrappers stage for a file on the host path: (fs, 1-D int16 / float32 array)."""
    fs, x = audioio.read_audio_file(path)
    with np.errstate(all="ignore"):                 # inf - inf, float64 beyond the float32 range
        return fs, _as_clip(audioio.stereo_to_mono(x))[0]


def same_bits(got, ref):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.dtype == ref.dtype and got.shape == ref.shape, (got.dtype, ref.dtype, got.shape, ref.shape)
    if got.dtype == np.float32:
        nan = np.isnan(ref)
        assert (np.isnan(got) == nan).all(), "NaN positions differ"
        bad = np.nonzero(got.view(np.uint32)[~nan] != ref.view(np.uint32)[~nan])[0]
    else:
        bad = np.nonzero(got != ref)[0]
    return bad


# ------------------------------------------------------------------------------------------------------------ conversion
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "pcm_host.cu", "-O1")


def host_convert(exe, tmp_path, path):
    """Run pcm_host over the raw data chunk of a file wav_pcm_layout accepts."""
    fs, ch, n, off, fmt = audioio.wav_pcm_layout(path)
    block = ch * audioio.PCM_SAMPLE_BYTES[fmt]
    raw = open(path, "rb").read()[off:off + n * block]
    src, dst = str(tmp_path / "payload.bin"), str(tmp_path / "out.bin")
    open(src, "wb").write(raw)
    int16 = ch == 1 and fmt in (audioio.PCM_U8, audioio.PCM_S16)
    res = subprocess.run([exe, str(fmt), str(ch), str(n), "0" if int16 else "1", src, dst], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return np.fromfile(dst, dtype=np.int16 if int16 else np.float32)


@pytest.mark.parametrize("name,channels", wavgen.FLAVOURS)
def test_conversion_matches_host_decode(exe, tmp_path, name, channels):
    p = str(tmp_path / ("%s_%d.wav" % (name, channels)))
    wavgen.write(p, 16000, wavgen.flavour_samples(name, channels, 11 + channels), name)
    _, ref = host_staged(p)
    got = host_convert(exe, tmp_path, p)
    bad = same_bits(got, ref)
    assert bad.size == 0, "%s x %d: %d frames differ, first %d: %r vs %r" % (name, channels, bad.size, bad[0], got[bad[0]],
                                                                           ref[bad[0]])


# ---------------------------------------------------------------------------------------------------------------- parser
def _case_files(d):
    """(file name, bytes, accepted by wav_pcm_layout) of the parser cases."""
    rng = np.random.default_rng(5)
    out = []
    for name, ch in wavgen.FLAVOURS:
        code, tag, bits = wavgen.FORMATS[name]
        for n in (0, 1, 777, 1001):
            x = wavgen.signal(name, ch, n, seed=n + 3 * code + ch)
            pay = wavgen.encode(x, name)
            base = "%s_%d_%d" % (name, ch, n)
            out.append((base + ".wav", wavgen.wav_bytes(16000, pay, ch, tag, bits), True))
            if n != 777:
                continue
            out.append((base + "_ext.wav", wavgen.wav_bytes(22050, pay, ch, tag, bits, extensible=True), True))
            out.append((base + "_chunks.wav", wavgen.wav_bytes(8000, pay, ch, tag, bits, before=[
                (b"LIST", b"INFOabcde"), (b"fact", b"\x01\x02\x03\x04"), (b"JUNK", b"xyz")],
                after=[(b"LIST", b"odd")]), True))
            mono16 = name == "s16" and ch == 1
            out.append((base + "_trunc.wav", wavgen.wav_bytes(16000, pay, ch, tag, bits, cut=5), mono16))
            out.append((base + "_nonmult.wav", wavgen.wav_bytes(16000, pay + b"\x00", ch, tag, bits),
                        mono16 or (name == "u8" and ch == 1)))
            out.append((base + "_long.wav", wavgen.wav_bytes(16000, pay, ch, tag, bits, data_size=len(pay) + 64), mono16))
            out.append((base + "_rifx.wav", wavgen.wav_bytes(16000, pay, ch, tag, bits, riff=b"RIFX"), False))
            if mono16:
                continue            # mono PCM16 keeps wav_pcm16_layout's rule (test_layout_keeps_the_pcm16_rule)
            out.append((base + "_twodata.wav", wavgen.wav_bytes(16000, pay, ch, tag, bits, after=[(b"data", pay[:16])]),
                        False))
            out.append((base + "_badguid.wav", wavgen.wav_bytes(16000, pay, ch, tag, bits, extensible=True)
                        .replace(wavgen._GUID_TAIL, b"\x00" * 12), False))
            if tag == 1:
                out.append((base + "_badrate.wav", wavgen.wav_bytes(16000, pay, ch, tag, bits, bytes_per_s=12345), False))
    x3 = rng.integers(-3000, 3000, size=(500, 3))
    out.append(("three.wav", wavgen.wav_bytes(16000, wavgen.encode(x3, "s16"), 3, 1, 16), False))
    out.append(("mulaw.wav", wavgen.wav_bytes(8000, bytes(range(200)), 1, 7, 8), False))
    out.append(("int12.wav", wavgen.wav_bytes(16000, wavgen.encode(rng.integers(-2048, 2048, 300) * 16, "s16"), 1, 1, 12,
                                              block_align=2), False))
    out.append(("padded24.wav", wavgen.wav_bytes(16000, wavgen.encode(rng.integers(-2 ** 20, 2 ** 20, 300), "s32"), 1, 1,
                                                 20, block_align=4), False))
    return out


def test_layout_accepts_exactly_the_device_flavours(tmp_path):
    from scipy.io import wavfile
    import warnings
    for fname, raw, accepted in _case_files(tmp_path):
        p = str(tmp_path / fname)
        open(p, "wb").write(raw)
        lay = audioio.wav_pcm_layout(p)
        assert (lay is not None) == accepted, fname
        if lay is None:
            continue
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            fs, x = wavfile.read(p)
        assert lay[0] == fs and lay[2] == x.shape[0] and lay[1] == (1 if x.ndim == 1 else x.shape[1]), fname
        c = _open_clip(p)
        assert c.data is None and c.layout == (lay[3], lay[4], lay[1]), fname
        hfs, h = host_staged(p)
        code = 0 if h.dtype == np.int16 else 1
        assert (c.fs, c.n, c.code) == (hfs, h.shape[0], code), fname
    assert audioio.wav_pcm_layout(str(tmp_path / "missing.wav")) is None


def test_layout_keeps_the_pcm16_rule(tmp_path):
    """Mono PCM16 is accepted exactly when wav_pcm16_layout accepts it, a truncated data chunk clamped to the file."""
    x = wavgen.signal("s16", 1, 1000, seed=1)
    pay = wavgen.encode(x, "s16")
    p = str(tmp_path / "t.wav")
    open(p, "wb").write(wavgen.wav_bytes(16000, pay, 1, 1, 16, cut=7))
    assert audioio.wav_pcm16_layout(p)[:3] == (16000, 1, (len(pay) - 7) // 2)
    assert audioio.wav_pcm_layout(p) == audioio.wav_pcm16_layout(p) + (audioio.PCM_S16,)
    open(p, "wb").write(wavgen.wav_bytes(16000, pay, 2, 1, 16))
    assert audioio.wav_pcm16_layout(p)[:3] == (16000, 2, 500)           # stereo PCM16: still a pcm16 layout


def test_three_channels_stay_on_the_host_and_raise(tmp_path):
    p = str(tmp_path / "three.wav")
    open(p, "wb").write(wavgen.wav_bytes(16000, wavgen.encode(np.zeros((100, 3), np.int64), "s16"), 3, 1, 16))
    assert audioio.wav_pcm_layout(p) is None
    with pytest.raises(ValueError):
        _open_clip(p)


# ------------------------------------------------------------------------------------------------------- argument errors
@pytest.fixture(scope="module")
def lib():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib.lib()


def test_decode_rejects_bad_arguments(lib):
    p = 256                                    # never dereferenced: every call below fails its argument check first

    def call(clips, arena=p, arena_bytes=1 << 20, n_clips=None, out_dtype=1, out=p, n_out=100, stride=100):
        d = np.array(clips or [], dtype=audioio._PCM_CLIP)
        return lib.b200aa_decode_pcm(arena, arena_bytes, d.ctypes.data if clips else None,
                                     len(d) if n_clips is None else n_clips, out_dtype, out, n_out, stride, None)

    good = (0, 100, audioio.PCM_S16, 2)
    assert call([good], arena=None) == INVALID
    assert call(None, n_clips=1) == INVALID
    assert call([good], out=None) == INVALID
    assert call([good], n_clips=-1) == INVALID
    assert call([good], n_out=-1, stride=10) == INVALID
    assert call([good], stride=99) == INVALID
    assert call([good], arena_bytes=-16) == INVALID
    assert call([good], out_dtype=2) == INVALID
    assert call([good], out_dtype=-1) == INVALID
    for bad in [(0, 100, 6, 1), (0, 100, -1, 1), (0, 100, audioio.PCM_S16, 0), (0, 100, audioio.PCM_S16, 3),
                (8, 10, audioio.PCM_S16, 1), (-16, 10, audioio.PCM_S16, 1), (0, -1, audioio.PCM_F32, 1),
                (0, 101, audioio.PCM_F32, 1),                                  # more frames than the row holds
                (1 << 20, 1, audioio.PCM_U8, 1),                              # slot past the arena
                ((1 << 20) - 1584, 100, audioio.PCM_F64, 2),                 # 1600 bytes of frames, 1584 left
                ((1 << 20) - 16, 6, audioio.PCM_S24, 1)]:                    # 18 bytes of frames, a 32-byte slot
        assert call([good, bad]) == INVALID, bad
    for stereo_or_float in [(0, 10, audioio.PCM_S16, 2), (0, 10, audioio.PCM_U8, 2), (0, 10, audioio.PCM_F32, 1),
                            (0, 10, audioio.PCM_S24, 1), (0, 10, audioio.PCM_S32, 1), (0, 10, audioio.PCM_F64, 1)]:
        assert call([(0, 10, audioio.PCM_U8, 1), stereo_or_float], out_dtype=0) == INVALID, stereo_or_float

"""GPU: the WAV decode kernel (b200aa_decode_pcm) and the directory wrappers that stage every file through it.

* One ragged launch over all 12 (format, channels) flavours, with a 0-frame and a 1-frame clip and 24-bit payloads that
  are not a multiple of 4 or 16 bytes, into a NaN-filled output of odd row stride: exactly [B, N] is written, each row
  bit for bit the host staging of its file (NaN only as NaN) and zero past its length.  Also an int16 launch and a
  70 000-clip batch.
* The wrappers on a folder of every flavour plus an AIFF file give the same results and files as the host decode path
  (``wav_pcm_layout`` patched to accept nothing), and no accepted file keeps a decoded array.
* The reference's own results on seeded files of every format (tests/golden/pcm_formats.npz) hold to the mid-term check.
"""
import os

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import wavgen
from tests.parity import check_mid_propagated

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    pkg.ShortTermFeatures.PRINT_SPECTROGRAM_SHAPE = False
    pkg.MidTermFeatures.VERBOSE = False
    return pkg


def host_staged(path):
    from pyaudioanalysis_b200 import audioio
    from pyaudioanalysis_b200.ShortTermFeatures import _as_clip
    fs, x = audioio.read_audio_file(path)
    with np.errstate(all="ignore"):
        return _as_clip(audioio.stereo_to_mono(x))[0]


def same(got, ref, what):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    if got.dtype.kind == "f":
        nan = np.isnan(ref)
        assert (np.isnan(got) == nan).all(), what + ": NaN positions"
        bits = np.dtype("u%d" % got.dtype.itemsize)
        assert np.array_equal(got[~nan].view(bits), ref[~nan].view(bits)), what
    else:
        assert np.array_equal(got, ref), what


def decode(clips, arena, n_out, stride, out_dtype, fill):
    """Run b200aa_decode_pcm on a host arena and descriptor list into a [B, stride] tensor filled with `fill`."""
    import torch
    from pyaudioanalysis_b200 import audioio
    from pyaudioanalysis_b200._lib import lib
    desc = np.array(clips, dtype=audioio._PCM_CLIP)
    d_arena = torch.from_numpy(arena).cuda()
    out = torch.full((len(clips), stride), fill, dtype=torch.int16 if out_dtype == 0 else torch.float32, device="cuda")
    rc = lib().b200aa_decode_pcm(d_arena.data_ptr(), arena.size, desc.ctypes.data, len(clips), out_dtype, out.data_ptr(),
                                 n_out, stride, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return out.cpu().numpy()


def arena_of(payloads):
    """(arena uint8, offsets): each payload at a 16-byte aligned offset, its slot zero-padded to 16 bytes."""
    offs, off = [], 0
    for p in payloads:
        offs.append(off)
        off += (len(p) + 15) // 16 * 16
    arena = np.zeros(max(off, 16), dtype=np.uint8)
    for o, p in zip(offs, payloads):
        arena[o:o + len(p)] = np.frombuffer(p, dtype=np.uint8)
    return arena, offs


def test_one_ragged_launch_all_flavours(P, tmp_path):
    from pyaudioanalysis_b200 import audioio
    # 0 and 1 frames; 24-bit payloads of 9003 and 17 970 bytes, not a multiple of 4 or 16
    frames = [0, 1, 3000, 2999, 3001, 2995, 2998, 2500, 3000, 2997, 3001, 4000]
    lens, files = {}, []
    for k, (name, ch) in enumerate(wavgen.FLAVOURS):
        x = wavgen.flavour_samples(name, ch, 30 + k)
        assert x.shape[0] >= frames[k]
        p = str(tmp_path / ("%02d_%s_%d.wav" % (k, name, ch)))
        wavgen.write(p, 16000, x[:frames[k]], name)
        files.append(p)
        lens[p] = frames[k]
    payloads, clips = [], []
    for p in files:
        fs, ch, n, off, fmt = audioio.wav_pcm_layout(p)
        assert n == lens[p]
        payloads.append(open(p, "rb").read()[off:off + n * ch * audioio.PCM_SAMPLE_BYTES[fmt]])
        clips.append((0, n, fmt, ch))
    arena, offs = arena_of(payloads)
    clips = [(o,) + c[1:] for o, c in zip(offs, clips)]
    N = max(lens.values())
    stride = N + 3 if (N + 3) % 2 else N + 4
    got = decode(clips, arena, N, stride, 1, float("nan"))
    for b, p in enumerate(files):
        ref = host_staged(p).astype(np.float32)                # mono 8 / 16-bit: the int16 values, exact in float32
        n = lens[p]
        same(got[b, :n], ref, os.path.basename(p))
        assert (got[b, n:N] == 0).all(), os.path.basename(p) + ": zeros past the clip"
        assert np.isnan(got[b, N:]).all(), os.path.basename(p) + ": nothing past n_out"
    # int16 output: mono 8 / 16-bit only
    ints = [k for k, (name, ch) in enumerate(wavgen.FLAVOURS) if ch == 1 and name in ("u8", "s16")]
    got16 = decode([clips[k] for k in ints], arena, N, stride, 0, 0x5A5A)
    for r, k in enumerate(ints):
        n = lens[files[k]]
        same(got16[r, :n], host_staged(files[k]), files[k])
        assert (got16[r, n:N] == 0).all() and (got16[r, N:] == 0x5A5A).all()


def _numpy_decode(raw, fmt, ch):
    """The host staging of a raw data chunk, the way scipy + stereo_to_mono + _as_clip compute it."""
    from pyaudioanalysis_b200.ShortTermFeatures import _as_clip
    from pyaudioanalysis_b200.audioio import stereo_to_mono
    if fmt == 2:
        b = np.frombuffer(raw, np.uint8).reshape(-1, 3)
        x = np.zeros((b.shape[0], 4), np.uint8)
        x[:, 1:] = b
        x = x.view("<i4").reshape(-1)
    else:
        x = np.frombuffer(raw, ("u1", "<i2", None, "<i4", "<f4", "<f8")[fmt])
    x = x.reshape(-1, ch) if ch == 2 else x
    with np.errstate(all="ignore"):
        return _as_clip(stereo_to_mono(x))[0]


def test_seventy_thousand_clips(P):
    rng = np.random.default_rng(70000)
    B = 70000
    fmts = rng.integers(0, 6, B)
    chans = rng.integers(1, 3, B)
    lens = rng.integers(0, 41, B)
    payloads = [rng.integers(0, 256, int(n) * int(c) * (1, 2, 3, 4, 4, 8)[f], dtype=np.uint8).tobytes()
                for f, c, n in zip(fmts, chans, lens)]
    arena, offs = arena_of(payloads)
    N = int(lens.max())
    got = decode([(o, int(n), int(f), int(c)) for o, n, f, c in zip(offs, lens, fmts, chans)], arena, N, N, 1, float("nan"))
    for b in range(B):
        n = int(lens[b])
        same(got[b, :n], _numpy_decode(payloads[b], int(fmts[b]), int(chans[b])).astype(np.float32), "clip %d" % b)
        assert (got[b, n:] == 0).all()


# ------------------------------------------------------------------------------------------------------ wrappers
WIN = (1.0, 1.0, 0.05, 0.05)


def write_mixed_folder(d):
    """Every flavour at 16 kHz (two 8-bit mono files, so int16 chunks mix 8 and 16-bit files), an AIFF file."""
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import aifc
    d.mkdir()
    for k, (name, ch) in enumerate(wavgen.FLAVOURS):
        n = 9000 + 1733 * k
        wavgen.write(str(d / ("%02d_%s_%d.wav" % (k, name, ch))), 16000, wavgen.signal(name, ch, n, 40 + k), name)
    wavgen.write(str(d / "20_u8_1b.wav"), 16000, wavgen.signal("u8", 1, 17001, 99), "u8")
    x = O.synth_clip(41, 15000, 16000)
    with aifc.open(str(d / "30_t.aiff"), "wb") as a:
        a.setnchannels(1)
        a.setsampwidth(2)
        a.setframerate(16000)
        a.writeframes(x.astype(">i2").tobytes())


def _equal(a, b, what):
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for k, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, "%s[%d]" % (what, k))
        return
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        assert a.shape == b.shape and a.dtype == b.dtype, what
        assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f"), what
        return
    assert a == b, what


def test_wrappers_unchanged(P, tmp_path, monkeypatch):
    from pyaudioanalysis_b200 import audioio
    M = P.MidTermFeatures
    src = tmp_path / "mix"
    write_mixed_folder(src)
    other = tmp_path / "other"
    other.mkdir()
    for k, (name, ch) in enumerate(wavgen.FLAVOURS[::3]):
        wavgen.write(str(other / ("o%d.wav" % k)), 16000, wavgen.signal(name, ch, 12000 + 999 * k, 70 + k), name)
    clips = M._folder_clips(str(src))
    wav = [c for c in clips if c.path.endswith(".wav")]
    assert len(wav) == 13 and all(c.data is None and c.layout is not None for c in wav), "every WAV flavour opens lazily"
    assert all(c.data is not None for c in clips if not c.path.endswith(".wav"))

    def run(tag):
        out = {"dfe_beat": M.directory_feature_extraction(str(src), *WIN, compute_beat=True),
               "dfe": M.directory_feature_extraction(str(src), *WIN, compute_beat=False),
               "multi": M.multiple_directory_feature_extraction([str(src), str(other)], *WIN, compute_beat=True),
               "no_avg": M.directory_feature_extraction_no_avg(str(src), 1.0, 0.5, 0.05, 0.025)}
        d = tmp_path / ("files_" + tag)
        d.mkdir()
        import shutil
        for f in sorted(os.listdir(str(src))):
            if f.endswith(".wav"):
                shutil.copy(str(src / f), str(d / f))
        M.mid_feature_extraction_file_dir(str(d), *WIN, store_short_features=True, store_csv=True)
        out["files"] = {f: open(str(d / f), "rb").read() for f in sorted(os.listdir(str(d))) if not f.endswith(".wav")}
        return out

    device = run("device")
    monkeypatch.setattr(audioio, "wav_pcm_layout", lambda path: None)
    host = run("host")
    monkeypatch.undo()
    for key in ("dfe_beat", "dfe", "multi", "no_avg"):
        _equal(device[key], host[key], key)
    assert sorted(device["files"]) == sorted(host["files"]) and len(device["files"]) == 13 * 4
    for f in device["files"]:
        assert device["files"][f] == host["files"][f], f


def test_three_channels_still_raise(P, tmp_path):
    d = tmp_path / "three"
    d.mkdir()
    wavgen.write(str(d / "a.wav"), 16000, wavgen.signal("s16", 2, 9000, 1), "s16")
    x3 = np.stack([wavgen.signal("s16", 1, 9000, s) for s in (2, 3, 4)], axis=1)
    wavgen.write(str(d / "b.wav"), 16000, x3, "s16")
    with pytest.raises(ValueError, match="one-dimensional"):
        P.MidTermFeatures.directory_feature_extraction(str(d), *WIN)


def test_load_batch(P, tmp_path):
    from pyaudioanalysis_b200 import audioio
    paths = []
    for k, (name, ch) in enumerate([("s24", 2), ("f32", 1), ("s16", 2), ("f64", 1)]):
        paths.append(str(tmp_path / ("l%d.wav" % k)))
        wavgen.write(paths[-1], 22050, wavgen.signal(name, ch, 5000 + 77 * k, k), name)
    fs, sig, lengths = P.load_batch(paths)
    assert fs == 22050 and sig.dtype.is_floating_point and lengths.tolist() == [5000 + 77 * k for k in range(4)]
    s = sig.cpu().numpy()
    for b, p in enumerate(paths):
        n = int(lengths[b])
        same(s[b, :n], host_staged(p), p)
        assert (s[b, n:] == 0).all()
    wavgen.write(str(tmp_path / "m.wav"), 22050, wavgen.signal("u8", 1, 3000, 5), "u8")
    with pytest.raises(ValueError):
        P.load_batch(paths + [str(tmp_path / "m.wav")])            # int16-staged next to float32-staged
    wavgen.write(str(tmp_path / "r.wav"), 16000, wavgen.signal("f32", 1, 3000, 5), "f32")
    with pytest.raises(ValueError):
        P.load_batch(paths + [str(tmp_path / "r.wav")])            # another sampling rate
    assert audioio.load_batch is P.load_batch


def test_reference_goldens(P, tmp_path):
    """Files of every format against the unmodified reference's read_audio_file + stereo_to_mono +
    mid_feature_extraction (oracle/make_golden_pcm.py), through the device decode."""
    from oracle import make_golden_pcm as G
    from tests.conftest import load_golden
    g = load_golden("pcm_formats.npz")
    M = P.MidTermFeatures
    paths = G.write_files(str(tmp_path))
    clips = [M._open_clip(p) for p in paths.values()]
    assert all(c.data is None for c in clips)
    res = M._mid_per_clip(clips, G.MID_WINDOW / G.FS, G.MID_STEP / G.FS, G.WINDOW / G.FS, G.STEP / G.FS, want_short=True)
    ratio, stepr = O.mid_ratios(G.MID_WINDOW, G.MID_STEP, G.WINDOW, G.STEP)
    for stem, (mid, st, _) in zip(paths, res):
        check_mid_propagated(mid, st, g[stem + "_st"], ratio, stepr, G.WINDOW // 2, stem, ref_mid=g[stem + "_mid"])

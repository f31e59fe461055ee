"""Golden mid-term results of the UNMODIFIED reference on WAV files of the flavours the device decode reads (run where the
reference tree exists):

    python -m oracle.make_golden_pcm

* pcm_formats.npz -- for every file of FILES (written by tests/wavgen.py from its seed: stereo 16-bit, 8-bit, 24-bit,
  32-bit, float32 and float64 files, 16 kHz), the reference's audioBasicIO.read_audio_file + stereo_to_mono +
  MidTermFeatures.mid_feature_extraction(x, fs, MID_WINDOW, MID_STEP, WINDOW, STEP): keys <file>_mid [136, M] and
  <file>_st [68, T], float64.  The files themselves are not stored; the tests regenerate them with ``write_files``.
"""
import os
import sys
import tempfile
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "pcm_formats.npz")
sys.path.insert(0, ROOT)

FS = 16000
MID_WINDOW, MID_STEP, WINDOW, STEP = 8000, 4000, 800, 400
# file stem -> (wavgen format, channels, frames, seed)
FILES = {"s16_stereo": ("s16", 2, 21111, 1), "u8_mono": ("u8", 1, 20000, 2), "u8_stereo": ("u8", 2, 19001, 3),
         "s24_mono": ("s24", 1, 22222, 4), "s24_stereo": ("s24", 2, 20001, 5), "s32_stereo": ("s32", 2, 20500, 6),
         "f32_mono": ("f32", 1, 18000, 7), "f32_stereo": ("f32", 2, 23333, 8), "f64_stereo": ("f64", 2, 19999, 9)}


def write_files(d):
    """Write FILES into directory d; returns {stem: path}."""
    from tests import wavgen
    out = {}
    for stem, (name, ch, n, seed) in FILES.items():
        out[stem] = os.path.join(d, stem + ".wav")
        wavgen.write(out[stem], FS, wavgen.signal(name, ch, n, seed, FS), name)
    return out


def main():
    from oracle.ref_import import load_reference
    _, M, A = load_reference()
    g = {}
    with tempfile.TemporaryDirectory() as d:
        for stem, path in write_files(d).items():
            fs, x = A.read_audio_file(path)
            x = A.stereo_to_mono(x)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)
                mid, st, _ = M.mid_feature_extraction(x, fs, MID_WINDOW, MID_STEP, WINDOW, STEP)
            g[stem + "_mid"] = np.asarray(mid, dtype=np.float64)
            g[stem + "_st"] = np.asarray(st, dtype=np.float64)
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()

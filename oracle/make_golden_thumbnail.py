"""Golden music-thumbnail results of the UNMODIFIED reference (run where the reference tree exists):

    python -m oracle.make_golden_thumbnail

The reference's audioSegmentation imports hmmlearn and matplotlib at module level, so self_similarity_matrix and
music_thumbnailing are executed from its source text (as in make_golden_hmm.py), with the reference's own
audioBasicIO, scipy and scikit-learn.

Writes tests/golden/thumbnail.npz:
- stub cases (tests/thumb_cases.STUB_CASES): stf.feature_extraction replaced by a stub that returns the case's seeded
  matrix <c>_st [F, T]; music_thumbnailing's four times <c>_times, its masked matrix <c>_C, and the name of the exception
  it raised (<c>_error, '' for none).  <c>_S is self_similarity_matrix(<c>_st) for the cases of at most 70 frames;
- end-to-end cases with the reference's own features (int16 signals at 16 kHz): doremi (the signal of doremi.npz) at a
  2 s thumbnail and a 0.25 s step, and at the defaults; the planted-repeat track (thumb_cases.planted_track), mono and
  stereo; a clip shorter than one window.  e2e_<c>_times and e2e_<c>_error.
"""
import os

import numpy as np

from oracle.ref_import import REFERENCE_ROOT, load_reference
from tests.thumb_cases import STUB_CASES, planted_track, stub_features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "thumbnail.npz")
REF = os.path.join(REFERENCE_ROOT, "pyAudioAnalysis")


def reference_env(stf):
    import scipy
    import scipy.signal  # noqa: F401  (music_thumbnailing calls scipy.signal.convolve2d)
    from scipy.spatial import distance
    from sklearn.preprocessing import StandardScaler
    _, _, audio_basic_io = load_reference()
    env = {"np": np, "scipy": scipy, "distance": distance, "StandardScaler": StandardScaler,
           "audioBasicIO": audio_basic_io, "stf": stf}
    src = open(os.path.join(REF, "audioSegmentation.py")).read()
    for start, stop in (("def self_similarity_matrix", "def labels_to_segments"),
                        ("def music_thumbnailing", "\nif __name__")):
        a = src.index(start)
        b = src.find(stop, a)
        exec(src[a:b if b >= 0 else len(src)], env)
    return env


class Stub:
    def __init__(self, st):
        self.st = st

    def feature_extraction(self, signal, sampling_rate, window, step):
        return self.st.copy(), []


def _run(fn, *args, **kw):
    try:
        return fn(*args, **kw), ""
    except Exception as e:          # the golden records the reference's exception by name
        return None, type(e).__name__


def main():
    out = {}
    for name, (F, T, step, thumb, l1, l2, _) in STUB_CASES.items():
        st = stub_features(name)
        env = reference_env(Stub(st))
        out[name + "_st"] = st
        res, err = _run(env["music_thumbnailing"], np.zeros(16000, dtype=np.int16), 16000, 1.0, step, thumb, l1, l2)
        out[name + "_error"] = np.array(err)
        if res is not None:
            out[name + "_times"] = np.array(res[:4], dtype=np.float64)
            out[name + "_C"] = res[4]
            assert all(type(t) is np.float64 for t in res[:4]), name
        S, err = _run(env["self_similarity_matrix"], st)
        if S is not None and T <= 70:
            out[name + "_S"] = S
    stf, _, _ = load_reference()
    env = reference_env(stf)
    doremi = np.load(os.path.join(ROOT, "tests", "golden", "doremi.npz"))["x"]
    e2e = {"doremi_short": (doremi, dict(short_step=0.25, thumb_size=2.0)),
           "doremi": (doremi, {}),
           "planted": (planted_track(), {}),
           "planted_stereo": (planted_track(channels=2), {}),
           "no_frames": (doremi[:8000], {})}
    for name, (x, kw) in e2e.items():
        res, err = _run(env["music_thumbnailing"], x, 16000, **kw)
        out["e2e_%s_error" % name] = np.array(err)
        if res is not None:
            out["e2e_%s_times" % name] = np.array(res[:4], dtype=np.float64)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
    for name in list(STUB_CASES) + ["e2e_" + n for n in e2e]:
        print(name, out.get(name + "_times"), out[name + "_error"])


if __name__ == "__main__":
    main()

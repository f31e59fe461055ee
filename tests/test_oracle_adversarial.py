"""CPU: the oracle against the UNMODIFIED reference on the adversarial signal bank (tests/signals.py).

The reference's outputs are stored as fingerprints (tests/test_oracle_vs_reference.fingerprint) in
tests/golden/adversarial.npz; oracle/make_golden_adversarial.py regenerates them where the reference tree exists.
Constant frames are noise-defined in the reference (float64 round-off through log10(. + eps)): both sides get the exact
DC-only values in those rows (signals.patch_noise_defined) before the fingerprint is taken.
"""
import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.conftest import load_golden
from tests.test_oracle_vs_reference import check_fingerprint

# (fs, window, hop, deltas, with spectrogram / chromagram, with the float32 variants)
CONFIGS = [(16000, 800, 400, True, True, True), (44100, 882, 441, False, True, False),
           (16000, 400, 160, True, False, False), (16000, 800, 333, False, False, False)]


def config_inputs(fs, w, s, floats):
    b = dict(SG.bank(fs, w, s))
    if floats:
        b.update(SG.float_bank(fs, w, s))
    return b


def as_reference_input(x):
    """float32 clips reach the reference as float64 (the values are exact)."""
    return x.astype(np.float64) if x.dtype == np.float32 else x


def key(fs, w, s, name, what):
    return "%d_%d_%d_%s_%s" % (fs, w, s, name, what)


@pytest.fixture(scope="module")
def ADV():
    return load_golden("adversarial.npz")


@pytest.mark.parametrize("fs,w,s,deltas,rows,floats", CONFIGS)
def test_oracle_matches_reference_on_bank(ADV, fs, w, s, deltas, rows, floats):
    for name, x in config_inputs(fs, w, s, floats).items():
        xx = as_reference_input(x)
        F, _ = O.feature_extraction(xx, fs, w, s, deltas=deltas)
        F, _ = SG.patch_noise_defined(F, x, w, s)
        check_fingerprint(F, ADV, key(fs, w, s, name, "st"), rtol=1e-9, atol=1e-12)
        if rows:
            check_fingerprint(O.spectrogram(xx, fs, w, s)[0], ADV, key(fs, w, s, name, "sp"), rtol=1e-9, atol=1e-12)
            check_fingerprint(O.chromagram(xx, fs, w, s)[0], ADV, key(fs, w, s, name, "ch"), rtol=1e-9, atol=1e-12)


def test_bank_properties():
    """What each signal is built to contain is really there."""
    for fs, w, s in ((16000, 800, 400), (16000, 800, 200), (44100, 882, 441), (8000, 600, 300)):
        b = SG.bank(fs, w, s)
        lengths = [x.size for x in b.values()]
        assert len(set(lengths)) == len(lengths), "the batch must be ragged"
        assert all(x.dtype == np.int16 for x in b.values())
        assert int(b["integer_mean"].astype(np.int64).sum()) % b["integer_mean"].size == 0
        assert (b["integer_mean"] == b["integer_mean"].astype(np.int64).sum() // b["integer_mean"].size).mean() > 0.35
        assert int(b["triangle"].astype(np.int64).sum()) == 0
        assert (b["rails"] == -32768).any() and (b["rails"] == 32767).any()
        # energies of frames: loud and quiet frames meet in pairs (2q, 2q + 1) in both orders, 70 dB apart or more
        x = b["loud_quiet"].astype(np.float64)
        T = O.frame_count(x.size, w, s)
        e = np.array([np.mean(x[t * s:t * s + w] ** 2) for t in range(T)])
        loud = e > 1e6
        assert (e[~loud] < 1e-7 * e[loud].min()).all()
        pairs = [(loud[2 * q], loud[2 * q + 1]) for q in range(T // 2)]
        assert (True, False) in pairs and (False, True) in pairs
        # constant frames exist, and frames with a single differing sample at their first / middle / last position
        c = b["constant_runs"]
        bad = SG.noise_defined_frames(c, w, s)
        assert bad.sum() >= 3
        where = {0: 0, w // 2: 0, w - 1: 0}
        for t in np.nonzero(~bad)[0]:
            fr = c[t * s:t * s + w]
            vals, counts = np.unique(fr, return_counts=True)
            if len(vals) == 2 and counts.min() == 1:
                p = int(np.nonzero(fr == vals[np.argmin(counts)])[0][0])
                if p in where:
                    where[p] += 1
        assert all(v > 0 for v in where.values()), where
        # impulses on first and last samples of frames
        imp = b["edge_impulses"]
        assert (np.abs(imp[s * np.arange(0, T, 5)]) == 20000).all()
        assert (np.abs(imp[s * np.arange(2, T, 5) + w - 1]) == 20000).all()

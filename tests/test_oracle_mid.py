"""CPU: the oracle's mid-term pooling against the UNMODIFIED reference where its window ratio is unusual.

The reference's ratio is round((mid_window - (short_window - short_step)) / short_step) (MidTermFeatures.py:100-101).
A mid-term window shorter than one short-term step makes it 0 or negative, and the reference still pools: its windows
are Python slices, so ratio 0 gives empty windows (mean / std of nothing: NaN, then 0 through np.nan_to_num) and
ratio -1 makes the first window every frame but the last and every later window empty.  tests/golden/mid_edges.npz holds
the reference's mid-term matrices (oracle/make_golden_mid.py); tests/test_gpu_mid.py holds the GPU to the same values.
"""
import warnings

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.conftest import load_golden

FS, W, S = 16000, 800, 400
SIGNALS = ("loud_quiet", "chirp")
# name -> (mid_window, mid_step) in samples, with the (ratio, step ratio) the reference derives from them
CASES = {
    "ratio_0": (400, 800, 0, 2),
    "ratio_minus_1": (0, 800, -1, 2),
    "tie_half_to_0": (600, 800, 0, 2),          # 0.5 rounds to even: 0
    "tie_3_halves_to_2": (1000, 800, 2, 2),     # 1.5 rounds to even: 2
    "longer_than_clip": (32000, 16000, 79, 40),
    "step_above_ratio": (1200, 2000, 2, 5),
}


def key(signal, case, what):
    return "%s_%s_%s" % (signal, case, what)


def clip(signal):
    return SG.bank(FS, W, S)[signal]


@pytest.fixture(scope="module")
def MID():
    return load_golden("mid_edges.npz")


def test_case_ratios():
    for name, (mw, ms, ratio, stepr) in CASES.items():
        assert O.mid_ratios(mw, ms, W, S) == (ratio, stepr), name


@pytest.mark.parametrize("signal", SIGNALS)
def test_oracle_matches_reference_mid_edges(MID, signal):
    x = clip(signal)
    assert not SG.noise_defined_frames(x, W, S).any()          # no round-off-defined reference values
    T = O.frame_count(x.size, W, S)
    for name, (mw, ms, ratio, stepr) in CASES.items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)       # mean of an empty slice
            mid, st, _ = O.mid_feature_extraction(x, FS, mw, ms, W, S)
        ref = MID[key(signal, name, "mid")]
        assert mid.shape == ref.shape == (136, -(-T // stepr)), name
        np.testing.assert_allclose(mid, ref, rtol=1e-9, atol=1e-12, err_msg="%s %s" % (signal, name))
        if ratio <= 0:
            assert not mid[:, 1:].any(), name                   # every window after the first is empty
            assert mid[:, 0].any() == (ratio < 0), name         # ratio -1: frames 0 .. T-2; ratio 0: empty

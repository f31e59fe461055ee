"""CPU: the comparison helpers of tests/parity.py reject planted errors of the kinds a subtly wrong kernel makes."""
import numpy as np
import pytest

from oracle import st_oracle as O
from tests import parity as PA
from tests import signals as SG


@pytest.fixture(scope="module")
def REF():
    """Oracle matrix of a clip with loud and quiet frames (800 / 400, deltas on), and its window."""
    x = SG.bank(16000, 800, 400)["loud_quiet"]
    return O.feature_extraction(x, 16000, 800, 400)[0], 800


def test_unmodified_passes(REF):
    F, w = REF
    got = F.astype(np.float32)
    PA.check_features(got, F, w // 2)
    PA.check_zcr_exact(got, F)
    PA.check_energy_relative(got, F)


def test_entry_at_three_times_tolerance(REF):
    F, w = REF
    got = F.copy()
    got[12, 5] += 3 * (PA.RTOL * abs(F[12, 5]) + PA.ATOL)
    with pytest.raises(AssertionError, match="outside tolerance"):
        PA.check_features(got, F, w // 2)
    PA.check_features(got, F, w // 2, allow={12: 4.0})          # an exception entry's bound lets it through


def test_rolloff_two_quanta(REF):
    F, w = REF
    got = F.copy()
    got[PA.ROLLOFF_ROW, 3] += 2.0 / (w // 2)
    with pytest.raises(AssertionError, match="rolloff"):
        PA.check_features(got, F, w // 2)
    one = F.copy()
    one[PA.ROLLOFF_ROW, 3] += 1.0 / (w // 2)                     # one quantum on one frame is a float32 tie
    PA.check_features(one, F, w // 2)


def test_zcr_one_quantum(REF):
    F, w = REF
    got = F.copy()
    got[PA.ZCR_ROW, 7] += 0.5 / (w - 1)
    with pytest.raises(AssertionError, match="zcr not exact"):
        PA.check_zcr_exact(got, F)


def test_quiet_frame_energy(REF):
    F, w = REF
    quiet = int(np.argmin(F[PA.ENERGY_ROW]))
    assert F[PA.ENERGY_ROW, quiet] < 1e-7
    got = F.copy()
    got[PA.ENERGY_ROW, quiet] *= 1.001
    PA.check_features(got, F, w // 2)                          # below the absolute term: the feature check is blind here
    with pytest.raises(AssertionError, match="energy off"):
        PA.check_energy_relative(got, F)


def test_exception_table():
    names = set(SG.NOTES) | set(SG.float_bank(16000, 800, 400))
    for e in PA.EXCEPTIONS:
        assert e["signal"] in names and e["reason"]
        assert e["measured"] <= e["bound"]
        assert set(e["kinds"]) <= {0, 1, 2, 3}
    assert PA.exception_bounds("chirp_f32", 3) == {13: 2.0, 47: 2.0}
    assert PA.exception_bounds("chirp_f32", 1) == {}            # every other kernel: the standard tolerance
    assert PA.exception_bounds("loud_quiet", 2) == {}

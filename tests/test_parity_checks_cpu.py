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


@pytest.fixture(scope="module")
def MID(REF):
    """A short-term matrix within tolerance of REF (every entry off by 0.9 tau, signs alternating; one rolloff flip)
    and its mid-term matrix at ratio 7 / step 4, pooled in float64 and rounded to float32."""
    F, w = REF
    tau = PA.RTOL * np.abs(F) + PA.ATOL
    sign = np.where((np.arange(F.size) % 2).reshape(F.shape) == 0, 1.0, -1.0)
    st = F + 0.9 * tau * sign
    st[PA.ROLLOFF_ROW, 11] = F[PA.ROLLOFF_ROW, 11] + 1.0 / (w // 2)
    PA.check_features(st, F, w // 2)
    return st, O.mid_pool(st, 7, 4).astype(np.float32)


def test_mid_propagated_passes(REF, MID):
    F, w = REF
    st, mid = MID
    PA.check_mid_propagated(mid, st, F, 7, 4, w // 2)
    PA.check_mid_propagated(O.mid_pool(F, 7, 4), F, F, 7, 4, w // 2)


def mid_bounds(F, ratio, stepr, row, j):
    """(mean bound, std bound) of window j of short-term row ``row``, as check_mid_propagated derives them."""
    a, b = PA.mid_slices(F.shape[1], ratio, stepr)[j]
    tau = PA.RTOL * np.abs(F[row, a:b]) + PA.ATOL
    return tau.mean(), np.sqrt((tau ** 2).mean())


def test_mid_mean_and_std_three_times_bound(REF, MID):
    F, w = REF
    st, mid = MID
    n = F.shape[0]
    mb, _ = mid_bounds(F, 7, 4, 12, 3)
    ref = O.mid_pool(F, 7, 4)
    got = mid.astype(np.float64)
    got[12, 3] = ref[12, 3] + 3 * mb
    with pytest.raises(AssertionError, match="propagated tolerance"):
        PA.check_mid_propagated(got, st, F, 7, 4, w // 2)
    got = mid.astype(np.float64)
    _, sb = mid_bounds(F, 7, 4, 40, 5)
    got[n + 40, 5] = ref[n + 40, 5] - 3 * sb
    with pytest.raises(AssertionError, match="propagated tolerance"):
        PA.check_mid_propagated(got, st, F, 7, 4, w // 2)


def test_mid_slices_follow_python():
    assert PA.mid_slices(10, 3, 4) == [(0, 3), (4, 7), (8, 10)]
    assert PA.mid_slices(10, 0, 4) == [(0, 0), (4, 4), (8, 8)]
    assert PA.mid_slices(10, -1, 4)[0] == (0, 9) and all(b <= a for a, b in PA.mid_slices(10, -1, 4)[1:])
    assert PA.mid_slices(10, -20, 20) == [(0, 0)]
    assert PA.mid_slices(5, 9, 1)[-1] == (4, 5)


def float32_spectra(x, starts, N):
    """|X[k]| / K of z = y_frame - y_frame[0] by numpy's float32 FFT, DC from the float64 sum: a correct float32 transform."""
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    fr = np.stack([y[s:s + N] for s in starts])
    z = (fr - fr[:, :1]).astype(np.complex64)
    got = (np.abs(np.fft.fft(z, axis=1)[:, :N // 2]) / np.float32(N // 2)).astype(np.float64)
    got[:, 0] = np.abs(fr.sum(axis=1)) / (N // 2)
    return got


@pytest.mark.parametrize("name", ["edge_impulses", "constant_runs", "loud_quiet"])
def test_spectrum_bound(name):
    """A float32 FFT passes the spectrum bound; one bin off by 1e-3 relative, a constant frame with a non-zero bin, a
    constant frame zeroed where one sample differs, and a DC bin off by 1e-4 of the frame's largest bin do not."""
    N, s = 800, 200
    x = SG.bank(16000, N, s)[name]
    starts = np.arange(0, len(x) - N + 1, s)
    got = float32_spectra(x, starts, N)
    r, rd = PA.check_spectrum(got, x, starts, N, name)
    assert r < 0.1 and rd < 0.1, (r, rd)
    ref, _, _, flat = PA.spectrum_reference(x, starts, N)
    j = int(np.argmax(ref[:, 1:].sum(axis=1)))
    k = 1 + int(np.argmax(ref[j, 1:]))
    for what, edit in (("bin", lambda g: g.__setitem__((j, k), g[j, k] * 1.001)),
                       ("DC", lambda g: g.__setitem__((j, 0), g[j, 0] + 1e-4 * ref[j, k]))):
        bad = got.copy()
        edit(bad)
        with pytest.raises(AssertionError, match="outside the spectrum bound"):
            PA.check_spectrum(bad, x, starts, N, what)
    if name == "constant_runs":
        c = int(np.nonzero(flat)[0][0])
        bad = got.copy()
        bad[c, 5] = 1e-30
        with pytest.raises(AssertionError, match="constant frames"):
            PA.check_spectrum(bad, x, starts, N, "constant")
        one = np.nonzero(~flat & (SG.constant_frames(x, N - 1, starts + 1) | SG.constant_frames(x, N - 1, starts)))[0]
        assert one.size
        bad = got.copy()
        bad[one[0], 1:] = 0.0
        with pytest.raises(AssertionError, match="outside the spectrum bound"):
            PA.check_spectrum(bad, x, starts, N, "one differing sample")


def test_exception_table():
    names = set(SG.NOTES) | set(SG.float_bank(16000, 800, 400))
    for e in PA.EXCEPTIONS:
        assert e["signal"] in names and e["reason"]
        assert e["measured"] <= e["bound"]
        assert set(e["kinds"]) <= {0, 1, 2, 3}
    assert PA.exception_bounds("chirp_f32", 3) == {13: 2.0, 47: 2.0}
    assert PA.exception_bounds("chirp_f32", 1) == {}            # every other kernel: the standard tolerance
    assert PA.exception_bounds("loud_quiet", 2) == {}

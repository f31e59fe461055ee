"""CPU: the oracle against the UNMODIFIED reference on randomised configurations.

The reference's outputs on these inputs are stored in tests/golden/reference_checks.npz
(oracle/make_golden_reference_checks.py regenerates them where the reference tree exists); its larger matrices as
fingerprints: shape, per-row sums of |values|, per-row sums under seeded +-1 signs (the first all +1) and a fixed seeded
sample of entries.
"""
import numpy as np
import pytest

from oracle import st_oracle as O
from tests.conftest import load_golden


@pytest.fixture(scope="module")
def REF():
    return load_golden("reference_checks.npz")


CASES = []
_rng = np.random.default_rng(20260922)
for _ in range(14):
    fs = int(_rng.choice([8000, 16000, 22050, 32000, 44100, 48000]))
    w = int(_rng.integers(max(240, fs // 70), fs // 12))
    s = int(_rng.integers(max(1, w // 8), w + 1))
    n = int(_rng.integers(3 * w, 12 * w))
    CASES.append((fs, w, s, n, int(_rng.integers(0, 10 ** 6))))
TABLE_CASES = [(16000, 400), (44100, 441), (8000, 200), (22050, 551), (48000, 1200)]
ERROR_CASES = [(4000, 100, 50, 50), (4000, 100, 50, 1000), (8000, 160, 80, 100),
               (8000, 160, 80, 1000), (4000, 400, 200, 100), (16000, 800, 400, 799)]


def case_input(fs, n, seed):
    x = O.synth_clip(seed, n, fs)
    if seed % 3 == 0:                       # float-valued input with a DC offset
        rng = np.random.default_rng(seed)
        x = x.astype(np.float64) * float(rng.uniform(0.01, 3.0)) + float(rng.uniform(-500, 500))
    return x


PROJ = 4          # signed row sums per row: all +1, then seeded random +-1


def fingerprint(key, a, picks=16):
    """One float64 vector for a 2-D array: its shape, per-row sums of |a|, PROJ per-row sums under +-1 signs seeded by `key`
    (the first all +1: the plain row sum), and `picks` entries at positions seeded by `key`.  A sign error or compensating
    errors inside a row change a signed sum unless they are within the tolerance."""
    rng = np.random.default_rng(sum(key.encode()))
    signs = rng.choice([-1.0, 1.0], size=(a.shape[1], PROJ))
    signs[:, 0] = 1.0
    idx = rng.choice(a.size, size=min(picks, a.size), replace=False)
    return np.concatenate([np.array(a.shape, dtype=np.float64), np.abs(a).sum(axis=1), (a @ signs).ravel(), a.ravel()[idx]])


def check_fingerprint(got, REF, key, rtol, atol):
    """`got` against the stored fingerprint of the reference's matrix.  Every element within rtol / atol of the reference
    bounds each row's sum of |values| and each signed row sum by rtol x the reference's sum of |values| plus atol per
    element; the sampled entries are held to rtol / atol themselves."""
    got = np.asarray(got, dtype=np.float64)
    ref = REF[key]
    assert got.shape == tuple(int(v) for v in ref[:2]), key
    R, C = got.shape
    fp = fingerprint(key, got)
    a0, p0, s0 = 2, 2 + R, 2 + R + R * PROJ
    bound = rtol * ref[a0:p0] + atol * C
    np.testing.assert_array_less(np.abs(fp[a0:p0] - ref[a0:p0]), bound + 1e-300, err_msg=key + " |row| sums")
    np.testing.assert_array_less(np.abs(fp[p0:s0] - ref[p0:s0]).reshape(R, PROJ), np.repeat(bound[:, None], PROJ, axis=1) + 1e-300,
                                 err_msg=key + " signed row sums")
    np.testing.assert_allclose(fp[s0:], ref[s0:], rtol=rtol, atol=atol, err_msg=key)


def mid_params(w, s, seed):
    rng = np.random.default_rng(seed)
    if seed % 3 == 0:                       # the draws case_input made from the same generator
        rng.uniform(0.01, 3.0), rng.uniform(-500, 500)
    return int(rng.integers(2, 9)) * s + w, int(rng.integers(1, 9)) * s


@pytest.mark.parametrize("fs,w,s,n,seed", CASES)
def test_random_configurations(REF, fs, w, s, n, seed):
    i = CASES.index((fs, w, s, n, seed))
    x = case_input(fs, n, seed)
    err = str(REF["c%d_error" % i])
    if err:
        with pytest.raises({"ValueError": ValueError, "IndexError": IndexError}[err]):
            O.feature_extraction(x, fs, w, s, deltas=bool(seed % 2))
        return
    got, gnames = O.feature_extraction(x, fs, w, s, deltas=bool(seed % 2))
    assert gnames == list(REF["names_%d" % (seed % 2)])
    check_fingerprint(got, REF, "c%d_st" % i, rtol=1e-8, atol=1e-10)
    loop, _ = O.feature_extraction_loop(x[: 4 * w], fs, w, s, deltas=bool(seed % 2))
    check_fingerprint(loop, REF, "c%d_loop" % i, rtol=1e-8, atol=1e-10)
    sp = O.spectrogram(x, fs, w, s)
    check_fingerprint(sp[0], REF, "c%d_sp" % i, rtol=1e-9, atol=1e-12)
    assert sp[1] == list(REF["c%d_sp_t" % i])
    check_fingerprint(np.array(sp[2])[None, :], REF, "c%d_sp_f" % i, rtol=0, atol=0)
    if str(REF["c%d_ch_error" % i]):
        with pytest.raises(ValueError):
            O.chromagram(x, fs, w, s)
    else:
        ch = O.chromagram(x, fs, w, s)
        check_fingerprint(ch[0], REF, "c%d_ch" % i, rtol=1e-9, atol=1e-12)
        assert ch[1] == list(REF["c%d_ch_t" % i]) and ch[2] == list(REF["chroma_names"])
    mw, ms = mid_params(w, s, seed)
    mid = O.mid_feature_extraction(x, fs, mw, ms, w, s)
    check_fingerprint(mid[0], REF, "c%d_mid" % i, rtol=1e-8, atol=1e-10)
    assert mid[2] == list(REF["mid_names_%d" % (seed % 2)])


def test_tables_match_reference(REF):
    for fs, K in TABLE_CASES:
        np.testing.assert_array_equal(O.mel_filterbank(fs, K), REF["mel_%d_%d" % (fs, K)])
        os_, osh = O.chroma_tables(fs, K)
        np.testing.assert_array_equal(os_, REF["semis_%d_%d" % (fs, K)])
        np.testing.assert_array_equal(osh, REF["share_%d_%d" % (fs, K)])
        rng = np.random.default_rng(K)
        X = rng.random(K)
        np.testing.assert_allclose(O.chroma_operator(fs, K) @ (X ** 2) / (X ** 2).sum(), REF["chroma_%d_%d" % (fs, K)],
                                   rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("fs,w,s,n", ERROR_CASES)
def test_error_precedence(REF, fs, w, s, n):
    """mel bank IndexError (before the loop) > no frames ValueError > chroma ValueError (frame 0)."""
    j = ERROR_CASES.index((fs, w, s, n))
    ref_type = {"ValueError": ValueError, "IndexError": IndexError}[str(REF["e%d_type" % j])]
    x = O.synth_clip(1, n, fs)
    with pytest.raises(ref_type) as got:
        O.feature_extraction(x, fs, w, s)
    assert ("need at least one array" in str(REF["e%d_text" % j])) == ("need at least one array" in str(got.value))
    with pytest.raises(ref_type):
        O.feature_extraction_loop(x, fs, w, s)

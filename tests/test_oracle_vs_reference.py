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
from tests.golden_cases import ERROR_CASES, REF_CASES, TABLE_CASES, case_input, check_fingerprint, mid_params


@pytest.fixture(scope="module")
def REF():
    return load_golden("reference_checks.npz")


@pytest.mark.parametrize("fs,w,s,n,seed", REF_CASES)
def test_random_configurations(REF, fs, w, s, n, seed):
    i = REF_CASES.index((fs, w, s, n, seed))
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

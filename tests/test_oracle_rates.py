"""CPU: the oracle against the UNMODIFIED reference across sample rates, from tests/golden/rates.npz
(oracle/make_golden_rates.py regenerates it where the reference tree exists).

* At every point of the (fs, window) sweep of tests/test_rates_cpu.py, the oracle's mel bank and chroma operator raise
  what the reference's raise (IndexError below 6 854 Hz at every specialised window, nothing above).  The kernels' host
  tables are held to the oracle's statuses there, so their refusals are the reference's.
* At the common rates and the lowest accepted ones, the mel bank and the chroma operator are the reference's.
* At every GPU rate config (tests.kernels.RATE_CONFIGS, hops longer than the window among them), the oracle's
  feature_extraction and chromagram of a seeded clip are the reference's, as fingerprints
  (tests/test_oracle_vs_reference.fingerprint).
"""
import warnings

import numpy as np
import pytest

from oracle import st_oracle as O
from tests.conftest import load_golden
from tests.kernels import RATE_CONFIGS
from tests.test_oracle_vs_reference import check_fingerprint
from tests.test_rates_cpu import RATES

TABLE_RATES = set(RATES) | set(range(6854, 6871))
EXC = {0: None, 1: IndexError, 2: ValueError}


@pytest.fixture(scope="module")
def REF():
    return load_golden("rates.npz")


def mel_probe(K):
    return np.random.default_rng(K).uniform(0.5, 1.5, K)


def chroma_input(K):
    return np.random.default_rng(K + 1).uniform(0.1, 1.0, K)


def rate_input(fs, w, s):
    """Half a second of the oracle's synthetic clip plus a few frames, the seed from the config."""
    return O.synth_clip(fs + w + s, fs // 2 + 3 * w + s // 3, fs)


def raised(fn, *a):
    try:
        fn(*a)
    except (IndexError, ValueError) as e:
        return type(e)
    return None


def test_table_statuses_match_reference(REF):
    rates, windows = REF["rates"].tolist(), REF["windows"].tolist()
    for i, fs in enumerate(rates):
        for j, w in enumerate(windows):
            K = w // 2
            assert raised(O.mel_filterbank, fs, K) is EXC[int(REF["mel_exc"][i, j])], ("mel", fs, w)
            assert raised(O.chroma_operator, fs, K) is EXC[int(REF["chroma_exc"][i, j])], ("chroma", fs, w)
    assert (REF["mel_exc"] == 1).any() and (REF["mel_exc"] == 0).any()


def test_tables_match_reference(REF):
    n = 0
    for fs in sorted(TABLE_RATES):
        for w in REF["windows"].tolist():
            K = w // 2
            if "mel_%d_%d" % (fs, w) in REF:
                mel = O.mel_filterbank(fs, K)
                np.testing.assert_allclose(mel @ mel_probe(K), REF["mel_%d_%d" % (fs, w)],
                                           rtol=1e-13, atol=1e-15, err_msg="mel fs=%d w=%d" % (fs, w))
                n += 1
            if "chroma_%d_%d" % (fs, w) in REF:
                X2 = chroma_input(K) ** 2
                np.testing.assert_allclose(O.chroma_operator(fs, K) @ X2 / X2.sum(), REF["chroma_%d_%d" % (fs, w)],
                                           rtol=1e-12, atol=1e-15, err_msg="chroma fs=%d w=%d" % (fs, w))
    assert n >= len(RATES) * len(REF["windows"])


@pytest.mark.parametrize("fs,w,s", [c[:3] for c in RATE_CONFIGS], ids=["%d-%d-%d" % c[:3] for c in RATE_CONFIGS])
def test_features_match_reference(REF, fs, w, s):
    x = rate_input(fs, w, s)
    key = "%d_%d_%d" % (fs, w, s)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        check_fingerprint(O.feature_extraction(x, fs, w, s, deltas=True)[0], REF, "st_" + key, rtol=1e-8, atol=1e-10)
        check_fingerprint(O.chromagram(x, fs, w, s)[0], REF, "ch_" + key, rtol=1e-9, atol=1e-12)

"""GPU: the float64 path, through the drop-ins under set_precision("float64"), held to every golden set of the reference
by the same checks, tolerances and documented exceptions that hold the float64 oracle to them.

The golden tests of tests/test_oracle_golden.py, test_oracle_adversarial.py, test_oracle_rates.py and test_oracle_mid.py
that compute features run once more in a nested pytest session, with the oracle's feature entry points
(feature_extraction, its loop flavour, spectrogram, chromagram, mid_feature_extraction) rebound to ShortTermFeatures /
MidTermFeatures for the duration of each test: every assertion, tolerance and exception (digitally silent frames,
noise-defined rows) is the one written for the oracle, so the float64 path meets the oracle's own contract with the
reference, and each check has one statement."""
import os

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

GOLDEN_TESTS = {
    "test_oracle_golden.py": ["test_doremi_short_term", "test_doremi_loop_flavour", "test_doremi_spectrogram_chromagram_mid",
                              "test_reference_pytest_inputs", "test_synthetic", "test_edges"],
    "test_oracle_adversarial.py": ["test_oracle_matches_reference_on_bank"],
    "test_oracle_rates.py": ["test_features_match_reference"],
    "test_oracle_mid.py": ["test_oracle_matches_reference_mid_edges"],
}


class Float64DropIns:
    """pytest plugin: every test of the nested session runs with the oracle's feature functions rebound to the drop-ins
    under set_precision("float64")."""

    @pytest.fixture(autouse=True)
    def float64_drop_ins(self, monkeypatch):
        import pyaudioanalysis_b200 as pkg
        from oracle import st_oracle as O
        from pyaudioanalysis_b200 import MidTermFeatures as MT
        from pyaudioanalysis_b200 import ShortTermFeatures as ST

        def st(signal, fs, window, step, deltas=True, tables_per_frame=True):
            return ST.feature_extraction(signal, fs, window, step, deltas=deltas)

        def mid(signal, fs, mid_window, mid_step, short_window, short_step, loop=False):
            return MT.mid_feature_extraction(signal, fs, mid_window, mid_step, short_window, short_step)

        monkeypatch.setattr(ST, "PRINT_SPECTROGRAM_SHAPE", False)
        for name, fn in (("feature_extraction", st), ("feature_extraction_loop", st), ("mid_feature_extraction", mid),
                         ("spectrogram", lambda x, fs, w, s: ST.spectrogram(x, fs, w, s)),
                         ("chromagram", lambda x, fs, w, s: ST.chromagram(x, fs, w, s))):
            monkeypatch.setattr(O, name, fn)
        pkg.set_precision("float64")
        yield
        pkg.set_precision("float32")


@pytest.mark.parametrize("module", sorted(GOLDEN_TESTS))
def test_float64_path_meets_the_oracle_goldens(module):
    ids = [os.path.join(ROOT, "tests", module) + "::" + t for t in GOLDEN_TESTS[module]]
    rc = pytest.main(["-q", "-p", "no:cacheprovider", "--rootdir", ROOT, *ids], plugins=[Float64DropIns()])
    assert rc == 0, "%s: the float64 drop-ins fail the oracle's golden checks (see the nested session's report)" % module

"""The inputs the golden files were generated from, which a generator (oracle/make_golden_*.py) and the test that holds the
oracle to its golden must agree on.  Only the reference's outputs are stored; the inputs are regenerated from the seeds
and lists here, so a change to any of them breaks its golden until the generator is run again."""
import numpy as np

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import RATES


# ---------------------------------------------------------------------------------------------------------------------
# Fingerprints: how the goldens store the reference's larger matrices
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


# ---------------------------------------------------------------------------------------------------------------------
# reference_checks.npz (oracle/make_golden_reference_checks.py, tests/test_oracle_vs_reference.py)
REF_CASES = []
_rng = np.random.default_rng(20260922)
for _ in range(14):
    fs = int(_rng.choice([8000, 16000, 22050, 32000, 44100, 48000]))
    w = int(_rng.integers(max(240, fs // 70), fs // 12))
    s = int(_rng.integers(max(1, w // 8), w + 1))
    n = int(_rng.integers(3 * w, 12 * w))
    REF_CASES.append((fs, w, s, n, int(_rng.integers(0, 10 ** 6))))
TABLE_CASES = [(16000, 400), (44100, 441), (8000, 200), (22050, 551), (48000, 1200)]
ERROR_CASES = [(4000, 100, 50, 50), (4000, 100, 50, 1000), (8000, 160, 80, 100),
               (8000, 160, 80, 1000), (4000, 400, 200, 100), (16000, 800, 400, 799)]


def case_input(fs, n, seed):
    x = O.synth_clip(seed, n, fs)
    if seed % 3 == 0:                       # float-valued input with a DC offset
        rng = np.random.default_rng(seed)
        x = x.astype(np.float64) * float(rng.uniform(0.01, 3.0)) + float(rng.uniform(-500, 500))
    return x


def mid_params(w, s, seed):
    rng = np.random.default_rng(seed)
    if seed % 3 == 0:                       # the draws case_input made from the same generator
        rng.uniform(0.01, 3.0), rng.uniform(-500, 500)
    return int(rng.integers(2, 9)) * s + w, int(rng.integers(1, 9)) * s


# ---------------------------------------------------------------------------------------------------------------------
# adversarial.npz (oracle/make_golden_adversarial.py, tests/test_oracle_adversarial.py)
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


def adv_key(fs, w, s, name, what):
    return "%d_%d_%d_%s_%s" % (fs, w, s, name, what)


# ---------------------------------------------------------------------------------------------------------------------
# mid_edges.npz (oracle/make_golden_mid.py, tests/test_oracle_mid.py)
FS, W, S = 16000, 800, 400
SIGNALS = ("loud_quiet", "chirp")
# name -> (mid_window, mid_step) in samples, with the (ratio, step ratio) the reference derives from them
MID_CASES = {
    "ratio_0": (400, 800, 0, 2),
    "ratio_minus_1": (0, 800, -1, 2),
    "tie_half_to_0": (600, 800, 0, 2),          # 0.5 rounds to even: 0
    "tie_3_halves_to_2": (1000, 800, 2, 2),     # 1.5 rounds to even: 2
    "longer_than_clip": (32000, 16000, 79, 40),
    "step_above_ratio": (1200, 2000, 2, 5),
}


def mid_key(signal, case, what):
    return "%s_%s_%s" % (signal, case, what)


def clip(signal):
    return SG.bank(FS, W, S)[signal]


# ---------------------------------------------------------------------------------------------------------------------
# rates.npz (oracle/make_golden_rates.py, tests/test_oracle_rates.py)
TABLE_RATES = set(RATES) | set(range(6854, 6871))


def mel_probe(K):
    return np.random.default_rng(K).uniform(0.5, 1.5, K)


def chroma_input(K):
    return np.random.default_rng(K + 1).uniform(0.1, 1.0, K)


def rate_input(fs, w, s):
    """Half a second of the oracle's synthetic clip plus a few frames, the seed from the config."""
    return O.synth_clip(fs + w + s, fs // 2 + 3 * w + s // 3, fs)

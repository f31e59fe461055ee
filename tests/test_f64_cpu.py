"""CPU: the float64 path's pieces (csrc/f64.cuh) run on the host by tests/f64_host.cu -- the clip normalisation, rows 0-2,
the mid-term pooling and the fp64 transform -- against the float64 oracle and NumPy, bit for bit where the kernels
promise it; the C ABI's argument checks, which return before any CUDA call."""
import ctypes

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import host_exe
from tests import signals as SG
from tests.host_exe import bits, floats, hexes, run


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "f64_host.cu", "-O2")


def host_norm(exe, x):
    v = floats(run(exe, "norm %d %s\n" % (len(x), hexes(x)))[0][1:])
    return v[0], v[1], v[2:]


def clips(n, rng):
    i16 = np.clip(np.round(rng.normal(0, 4000, n) + 1234.5), -32768, 32767).astype(np.int16)
    f32 = (rng.normal(0, 0.3, n) + 0.01).astype(np.float32)
    f64 = rng.normal(0, 1e4, n) + 3e5
    return {"i16": i16, "f32": f32, "f64": f64, "const": np.full(n, 77, np.int16)}


@pytest.mark.parametrize("n", [1, 2, 7, 8, 127, 128, 129, 1000, 4097, (1 << 17) + 5])
def test_normalisation_bit_for_bit(exe, n):
    rng = np.random.default_rng(n)
    for kind, x in clips(n, rng).items():
        mean, scale, y = host_norm(exe, x)
        ref = O.normalize_clip(x)
        z = np.asarray(x, dtype=np.float64) / 32768.0
        assert bits(mean) == bits(z.mean()), kind
        assert bits(scale) == bits(np.abs(z - z.mean()).max() + 1e-10), kind
        np.testing.assert_array_equal(bits(y), bits(ref), err_msg=kind)


def test_normalisation_signal_bank(exe):
    for name, x in SG.bank(16000, 800, 400).items():
        _, _, y = host_norm(exe, x)
        np.testing.assert_array_equal(bits(y), bits(O.normalize_clip(x)), err_msg=name)


@pytest.mark.parametrize("w", [2, 9, 10, 400, 441, 800, 801, 44100])
def test_time_rows_bit_for_bit(exe, w):
    rng = np.random.default_rng(w)
    y = O.normalize_clip(rng.normal(0, 1000, w + 50))[25:25 + w]
    y[::7] = 0.0                                    # sign 0 samples
    v = floats(run(exe, "time %d %s\n" % (w, hexes(y)))[0][1:])
    assert bits(v[0]) == bits(O._zcr(y))
    assert bits(v[1]) == bits(O._energy(y))
    np.testing.assert_allclose(v[2], O._block_entropy(y), rtol=1e-13, atol=1e-15)   # log2 of the host libm


def host_pool(exe, X, ratio, stepr):
    F, T = X.shape
    v = floats(run(exe, "pool %d %d %d %d %s\n" % (F, T, ratio, stepr, hexes(X)))[0][1:])
    return v.reshape(2 * F, -1)


@pytest.mark.parametrize("ratio,stepr", [(-5, 1), (-1, 3), (0, 2), (1, 1), (3, 2), (7, 7), (41, 20), (300, 1), (5000, 3)])
def test_pooling_bit_for_bit(exe, ratio, stepr):
    rng = np.random.default_rng(abs(ratio) * 31 + stepr)
    X = rng.normal(size=(5, 257)) * np.array([[1e-3], [1.0], [1e6], [3.0], [0.0]]) + 0.5
    X[1, 10:20] = np.inf
    X[2, 100] = np.nan
    np.testing.assert_array_equal(bits(host_pool(exe, X, ratio, stepr)), bits(O.mid_pool(X, ratio, stepr)))


# fp64 transform: |X - fft| <= c * log2(n) * eps * sum|x| per bin, c = 4 (the passes' rounding, the tables' 1-ulp
# twiddles); primes transform in one direct pass of n terms: log2(n) -> n there
@pytest.mark.parametrize("n", [8, 400, 441, 800, 801, 882, 1024, 2 * 3 * 5 * 7 * 11, 997])
def test_transform_against_numpy(exe, n):
    rng = np.random.default_rng(n)
    x = rng.normal(size=n)
    v = floats(run(exe, "fft %d %s\n" % (n, hexes(x)))[0][1:])
    Z = np.fft.fft(x)
    depth = n if all(n % p for p in range(2, int(n ** 0.5) + 1)) else np.log2(n)
    bound = 4 * depth * np.finfo(float).eps * np.abs(x).sum()
    assert np.abs(v[:n] - Z.real).max() <= bound
    assert np.abs(v[n:] - Z.imag).max() <= bound


def test_abi_argument_checks():
    from pyaudioanalysis_b200 import _lib
    L = _lib.lib()
    vp = ctypes.c_void_p(8)
    INV = _lib.ERR_INVALID
    assert L.b200aa_clip_stats_f64(None, 0, 1, 10, 10, None, vp, None) == INV
    assert L.b200aa_clip_stats_f64(vp, 3, 1, 10, 10, None, vp, None) == INV
    assert L.b200aa_clip_stats_f64(vp, 2, 1, 10, 9, None, vp, None) == INV          # clip_stride < n_samples
    assert L.b200aa_clip_stats_f64(vp, 2, -1, 10, 10, None, vp, None) == INV
    assert L.b200aa_st_features_f64(None, vp, 0, 1, 10, 10, None, vp, 1, vp, 1, None) == INV
    for fn in (L.b200aa_spectrogram_f64, L.b200aa_chromagram_f64):
        assert fn(None, vp, 0, 1, 10, 10, vp, vp, None) == INV
    for fn in (L.b200aa_spectrogram_ragged_f64, L.b200aa_chromagram_ragged_f64):
        assert fn(None, vp, 0, 1, 10, 10, vp, vp, vp, None) == INV
    assert L.b200aa_mid_pool_f64(vp, 1, 68, 10, 10, 4, 0, vp, None) == INV           # step_ratio < 1
    assert L.b200aa_mid_pool_f64(vp, 1, 68, 10, 9, 4, 1, vp, None) == INV            # t_stride < n_frames
    assert L.b200aa_mid_pool_f64(None, 1, 68, 10, 10, 4, 1, vp, None) == INV
    assert L.b200aa_mid_pool_ragged_f64(vp, 1, 68, 10, None, 4, 1, vp, None) == INV
    assert L.b200aa_long_term_mean_f64(vp, 1, 0, 3, vp, None) == INV
    assert L.b200aa_long_term_mean_ragged_f64(vp, 1, 4, 3, None, vp, None) == INV


def test_precision_setting_and_install():
    import types
    import pyaudioanalysis_b200 as pkg
    from pyaudioanalysis_b200 import precision
    assert pkg.get_precision() == "float32"
    with pytest.raises(ValueError):
        pkg.set_precision("float16")
    fake = types.SimpleNamespace(ShortTermFeatures=types.ModuleType("ST"), MidTermFeatures=types.ModuleType("MT"))
    for n in ("feature_extraction", "spectrogram", "chromagram"):
        setattr(fake.ShortTermFeatures, n, None)
    for n in ("mid_feature_extraction", "beat_extraction", "directory_feature_extraction",
              "multiple_directory_feature_extraction", "directory_feature_extraction_no_avg",
              "mid_feature_extraction_to_file", "mid_feature_extraction_file_dir"):
        setattr(fake.MidTermFeatures, n, None)
    try:
        pkg.install(fake)
        assert precision.get_precision() == "float32"
        pkg.install(fake, precision="float64")
        assert precision.wide() and fake.ShortTermFeatures.feature_extraction is pkg.ShortTermFeatures.feature_extraction
    finally:
        pkg.uninstall()
        pkg.set_precision("float32")


def test_float64_decode_rule():
    """Files whose device staging is not their host decode exactly are read on the host under float64 precision."""
    from pyaudioanalysis_b200 import audioio as A
    from pyaudioanalysis_b200.MidTermFeatures import _staged_exactly
    host = {(A.PCM_S24, 2), (A.PCM_S32, 1), (A.PCM_S32, 2), (A.PCM_F64, 1), (A.PCM_F64, 2)}
    for fmt in range(6):
        for ch in (1, 2):
            assert _staged_exactly(fmt, ch) == ((fmt, ch) not in host), (fmt, ch)

"""CPU: the pieces of the beat-extraction kernel (csrc/beat.cuh, __host__ __device__) run on the host by tests/beat_host.cu --
NumPy's pairwise summation order, the chunked three-phase peak scan, and the whole per-clip computation -- against NumPy and
the host MidTermFeatures.beat_extraction, bit for bit."""

import numpy as np
import pytest

from pyaudioanalysis_b200.MidTermFeatures import _peak_positions, beat_extraction
from tests import host_exe
from tests.host_exe import hexes, run
from tests.conftest import load_golden
from tests.signals import peak_inputs

pytestmark = pytest.mark.skipif(host_exe.nvcc() is None, reason="nvcc not available")

PRODUCTION_CHUNK = 1024          # beat::kChunk
CHUNKS = (1, 2, 3, 31, 32, PRODUCTION_CHUNK)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "beat_host.cu", "-O1")


def _same(a, b):
    """Bit-for-bit equality, NaN equal to NaN."""
    a, b = float(a), float(b)
    return (np.isnan(a) and np.isnan(b)) or np.float64(a).tobytes() == np.float64(b).tobytes()


def test_pairwise_sum_matches_numpy(exe):
    rng = np.random.default_rng(1)
    d = np.abs(np.diff(rng.standard_normal(200001).astype(np.float32).astype(np.float64)))
    lengths = list(range(0, 301)) + [1000, 8191, 8192, 8193, 16384, 143998, 200000]
    out = run(exe, "sum %d %s %d %s\n" % (d.size, hexes(d), len(lengths), " ".join(map(str, lengths))))
    assert len(out) == len(lengths)
    for n, line in zip(lengths, out):
        ref = float(np.add.reduce(d[:n]))
        assert int(line[1]) == n
        for got in line[2:]:                                  # serial, 32 lanes, 256 lanes
            assert _same(float.fromhex(got), ref), (n, got, ref.hex())


def _scan_rows():
    """Rows for the chunked scan, each with the threshold the host would use, plus hand-made deltas."""
    rng = np.random.default_rng(7)
    rows = []
    for k in range(6):                                        # random walks
        rows.append(np.cumsum(rng.standard_normal(300 + 97 * k)).astype(np.float32).astype(np.float64))
    for period in (1, 2, 3, 31, 32, 64):                      # sawtooth whose period is a chunk length
        rows.append((np.arange(200) % period).astype(np.float64))
    for C in (2, 3, 31, 32):                                  # peaks on the first and the last frame of a chunk
        v = np.zeros(8 * C)
        v[::C] = 5.0
        v[C - 1::C] += 3.0
        rows.append(v)
    rows.append(np.arange(150, dtype=np.float64))             # monotone up / down
    rows.append(-np.arange(150, dtype=np.float64))
    rows.append(np.full(120, 2.5))                            # constant
    rows.append(np.repeat(rng.standard_normal(40), 5))        # plateaus
    v = np.cumsum(rng.standard_normal(250))                   # NaN inside
    v[[17, 100, 101]] = np.nan
    rows.append(v)
    for k in range(4):                                        # integer-valued: x < mx - delta can be an exact tie
        rows.append(np.cumsum(rng.integers(-3, 4, 180 + 40 * k)).astype(np.float64))
    out = []
    for v in rows:
        delta = 2.0 * np.abs(v[:-1] - v[1:]).mean()
        if not delta > 0:
            delta = 1e-16 if delta <= 0 else delta
        out.append((v, delta))
        if np.isfinite(v).all() and np.all(v == np.round(v)):
            out.append((v, 2.0))                              # integer delta: ties on integer rows
    return out


def test_chunked_scan_matches_peakdet(exe):
    cases = _scan_rows()
    script = []
    for v, delta in cases:
        for C in CHUNKS:
            script.append("peaks %d %d %s %s" % (C, v.size, float(delta).hex(), hexes(v)))
    out = run(exe, "\n".join(script) + "\n")
    i = 0
    for v, delta in cases:
        ref = _peak_positions(v, delta)
        for C in CHUNKS:
            assert [int(p) for p in out[i][1:]] == ref, (v.size, delta, C)
            i += 1


def _beat_cases():
    g = load_golden("beat.npz")
    cases = [(g["st_%d" % i], float(g["win_%d" % i])) for i in range(int(g["n"]))]
    for _, _, st in peak_inputs():
        for win in (0.05, 0.025, 0.1):
            cases.append((st, win))
    for st, _ in cases[:3]:                                   # more bins than frames: bins past T - 1 are never counted
        cases += [(st, 0.0005), (st[:, :30], 0.025), (st[:, :2], 0.05), (st, 1.5)]
    return [(np.asarray(st, dtype=np.float32).astype(np.float64), w) for st, w in cases]


def test_whole_clip_matches_host_beat_extraction(exe):
    cases = _beat_cases()
    script = ["beat %d %d %d %s %s" % (C, st.shape[0], st.shape[1], float(w).hex(), hexes(st)) for st, w in cases
              for C in (3, 32, PRODUCTION_CHUNK)]
    out = run(exe, "\n".join(script) + "\n")
    i = 0
    for st, w in cases:
        bpm, ratio = beat_extraction(st, w)
        for C in (3, 32, PRODUCTION_CHUNK):
            assert _same(float.fromhex(out[i][1]), bpm) and _same(float.fromhex(out[i][2]), ratio), (st.shape, w, C, out[i], bpm, ratio)
            i += 1

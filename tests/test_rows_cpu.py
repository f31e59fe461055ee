"""CPU: the row arithmetic of spectrogram() / chromagram() (csrc/rows.cuh, __host__ __device__) run on the host by
tests/rows_host.cu, for every clip length 0 .. 3 * window, against the oracle's row shapes, the rows its loops fill, and
the single-clip entry points' refusals; and the argument checks of the ragged row entry points, which return before
touching a device."""
import ctypes
import subprocess
import warnings

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import host_exe

CONFIGS = [(800, 400), (800, 200), (800, 333), (882, 441), (800, 800), (400, 160),
           (800, 1000), (600, 900), (882, 1323), (320, 400)]          # hops longer than the window: frames skip samples
FS = {882: 44100}


@pytest.fixture(scope="module")
def table(tmp_path_factory):
    exe = host_exe.build(tmp_path_factory, "rows_host.cu", "-O1")
    script = "".join("%d %d %d\n" % (w, s, 3 * w) for w, s in CONFIGS)
    out = subprocess.run([exe], input=script, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.splitlines()
    tables = {}
    for w, s in CONFIGS:
        max_clipped = int(lines.pop(0))
        rows = np.array([[int(v) for v in lines.pop(0).split()] for _ in range(3 * w + 1)], dtype=np.int64)
        tables[(w, s)] = (max_clipped, rows)
    return tables


@pytest.fixture(scope="module")
def lib():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib.lib()


def oracle_rows(fn, x, fs, w, s):
    """(rows allocated, rows filled) of the oracle's spectrogram / chromagram of x, or None where it raises."""
    try:
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore")
            out = fn(x, fs, w, s)[0]
    except ValueError:
        return None
    return out.shape[0], int(np.count_nonzero(np.abs(out).sum(axis=1)))


@pytest.mark.parametrize("w,s", CONFIGS, ids=["%d-%d" % c for c in CONFIGS])
def test_rows_match_oracle(table, lib, w, s):
    fs = FS.get(w, 16000)
    max_clipped, rows = table[(w, s)]
    x = np.random.default_rng(w + s).normal(0, 3000, 3 * w).astype(np.int16)     # every frame the loops fill is nonzero
    for n, sR, s_it, s_full, s_ref, cR, c_it, c_full, c_ref in rows.tolist():
        what = "w=%d s=%d n=%d" % (w, s, n)
        assert sR == lib.b200aa_spectrogram_rows(n, w, s) and cR == lib.b200aa_chromagram_rows(n, w, s), what
        # spectrogram: refused where np.zeros raises or gives no rows; every filled row is a full frame
        sp = oracle_rows(O.spectrogram, x[:n], fs, w, s)
        assert bool(s_ref) == (sp is None or sp[0] == 0), what
        if not s_ref:
            assert (sR, s_it, s_full) == (sp[0], sp[1], sp[1]), what
        # chromagram: refused where the oracle raises (no rows, a clipped frame shorter than K) and for clips shorter than
        # w + s, whose single zero row the single-clip entry point does not produce
        ch = oracle_rows(O.chromagram, x[:n], fs, w, s)
        assert bool(c_ref) == (ch is None or ch[0] == 0 or n - s - w < 0), what
        if not c_ref:
            starts = list(range(w, n - s, s))
            assert (cR, c_it) == ch and c_it == len(starts), what
            assert c_full == sum(1 for p in starts if p + w <= n), what
            assert all(w // 2 <= n - p < w for p in starts[c_full:]), what
            assert c_it - c_full <= max_clipped, what
    # the clipped-frame kernel's candidates per clip: a bound on the clipped frames of every clip, refused ones included
    clipped = [sum(1 for p in range(w, n - s, s) if p + w > n) for n in range(3 * w + 1)]
    assert max(clipped) == max_clipped, "the bound is reached for some length"


def test_ragged_row_entry_points_reject_bad_arguments(lib):
    INVALID = -1
    p = ctypes.c_void_p(256)                   # never dereferenced: every call below fails its argument check first
    n = None
    for fn in (lib.b200aa_spectrogram_ragged, lib.b200aa_chromagram_ragged):
        # (plan, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out, stream)
        assert fn(n, p, 0, 4, 16000, 16000, p, p, p, n) == INVALID
        assert fn(p, n, 0, 4, 16000, 16000, p, p, p, n) == INVALID
        assert fn(p, p, 0, 4, 16000, 16000, n, p, p, n) == INVALID
        assert fn(p, p, 0, 4, 16000, 16000, p, n, p, n) == INVALID
        assert fn(p, p, 0, 4, 16000, 16000, p, p, n, n) == INVALID
        assert fn(p, p, 2, 4, 16000, 16000, p, p, p, n) == INVALID
        assert fn(p, p, 0, -1, 16000, 16000, p, p, p, n) == INVALID
        assert fn(p, p, 0, 4, 16000, 15999, p, p, p, n) == INVALID
    # b200aa_row_counts(d_len, n_clips, window, step, which, d_rows, stream)
    assert lib.b200aa_row_counts(n, 4, 800, 400, 0, p, n) == INVALID
    assert lib.b200aa_row_counts(p, 4, 800, 400, 1, n, n) == INVALID
    assert lib.b200aa_row_counts(p, -1, 800, 400, 0, p, n) == INVALID
    assert lib.b200aa_row_counts(p, 4, 0, 400, 0, p, n) == INVALID
    assert lib.b200aa_row_counts(p, 4, 800, 0, 1, p, n) == INVALID
    assert lib.b200aa_row_counts(p, 4, 800, 400, 2, p, n) == INVALID


def test_ragged_rows_python_api_refuses_cpu_tensors():
    import torch
    import pyaudioanalysis_b200 as pkg
    with pytest.raises(TypeError):
        pkg.row_counts(torch.zeros(3, dtype=torch.int64), 800, 400, 0)
    with pytest.raises(TypeError):
        pkg.spectrogram_batch(torch.zeros(2, 4000, dtype=torch.int16), 16000, 800, 400,
                              lengths=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(TypeError):
        pkg.chromagram_batch(torch.zeros(2, 4000, dtype=torch.int16), 16000, 800, 400,
                             lengths=torch.zeros(2, dtype=torch.int64))

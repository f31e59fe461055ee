"""The per-entry chromagram bound of ``tests/parity.chromagram_bounds``: its derivation, float32 / fp64 emulations of the
kernels' chromagram paths held to it on the adversarial bank, the chroma tables and the clipped-frame kernel's
shared-memory boundary (no device needed).

**Rows.**  ``chromagram()`` allocates R = int((n - s - w) / s) + 1 rows and fills row r from the frame at w + r s
(ShortTermFeatures.py:347-355; csrc/rows.cuh, restated as ``parity.chromagram_rows`` and held to the library below).  A
row is *full* when its frame has all w samples (a row kernel transforms it), *clipped* when it has n = len - (w + r s)
samples, K <= n < w (``clipped_chroma_kernel``), *never filled* past the loop's last start (exactly 0), and a clip with a
clipped frame shorter than K is *refused*.  Every chroma class is c_j = (C X^2)_j / E, E = sum_k X_k^2 (E = 0: divided by
eps), with C the [12, K] chroma operator and X = |DFT|[0:K] / K of the normalised frame.

**Transform error, carried to the classes.**  With X'_k = X_k + d_k, c_j' - c_j = sum_k (C_jk - c_j)(X'_k^2 - X_k^2) / E'
(centred weights), |X'_k^2 - X_k^2| <= 2 X_k |d_k| + d_k^2 and E' >= E - sum_k (2 X_k |d_k| + d_k^2); where that reaches
0 the entry is unbounded (counted with its reason, never skipped).
* Full rows: the ball of ``spectrum_reference`` (|d_0| <= eps_0, |d_1..K-1|_2 <= eps_b, derived in
  tests/test_gpu_spectra.py), through ``_quad``: 2 |a X|_2 eps_b + max |a| eps_b^2, DC apart.  The same helper
  (``chroma_bound``) bounds the feature-mode chroma rows 21..32, and ``feature_bounds`` is unchanged by the move (same
  ``ref`` and ``bound`` arrays, bit for bit, on the bank at every window of test_feature_bounds_cpu).
* Clipped rows: ``clipped_chroma_kernel`` is a direct DFT in fp64 (u64 = 2^-53, gamma64_n = n u64 / (1 - n u64)), held per
  bin (``_quad_bins``: sum_k |C_jk - c_j| (2 X_k eps_k + eps_k^2)):
  - z_j = x_j - x_0 in fp64 is exact for int16 input; for float32 input it is rounded at most once, which one more step
    of gamma64 covers;
  - twiddles sincospi(2 j / n): the quotient is rounded once (|2 j / n| < 2, so the phase moves by at most 2 pi u64) and
    sincospi errs by 2 ulp per component (CUDA C++ Programming Guide, "Double-Precision Floating-Point Functions":
    sinpi / cospi 2 ulp, sincospi the same), < 4 u64 on [-1, 1]: (4 + 2 pi) u64 per component.  The phase index j k
    mod n is exact integer arithmetic, so every term uses the twiddle of its own phase;
  - n fma steps per component: gamma64(n + 2) |z|_1, plus the twiddle error times |z|_1; as a complex number sqrt(2)
    times that, which moves sqrt(re^2 + im^2) by no more;
  - a sqrt(re^2 + im^2): 4 u64 for the squares, sqrt and product, and the float32 record value a' = a (1 + alpha): a is
    computed in fp64 from the clip's fp64 mean (exact int64 sum for int16, a float64 sum in any order for float32, whose
    error gamma64(L) sum |x| / L moves max |x - mean| and bp) and rounded to float32 (u32 = 2^-24);
  - DC: a' re + n (a' (x_0 - m) + bp') with float32 a', m, bp': against a sum(x - mean) = a sum(x - m) + n a (m - mean)
    it errs by (a' - a) sum(x - m) + n (bp' - bp) (|m - mean| exactly for int16, whose mean is the same rounded quotient
    here, u32 |mean| + the mean's error for float32), plus the sum re (n additions) and 8 u64 of the expression's terms;
  - mag / K rounded to float once (u32 of the value), the double division 2 u64;
  - the float64 reference's own error: numpy's FFT of z (8 u64 ceil(log2 n) sqrt(n) |z|_2, the form of the spectrum
    bound), the DC sum(x - mean) taken exactly (Fractions) and rounded once, and a from the rounded mean.
  The clipped bound is fp64-tight: a few 1e-16 of the frame's |z|_1 per bin, so a clipped row's error is the float32
  rounding of X and of the chroma stage, a few u32 relative per class, quiet classes included.
* Rows never filled: exactly 0.  A frame whose normalised samples are all 0 (a run at the clip's exact integer mean) has
  X = 0 in every kernel and gets 0 exactly (the eps branch); a constant frame (X_1..K-1 = 0 exactly, from z = 0) gets its
  DC bin's class weights, C_j0, up to the chroma stage's roundings.

**Float32 chroma stage** (all kernels, ``chroma_lane`` and the solo kernel's inline taps): each class a sequential fma of
its squared taps, gamma(taps + 3); E = sum X^2 at depth ``sum_depth(K)`` = ceil(K / 16) + 12, which the solo kernel's
16-lane sums over Kp-padded rows set: 2 odd(ceil(K / 32)) <= ceil(K / 16) + 3 bins per lane, 4 shuffle levels and the
fma (the 32-lane layouts, the CTA kernel's DenseShape<K>::C bins per lane and the generic / clipped kernels' lane-strided
sums, hold half as many); one IEEE division (DIV_REL); products of (1 + err) factors to first order with a 1 % margin, and
1e-12 relative for the float64 reference's round-off.

**Soundness** (``test_emulation_within_bound``, ``test_clipped_signals_within_bound``): the bank, int16 and float32, at every
ROW_CONFIGS window plus 800 / 200.  Full rows: scipy's float32 FFT of z, the DC bin from float32 fmas as the kernels build
it, then the chroma stage in float32 in the generic kernel's order.  Clipped rows: the fp64 direct DFT with exact integer
phase reduction and float32 record values, rounded to float, then the chroma stage.  Spectra moved by the full bound in
each class's worst direction stay inside (``test_worst_direction_within_bound``).

**Sensitivity.**  Defects planted by hand in these emulations (not committed), over the bank at the windows above (101
accepted clips, 111 clipped rows) and the clipped-frame clips at the windows of ``test_clipped_signals_within_bound`` (88
clips); a clip counts when any of its entries fails:
* float32 twiddles in the clipped DFT: the bound fails on 0 of the 101 bank clips but 11 of the 88 clipped-frame clips
  (``clipped_clips``: the tones, at up to 3e8 times the bound); the flat check (1e-4 relative, 1e-6 absolute) on none;
* float32 accumulation in the clipped DFT: the bound fails on 5 bank clips (at up to 4x) and 24 clipped-frame clips (up to
  3e11x); the flat check on none;
* the phase index wrapped with ``ph > n`` (tw[n] then reads the sample array): the bound fails on 88 bank / 45 clipped
  clips, the flat check on 81 / 45;
* the DC bin rebuilt with w instead of n: bound 97 / 81, flat 94 / 76;
* a clipped frame zero-padded to w: bound 99 / 81, flat 99 / 81;
* one chroma tap moved to its neighbouring bin (first write wins in the scatter): bound 101 / 88, flat 101 / 86;
* sum X^2 without the DC bin: bound 101 / 84, flat 101 / 82.
On the H100, the clipped kernel built with ``sincospif`` twiddles, and again with float32 accumulation, fails 13 of 13
cases of tests/test_gpu_chroma_bounds.py (every row config and every clipped-kernel window; worst 8e8 and 838 times the
bound, on the tones) and passes all 21 flat chromagram checks of the GPU suite.
"""
import os
import subprocess

import numpy as np
import pytest
import scipy.fft

from oracle import st_oracle as O
from tests import host_exe
from tests import signals as SG
from tests.kernels import GENERIC_SWEEP, ROW_CONFIGS
from tests.parity import (DIV_REL, ROW_CLIPPED, ROW_EMPTY, ROW_FULL, _tables, check_chromagram_bounds, chromagram_bounds,
                          chromagram_rows, clip_norm, clipped_clips, clipped_targets, gamma, sum_depth)

CONFIGS = ROW_CONFIGS + [(16000, 800, 200)]
F = np.float32
EPS32 = F(O.EPS)
SMEM_CAP = 226 * 1024       # clipped-frame launcher's shared-memory cap (csrc/b200aa.cu), the per-CTA opt-in maximum less 1 KiB


def fmaf(a, b, c):
    """float32 fma: the product is exact in float64, the sum rounded there and then to float32 (a double rounding that
    may differ from a fused fma by one ulp, inside every bound here)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F)


def records(x):
    """(a, bp, m) as the float32 normalisation record holds them."""
    a, bp = clip_norm(x)
    xd = np.asarray(x, dtype=np.float64)
    m = float(np.rint(xd.mean())) if np.asarray(x).dtype == np.int16 else float(F(xd.mean()))
    return F(a), F(bp), F(m)


def chroma_taps(C):
    """Per class (bins, float32 weights) in ascending bin order."""
    return [(np.nonzero(C[j])[0], C[j][np.nonzero(C[j])[0]].astype(F)) for j in range(12)]


def chroma_stage(X, C, sxx_from=0):
    """Float32 chroma rows from float32 spectra X [T, K], in the generic / clipped kernels' order: lane-strided fma sums
    of X^2, a butterfly over 32 lanes, each class a sequential fma of its squared taps, one IEEE division."""
    T, K = X.shape
    m = -(-K // 32)
    Xp = np.zeros((T, 32 * m), dtype=F)
    Xp[:, sxx_from:K] = X[:, sxx_from:]
    lanes = np.zeros((T, 32), dtype=F)
    for i in range(m):
        v = Xp[:, 32 * i:32 * (i + 1)]
        lanes = fmaf(v, v, lanes)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, idx ^ o]).astype(F)
    sxx = lanes[:, 0]
    out = np.zeros((T, 12), dtype=F)
    for j, (bins, wts) in enumerate(chroma_taps(C)):
        acc = np.zeros(T, dtype=F)
        for b, wt in zip(bins, wts):
            v = X[:, b]
            acc = fmaf((v * v).astype(F), wt, acc)
        out[:, j] = acc
    return (out / np.where(sxx == 0, EPS32, sxx)[:, None]).astype(F)


def full_spectra(x, w, starts):
    """Float32 |X| / K of the full frames at ``starts`` as the row kernels build them: the float32 transform of d - d0 (d
    = x - m) scaled by a / K, the DC bin |a sum(d - d0) + w (a d0 + bp)| / K by float32 fmas."""
    x = np.asarray(x)
    a, bp, m = records(x)
    d = (x.astype(F) - m).astype(F)
    dfr = d[np.asarray(starts)[:, None] + np.arange(w)[None, :]]
    z = (dfr - dfr[:, :1]).astype(F)
    K = w // 2
    Z = scipy.fft.fft(z, axis=1)[:, :K]
    X = (np.abs(Z) * F(a / F(K))).astype(F)
    inner = fmaf(a, dfr[:, 0], bp)
    X[:, 0] = (np.abs(fmaf(a, Z[:, 0].real.astype(F), (F(w) * inner).astype(F))) / F(K)).astype(F)
    return X


def twiddles(n):
    """exp(-2 pi i j / n), j < n, in float64: (cos, -sin) of pi (2 j / n)."""
    t = np.pi * (2.0 * np.arange(n) / n)
    return np.cos(t), -np.sin(t)


def direct_dft(z, n, K, tw):
    """(re, im) [K] of sum_j z_j tw[j k mod n], fp64 accumulation."""
    ph = (np.arange(K)[:, None] * np.arange(n)[None, :]) % n
    return tw[0][ph] @ z, tw[1][ph] @ z


def clipped_spectrum(x, p, w):
    """Float32 |X| / K of the clipped frame x[p:] as clipped_chroma_kernel builds it."""
    x = np.asarray(x)
    a, bp, m = (float(v) for v in records(x))
    K = w // 2
    fr = x[p:].astype(np.float64)
    n = fr.size
    x0 = fr[0]
    z = fr - x0
    re, im = direct_dft(z, n, K, twiddles(n))
    mag = a * np.sqrt(re * re + im * im)
    mag[0] = abs(a * re[0] + n * (a * (x0 - m) + bp))
    return (mag / K).astype(F)


def emulate(x, fs, w, s):
    """Float32 chromagram rows [R, 12] of clip x through a row kernel and the clipped-frame kernel."""
    R, n_it, n_full, refused = chromagram_rows(x.size, w, s)
    C = _tables(fs, w // 2)[2]
    out = np.zeros((R, 12), dtype=F)
    if n_full:
        out[:n_full] = chroma_stage(full_spectra(x, w, w + s * np.arange(n_full)), C)
    if n_it > n_full:
        X = np.stack([clipped_spectrum(x, w + s * i, w) for i in range(n_full, n_it)])
        out[n_full:n_it] = chroma_stage(X, C)
    return out


def bank_clips(fs, w, s):
    return list(SG.bank(fs, w, s).items()) + list(SG.float_bank(fs, w, s).items())


CLIPPED_CPU = [(16000, 800, 200), (16000, 800, 400), (16000, 883, 300), (44100, 882, 441)]


@pytest.mark.parametrize("fs,w,s", CLIPPED_CPU, ids=["%d-%d-%d" % c for c in CLIPPED_CPU])
def test_clipped_signals_within_bound(fs, w, s):
    """The clipped-frame signals of the GPU module through the emulation: every row within its bound, the integer-mean
    run exactly zero."""
    worst = 0.0
    for n in clipped_targets(w, s):
        for name, x in clipped_clips(fs, w, s, n).items():
            cb = chromagram_bounds(x, fs, w, s)
            assert (cb.cls == ROW_CLIPPED).any(), (n, name)
            got = emulate(x, fs, w, s)
            r, u = check_chromagram_bounds(got, cb, "fs=%d w=%d s=%d, clipped length %d: %s" % (fs, w, s, n, name))
            assert not u, u
            worst = max(worst, r["clipped"])
            if name == "mean_run":
                assert not got[-1].any() and not cb.bound[-1].any(), n
    print("fs=%d w=%d s=%d clipped signals: worst clipped err / bound %.3g" % (fs, w, s, worst))


def oracle_chromagram(x, fs, w, s):
    try:
        return O.chromagram(x.astype(np.float64) if x.dtype == np.float32 else x, fs, w, s)[0]
    except ValueError:
        return None


@pytest.mark.parametrize("fs,w,s", CONFIGS, ids=["%d-%d-%d" % c for c in CONFIGS])
def test_emulation_within_bound(fs, w, s):
    """Every row class of the emulated kernels within the bound; the bound's reference is the oracle's chromagram."""
    worst, counts = {}, {}
    for name, x in bank_clips(fs, w, s):
        cb = chromagram_bounds(x, fs, w, s)
        ref = oracle_chromagram(x, fs, w, s)
        if cb.refused:
            assert ref is None or x.size - s - w < 0, name
            continue
        np.testing.assert_allclose(cb.ref, ref, rtol=1e-9, atol=1e-15, err_msg=name)
        r, u = check_chromagram_bounds(emulate(x, fs, w, s), cb, "float32 emulation, fs=%d w=%d s=%d: %s" % (fs, w, s, name))
        assert not u, (name, u)
        for k, v in r.items():
            worst[k] = max(worst.get(k, 0.0), v)
        for c in (ROW_FULL, ROW_CLIPPED, ROW_EMPTY):
            counts[c] = counts.get(c, 0) + int((cb.cls == c).sum())
    assert counts[ROW_FULL] and counts[ROW_CLIPPED], counts
    print("fs=%d w=%d s=%d: worst err / bound %s; rows (full, clipped, never filled) %s"
          % (fs, w, s, worst, [counts.get(c, 0) for c in (ROW_FULL, ROW_CLIPPED, ROW_EMPTY)]))


def _worst_moves(cb, x, fs, w, s):
    """Per row and class j, the float64 spectrum moved by the full bound in the direction that moves class j most: full
    rows along (C_j - c_j) X over bins 1 .. K-1 (norm eps_b) and eps_0 at DC, clipped rows by eps_k sgn(C_jk - c_j) in
    every bin; both signs, magnitudes kept >= 0."""
    from tests.parity import clipped_spectrum_reference, spectrum_reference
    K = w // 2
    C = _tables(fs, K)[2]
    R, n_it, n_full, _ = chromagram_rows(x.size, w, s)
    moves = []
    if n_full:
        X, eb, e0, flat = spectrum_reference(x, w + s * np.arange(n_full), w)
        eb = np.where(flat, 0.0, eb)
        for j in range(12):
            a = (C[j][None, :] - cb.ref[:n_full, j:j + 1]) * X
            a[:, 0] = 0
            nrm = np.linalg.norm(a, axis=1, keepdims=True)
            a = np.where(nrm > 0, a / np.where(nrm > 0, nrm, 1), 0)
            for sign in (1.0, -1.0):
                d = sign * eb[:, None] * a
                d[:, 0] = sign * np.sign(C[j, 0] - cb.ref[:n_full, j]) * e0
                moves.append((np.arange(n_full), np.maximum(X + d, 0.0)))
    for i in range(n_full, n_it):
        X, eps = clipped_spectrum_reference(x, w + s * i, K)
        for j in range(12):
            for sign in (1.0, -1.0):
                moves.append((np.array([i]), np.maximum(X + sign * eps * np.sign(C[j] - cb.ref[i, j]), 0.0)[None]))
    return C, moves


@pytest.mark.parametrize("fs,w,s", CONFIGS[::2], ids=["%d-%d-%d" % c for c in CONFIGS[::2]])
def test_worst_direction_within_bound(fs, w, s):
    for name, x in bank_clips(fs, w, s):
        cb = chromagram_bounds(x, fs, w, s)
        if cb.refused:
            continue
        C, moves = _worst_moves(cb, x, fs, w, s)
        for rows, Xq in moves:
            P = Xq ** 2
            E = P.sum(axis=1)
            got = cb.ref.copy()
            got[rows] = P @ C.T / np.where(E == 0, O.EPS, E)[:, None]
            check_chromagram_bounds(got, cb, "fs=%d w=%d s=%d %s: moved spectrum" % (fs, w, s, name))


def test_zero_and_constant_frames():
    """A frame-long run at the clip's exact integer mean (y = 0) gives exactly 0 with a zero bound, full or clipped; a
    constant frame elsewhere gives C[:, 0], with no transform allowance."""
    fs, w, s = 16000, 800, 400
    K = w // 2
    rng = np.random.default_rng(3)
    x = rng.integers(-3000, 3001, 3 * w + 600).astype(np.int64)    # rows: frames at 800, 1200, 1600, 2000 and 2400 (clipped)
    x[w:2 * w] = 0                                      # row 0: y = 0 once the clip mean is 0
    x[2 * w:3 * w] = 1234                               # row 2: constant, y != 0
    x[-600:] = 0                                        # row 4: a clipped frame of 600 samples, y = 0
    q, r = divmod(int(x.sum()), w)                      # the first w samples are in no row: make the clip mean exactly 0
    x[:w] -= q
    x[0] -= r
    assert np.abs(x).max() < 32768 and x.sum() == 0
    x = x.astype(np.int16)
    cb = chromagram_bounds(x, fs, w, s)
    assert list(cb.cls) == [ROW_FULL, ROW_FULL, ROW_FULL, ROW_FULL, ROW_CLIPPED], cb.cls
    for row in (0, 4):
        assert not cb.ref[row].any() and not cb.bound[row].any(), row
    C = _tables(fs, K)[2]
    np.testing.assert_allclose(cb.ref[2], C[:, 0], rtol=1e-15, atol=0)
    # only the chroma stage's roundings: zero where bin 0 is in no class
    stage = 1.01 * C[:, 0] * (gamma((C > 0).sum(axis=1) + 3) + gamma(sum_depth(K)) + DIV_REL) + 1e-12 * C[:, 0]
    assert (cb.bound[2] <= stage * (1 + 1e-9)).all(), (cb.bound[2], stage)
    got = emulate(x, fs, w, s)
    check_chromagram_bounds(got, cb, "zero and constant frames")
    assert not got[[0, 4]].any()


def test_sum_depth_covers_every_layout():
    """sum_depth(K) covers the sxx sums of every layout: the solo kernel's 16-lane sums of Kp = 32 odd(ceil(K / 32))
    padded bins (the deepest), the 32-lane layouts, then the shuffle levels and the fma."""
    for K in range(1, 10001):
        c = -(-K // 32) | 1
        assert 2 * c + 4 + 1 <= sum_depth(K) and c + 5 + 1 <= sum_depth(K) and -(-K // 32) + 5 + 1 <= sum_depth(K), K


@pytest.fixture(scope="module")
def lib():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib


TABLE_WINDOWS = sorted({(fs, w) for fs, w, _, _ in GENERIC_SWEEP} | {(fs, w) for fs, w, _ in CONFIGS}
                       | {(16000, 16000), (8000, 160), (16000, 8900), (16000, 8901)})


def test_chroma_tables_match_oracle(lib):
    """host_table(fs, w, 'chroma') is the oracle's operator at every sweep and row window; where the oracle raises, the
    table raises ValueError too.  Windows whose low bins have negative semitone indices (numpy's wrap) are among them."""
    negative = raised = 0
    for fs, w in TABLE_WINDOWS:
        K = w // 2
        try:
            ref = O.chroma_operator(fs, K)
        except ValueError:
            with pytest.raises(ValueError):
                lib.host_table(fs, w, "chroma")
            raised += 1
            continue
        np.testing.assert_allclose(lib.host_table(fs, w, "chroma"), ref, rtol=0, atol=1e-15, err_msg="fs=%d w=%d" % (fs, w))
        negative += int(O.chroma_tables(fs, K)[0].min() < 0)
    assert negative >= 3 and raised >= 3, (negative, raised)


def test_rows_rule_matches_library(tmp_path_factory):
    """parity.chromagram_rows is csrc/rows.cuh's rule (run on the host by tests/rows_host.cu) for every length 0 .. 3 w."""
    exe = host_exe.build(tmp_path_factory, "rows_host.cu", "-O1")
    configs = [(800, 400), (800, 200), (800, 100), (883, 300), (882, 441), (400, 160)]
    out = subprocess.run([exe], input="".join("%d %d %d\n" % (w, s, 3 * w) for w, s in configs), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.splitlines()
    for w, s in configs:
        lines.pop(0)
        for _ in range(3 * w + 1):
            n, _, _, _, _, cR, c_it, c_full, c_ref = (int(v) for v in lines.pop(0).split())
            R, n_it, n_full, refused = chromagram_rows(n, w, s)
            assert refused == bool(c_ref) and R == cR, (w, s, n)
            if not refused:
                assert (n_it, n_full) == (c_it, c_full), (w, s, n)


def test_clipped_kernel_scratch_boundary(tmp_path, tmp_path_factory):
    """clipped_chroma_kernel keeps its arrays (|X| row, w double2 twiddles, w double samples) in shared memory while
    clipped_bytes(w, w / 2) <= 226 KiB, else in global scratch: the last shared-memory window is 8 900, the first global one
    8 901 (tests/test_gpu_chroma_bounds.py runs both)."""
    src = tmp_path / "clipped_bytes.cu"
    src.write_text('#include <cstdio>\n#define B200AA_LAYOUT_ONLY 1\n#include "%s"\nint main() { for (int w = 2; w <= 20000; ++w) '
                   'printf("%%d %%zu\\n", w, b200aa::clipped_bytes(w, w / 2)); return 0; }\n'
                   % os.path.join(host_exe.ROOT, "pyaudioanalysis_b200", "csrc", "generic_kernel.cuh"))
    exe = host_exe.build(tmp_path_factory, str(src))
    sizes = {int(a): int(b) for a, b in (ln.split() for ln in subprocess.run([exe], capture_output=True, text=True).stdout.splitlines())}
    fits = [w for w, b in sizes.items() if b <= SMEM_CAP]
    assert max(fits) == 8900 and fits == list(range(2, 8901)), max(fits)
    assert sizes[8900] == 231408 and sizes[8901] == 231432

"""Shared comparison helpers for the GPU parity tests.

Tolerance (stated once, used everywhere): every feature column must satisfy
    |gpu - ref| <= RTOL * |ref| + ATOL      with RTOL = 1e-4, ATOL = 1e-5
(BASELINE.json north_star asks for 1e-4 rtol; the absolute term covers values that cross zero --
mfcc_2..13 and every delta column are differences of near-equal numbers -- see SURVEY.md 8d.)
Two rows are discrete: zcr moves in quanta of 0.5/(w-1) and spectral_rolloff in quanta of 1/K; a
float32-vs-float64 tie may move them by one quantum on a small fraction of frames, which is
counted and bounded separately.

The absolute term makes the feature check blind below ~1e-5: a quiet frame's energy (~1e-8) passes whatever its value.
Two row checks close that: ``check_energy_relative`` holds the energy row to RTOL with a negligible floor, and
``check_zcr_exact`` holds the zcr row of integer input to float32 rounding of the exact count.
``check_mid_propagated`` carries the per-frame tolerance through mid-term pooling (mean: mean of the frame tolerances,
std: their RMS).

``check_spectrum`` holds the magnitude spectrum |X[k]| / K of every frame, which every feature is built from, to a
float64 DFT under a bound derived from float32 FFT arithmetic (derivation: tests/test_gpu_spectra.py).
``feature_bounds`` / ``check_feature_bounds`` carry that bound, plus the float32 arithmetic of the feature stage, to a
bound on every entry of the 68 rows (derivation: tests/test_feature_bounds_cpu.py).
``chromagram_bounds`` / ``check_chromagram_bounds`` do the same for chromagram rows: full rows from the spectrum bound,
clipped rows from a per-bin model of the clipped-frame kernel's fp64 DFT (derivation: tests/test_chroma_bounds_cpu.py).

The GPU tests share the runs behind these checks: every clip of a batch under its spectrum bound for each kernel kind
(``pair_spectra``, ``row_spectra``, ``generic_spectra``), under its feature or chromagram bound (``batch_bounds``,
``ragged_bounds``, ``check_rows``, accumulated by ``note`` and printed by ``report``), the clips that end in clipped
chromagram frames (``clipped_clips``) and the exact check of a float32 clip record (``check_f32_clip``).
"""
import contextlib
import ctypes
import json
import math
from fractions import Fraction

import numpy as np

from tests.kernels import PAIR, ragged

RTOL, ATOL = 1e-4, 1e-5
ZCR_ROW, ENERGY_ROW, ROLLOFF_ROW = 0, 1, 7
MAX_FLIP_FRACTION = 2e-3
ENERGY_ATOL = 1e-12

# Known departures from the standard tolerance.  Each entry: the signal of tests/signals.py it applies to, the kernel
# kinds (2 pair, 3 solo, 1 CTA, 0 generic), the rows, the bound on max err / tol in those rows, and the ratio measured
# on one H100 80GB HBM3 (400 W power limit) by tests/test_gpu_adversarial.py.  Every other (signal, kernel, row) is held
# to the standard tolerance.  Constant frames are not an exception: their noise-defined reference values are replaced
# by the exact ones (tests/signals.patch_noise_defined).
EXCEPTIONS = [
    {"signal": "chirp_f32", "kinds": (3,), "rows": (13, 47), "bound": 2.0, "measured": 1.52,
     "reason": "float32 input, a chirp near 0.45 fs at 44.1 kHz: one frame's mfcc_6 (and its delta) near zero, where the "
               "absolute term governs, off by 2.0e-5 through the solo kernel's packed-real transform"},
    {"signal": "edge_impulses_f32", "kinds": (2,), "rows": (42,), "bound": 2.0, "measured": 1.13,
     "reason": "float32 input, window 960: one delta mfcc_1 near zero off by 1.15e-5 through the pair kernel"},
    {"signal": "small_f32", "kinds": (0, 2), "rows": (7, 41), "bound": 182.0, "measured": 181.8,
     "reason": "float32 input at 1e-3 full scale, window 960: a float32 tie moves one frame's rolloff by one quantum (1/K, "
               "39.5x the tolerance), and its delta on both sides; one flip counts three times against the flip limit"},
    {"signal": "edge_impulses", "kinds": (1,), "rows": (7, 41), "bound": 501.0, "measured": 500.0,
     "reason": "window 400, hop 200: a float32 tie moves one frame's rolloff by one quantum through the CTA kernel (50x the "
               "tolerance) and its delta on both sides (500x); one flip counts three times against the flip limit"},
]


def exception_bounds(signal, kind):
    """{row: bound on err / tol} of the EXCEPTIONS entries for one signal through one kernel kind."""
    out = {}
    for e in EXCEPTIONS:
        if e["signal"] == signal and kind in e["kinds"]:
            for r in e["rows"]:
                out[r] = max(out.get(r, 1.0), e["bound"])
    return out


def err_ratio(gpu, ref):
    """err / tol per entry under the standard tolerance."""
    gpu = np.asarray(gpu, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return np.abs(gpu - ref) / (RTOL * np.abs(ref) + ATOL)


def check_features(gpu, ref, K, what="", allow=None):
    """``allow``: {row: bound on err / tol} for the rows of an EXCEPTIONS entry (exception_bounds)."""
    gpu = np.asarray(gpu, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert gpu.shape == ref.shape, (what, gpu.shape, ref.shape)
    assert np.isfinite(gpu).all(), what + ": non-finite output"
    err = np.abs(gpu - ref)
    tol = RTOL * np.abs(ref) + ATOL
    if allow:
        tol = tol.copy()
        for r, bound in allow.items():
            if r < tol.shape[0]:
                tol[r] *= bound
    bad = err > tol
    F = ref.shape[0]
    flips = 0
    for r in (ROLLOFF_ROW, ROLLOFF_ROW + 34):
        if r < F and bad[r].any():
            q = err[r][bad[r]]
            assert (q <= (1.0 / K) * (2 if r >= 34 else 1) + 1e-6).all(), "%s: rolloff off by more than one quantum" % what
            flips += int(bad[r].sum())
            bad[r] = False
    assert flips <= max(2, MAX_FLIP_FRACTION * ref.shape[1] * 2), "%s: %d rolloff quantum flips" % (what, flips)
    if bad.any():
        rows = np.unique(np.nonzero(bad)[0])
        worst = [(int(r), float(err[r].max()), float((err[r] / tol[r]).max())) for r in rows]
        raise AssertionError("%s: rows outside tolerance (row, max abs err, max err/tol): %s" % (what, worst))
    return flips


def check_zcr_exact(gpu, ref, what=""):
    """zcr of integer input is an exact count of sign changes: the float32 result is that count rounded once,
    |gpu - ref| <= 2^-24 |ref|."""
    g = np.asarray(gpu, dtype=np.float64)[ZCR_ROW]
    r = np.asarray(ref, dtype=np.float64)[ZCR_ROW]
    bad = np.abs(g - r) > 2.0 ** -24 * np.abs(r)
    if bad.any():
        t = np.nonzero(bad)[0]
        raise AssertionError("%s: zcr not exact in %d frames, first %d: %r vs %r" % (what, t.size, t[0], g[t[0]], r[t[0]]))


def check_energy_relative(gpu, ref, what="", rtol=RTOL, atol=ENERGY_ATOL):
    """The energy row relative to each frame's own level, so that quiet frames count."""
    g = np.asarray(gpu, dtype=np.float64)[ENERGY_ROW]
    r = np.asarray(ref, dtype=np.float64)[ENERGY_ROW]
    bad = np.abs(g - r) > rtol * np.abs(r) + atol
    if bad.any():
        t = np.nonzero(bad)[0]
        rel = np.abs(g[t] - r[t]) / np.maximum(np.abs(r[t]), 1e-300)
        raise AssertionError("%s: energy off in %d frames, worst relative error %.3g (frame %d, ref %.3g)"
                             % (what, t.size, rel.max(), t[np.argmax(rel)], r[t[np.argmax(rel)]]))


def mid_slices(T, ratio, stepr):
    """(start, stop) of every mid-term window: the Python slice st[c : min(c + ratio, T)], c = 0, stepr, ...
    (MidTermFeatures.py:116-124; ratio may be 0 or negative there)."""
    return [slice(c, min(c + ratio, T)).indices(T)[:2] for c in range(0, T, stepr)]


def check_mid_propagated(mid, st_gpu, st_ref, ratio, stepr, K, what="", allow=None, ref_mid=None):
    """Mid-term matrix ``mid`` [2F, M] (pooled from ``st_gpu``) against pooling of the reference's short-term matrix
    ``st_ref`` [F, T], with the short-term tolerance propagated through the pooling.

    Frame t of row r may be off by tau = RTOL |ref| + ATOL (times the ``allow`` bound of the row, as in check_features);
    on a rolloff frame that check_features accepts as a flip, by one quantum 1/K (delta rolloff: two) instead.  A window
    mean may then be off by mean(tau) over the window, and a population std by rms(tau): std is 1-Lipschitz in the RMS
    norm, |std(x) - std(y)| <= rms(x - y).  Each output is also rounded to float32 once (2^-24 relative).  ``ref_mid``: the
    reference's own mid-term matrix, compared instead of the pooling of ``st_ref`` (which still gives the bounds)."""
    mid = np.asarray(mid, dtype=np.float64)
    g = np.asarray(st_gpu, dtype=np.float64)
    r = np.asarray(st_ref, dtype=np.float64)
    F, T = r.shape
    assert g.shape == r.shape, (what, g.shape, r.shape)
    win = mid_slices(T, ratio, stepr)
    assert mid.shape == (2 * F, len(win)), (what, mid.shape, (2 * F, len(win)))
    tau = RTOL * np.abs(r) + ATOL
    for row, bound in (allow or {}).items():
        if row < F:
            tau[row] *= bound
    for row in (ROLLOFF_ROW, ROLLOFF_ROW + 34):
        if row < F:
            quantum = (1.0 / K) * (2 if row >= 34 else 1) + 1e-6
            flip = np.abs(g[row] - r[row]) > tau[row]
            tau[row, flip] = quantum
    ref = np.zeros_like(mid)
    bound = np.zeros_like(mid)
    for j, (a, b) in enumerate(win):
        if b > a:
            seg = r[:, a:b]
            ref[:F, j], ref[F:, j] = seg.mean(axis=1), seg.std(axis=1)
            bound[:F, j] = tau[:, a:b].mean(axis=1)
            bound[F:, j] = np.sqrt((tau[:, a:b] ** 2).mean(axis=1))
    if ref_mid is not None:
        assert np.shape(ref_mid) == ref.shape, (what, np.shape(ref_mid), ref.shape)
        ref = np.asarray(ref_mid, dtype=np.float64)
    bound += 2.0 ** -24 * np.abs(ref)
    assert np.isfinite(mid).all(), what + ": non-finite mid-term output"
    err = np.abs(mid - ref)
    bad = err > bound
    if bad.any():
        rows, cols = np.nonzero(bad)
        k = int(np.argmax(err[bad] / bound[bad]))
        raise AssertionError("%s: %d mid-term entries outside the propagated tolerance, rows %s; worst (row %d, window %d): "
                             "%r vs %r, bound %.3g" % (what, rows.size, np.unique(rows)[:10].tolist(), rows[k], cols[k],
                                                       mid[rows[k], cols[k]], ref[rows[k], cols[k]], bound[rows[k], cols[k]]))


def check_close(gpu, ref, what="", rtol=RTOL, atol=ATOL):
    gpu = np.asarray(gpu, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert gpu.shape == ref.shape, (what, gpu.shape, ref.shape)
    np.testing.assert_allclose(gpu, ref, rtol=rtol, atol=atol, err_msg=what)


U32 = 2.0 ** -24        # unit round-off of float32
SPECTRUM_C = 8.0        # constant of the spectrum bound, fixed by the error analysis in tests/test_gpu_spectra.py


def spectrum_reference(x, starts, N):
    """Per frame (frame j = y[starts[j] : starts[j] + N], y = the normalised clip as O.spectrogram computes it): the
    float64 magnitudes |DFT|[0:K] / K, the bound on the 2-norm of the error in bins 1 .. K-1, the bound on the error of
    the DC bin, and whether the frame is constant.

    z = y_frame - y_frame[0] is what every kernel transforms; nu = sqrt(N) |z|_2 / K is the 2-norm of its whole
    spectrum on the output's scale (Parseval).  Bins:  C u ceil(log2 N) nu.  DC (a sum, then N times the first sample
    added back):  C u (|z|_1 + N |y_frame[0]|) / K.  float32 input rounds x - x[0] once per sample: u |y_frame|_2 is
    added to |z|_2."""
    from oracle import st_oracle as O
    f32 = np.asarray(x).dtype == np.float32
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    K = N // 2
    fr = np.stack([y[s:s + N] for s in starts]) if len(starts) else np.zeros((0, N))
    z = fr - fr[:, :1]
    # bins k >= 1 of y_frame and of z are the same numbers; from z a constant frame's are exactly 0, not float64 round-off
    ref = np.abs(np.fft.fft(z, axis=1)[:, :K]) / K
    ref[:, 0] = np.abs(fr.sum(axis=1)) / K
    nz = np.linalg.norm(z, axis=1)
    if f32:
        nz = nz + U32 * np.linalg.norm(fr, axis=1)
    levels = max(1, math.ceil(math.log2(N)))
    bins = SPECTRUM_C * U32 * levels * math.sqrt(N) * nz / K
    dc = SPECTRUM_C * U32 * (np.abs(z).sum(axis=1) + N * np.abs(fr[:, 0])) / K
    return ref, bins, dc, ~z.any(axis=1)


def check_spectrum(got, x, starts, N, what=""):
    """Rows ``got`` [len(starts), K] against spectrum_reference: the 2-norm of the error over bins 1 .. K-1 of every
    frame within its own bound, the DC bin within its own, and a constant frame's bins 1 .. K-1 exactly zero.
    Returns (worst bins err / bound, worst DC err / bound)."""
    got = np.asarray(got, dtype=np.float64)
    ref, bins, dc, flat = spectrum_reference(x, starts, N)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.isfinite(got).all(), what + ": non-finite spectrum"
    nonzero = np.nonzero(flat & (got[:, 1:] != 0).any(axis=1))[0]
    assert nonzero.size == 0, "%s: constant frames %s have non-zero bins beyond DC" % (what, nonzero[:10].tolist())
    e = np.linalg.norm(got[:, 1:] - ref[:, 1:], axis=1)
    d = np.abs(got[:, 0] - ref[:, 0])
    r = np.where(bins > 0, e / np.where(bins > 0, bins, 1.0), np.where(e > 0, np.inf, 0.0))
    rd = np.where(dc > 0, d / np.where(dc > 0, dc, 1.0), np.where(d > 0, np.inf, 0.0))
    bad = np.nonzero((r > 1.0) | (rd > 1.0))[0]
    if bad.size:
        j = bad[np.argmax(np.maximum(r, rd)[bad])]
        k = int(np.argmax(np.abs(got[j] - ref[j])))
        raise AssertionError("%s: %d of %d frames outside the spectrum bound; worst frame %d (start %d): bins err / bound "
                             "%.3g, DC err / bound %.3g, largest error in bin %d: %r vs %r"
                             % (what, bad.size, len(starts), j, starts[j], r[j], rd[j], k, got[j, k], ref[j, k]))
    return (float(r.max()) if r.size else 0.0), (float(rd.max()) if rd.size else 0.0)


def check_spectrogram_rows(got, x, w, s, what=""):
    """Spectrogram rows of clip x (row r transforms the frame at w + r s, ShortTermFeatures.py:413-415) under
    check_spectrum; the rows the reference's loop never reaches are exactly zero."""
    got = np.asarray(got, dtype=np.float64)
    starts = np.arange(w, len(x) - w + 1, s)
    assert got.shape == (int((len(x) - w) / s) + 1, w // 2), (what, got.shape)
    assert not got[len(starts):].any(), what + ": rows past the last full frame are not zero"
    return check_spectrum(got[:len(starts)], x, starts, w, what)


# ---------------------------------------------------------------------------------------------------------------------
# Per-entry bound of the 68 feature rows, carried from the spectrum bound (derivation: tests/test_feature_bounds_cpu.py)
LOG2_ABS = 2.0 ** -22   # lg2.approx.f32 (__log2f): absolute error 2^-22 on [0.5, 2], else 2 ulp of the result
DIV_REL = 4 * U32       # __fdividef: 2 ulp
SQRT_REL = 5 * U32      # x * rsqrt.approx(x): 2 ulp and one rounding; sqrt.approx / sqrtf: 2 ulp assumed
MARGIN = 1.01           # products of (1 + relative error) terms, kept to first order, are covered by 1 %
F64_REL = 1e-12         # round-off of the float64 reference itself (sums of at most ~10^4 terms)
ROW_GROUPS = {"time": (0, 1, 2), "spectral": (3, 4, 5, 6, 7), "mfcc": tuple(range(8, 21)), "chroma": tuple(range(21, 34))}


def gamma(n):
    """gamma_n = n u / (1 - n u): a float32 sum of non-negative terms whose every term passes through at most n
    roundings errs by at most gamma_n times the sum (Higham, Accuracy and Stability, 2nd ed., section 3.1)."""
    n = np.asarray(n, dtype=np.float64)
    return n * U32 / (1.0 - n * U32)


def sum_depth(n):
    """Roundings a term of a float32 sum over n values (bins or samples) passes through in any kernel: per-lane
    sequential chunks of at most ceil(n / 16) terms (16-lane half-warp layouts; 32-lane layouts hold half as many),
    then at most 5 shuffle levels, the chunk's split into entropy parts and their sum, and the fma / product roundings
    of the term itself."""
    return math.ceil(n / 16) + 12


def _lin(a, e0, eb):
    """max |sum_k a_k d_k| over |d_0| <= e0, |d_1..K-1|_2 <= eb; a [..., K], e0 / eb broadcast against a[..., 0]."""
    return np.abs(a[..., 0]) * e0 + np.linalg.norm(a[..., 1:], axis=-1) * eb


def _quad(a, X, e0, eb):
    """max |sum_k a_k ((X_k + d_k)^2 - X_k^2)| over the same set: 2 |a X|_2 eb + max |a| eb^2, DC apart."""
    return (np.abs(a[..., 0]) * (2 * X[..., 0] * e0 + e0 ** 2) + 2 * np.linalg.norm((a * X)[..., 1:], axis=-1) * eb
            + np.abs(a[..., 1:]).max(axis=-1) * eb ** 2)


def _ratio_den(den, dden):
    """den - dden where it stays positive, else nan (the interval of the denominator reaches 0)."""
    return np.where(den - dden > 0, den - dden, np.nan)


def _h(s):
    return -s * np.log2(s + O_EPS)


O_EPS = np.finfo(np.float64).eps


def _entropy_bound(s, ds):
    """Bound on |H' - H|, H = sum_j h(s_j), h(s) = -s log2(s + eps), each s_j' within ds_j of s_j (nan: unbounded).
    h is concave on [0, inf) with its maximum at ~1/e, so over an interval its extremes are the endpoints and, where
    the interval holds it, the maximum.  Plus the float32 evaluation of each term: lg2.approx's error times s, and two
    roundings of the product and of the 10-term sum (gamma_12)."""
    lo = np.maximum(s - ds, 0.0)
    hi = s + ds
    top = np.where((lo <= 1 / math.e) & (hi >= 1 / math.e), _h(1 / math.e), np.maximum(_h(lo), _h(hi)))
    dev = np.maximum(_h(s) - np.minimum(_h(lo), _h(hi)), top - _h(s))
    lg = np.maximum(1.0, np.abs(np.log2(lo + O_EPS)))
    dev = dev + hi * LOG2_ABS * lg + gamma(12) * (np.abs(_h(s)) + dev)
    return dev.sum(axis=-1)


def _quad_bins(a, X, eps):
    """max |sum_k a_k ((X_k + d_k)^2 - X_k^2)| over |d_k| <= eps_k, bin by bin: sum |a_k| (2 X_k eps_k + eps_k^2)."""
    return (np.abs(a) * (2 * X * eps + eps ** 2)).sum(axis=-1)


def chroma_bound(X, C, cj, e0=None, eb=None, eps=None):
    """Per-entry bound [T, 12] on the chroma classes c_j = (C X^2)_j / E, E = sum X^2 (E == 0: divided by eps, as the
    reference does) that a kernel may return for frames whose float64 spectrum is X [T, K] and whose float64 classes are
    cj [T, 12]; nan where the interval of E reaches 0 (unbounded).

    Transform error, either the ball of spectrum_reference (|d_0| <= e0, |d_1..K-1|_2 <= eb, a float32 FFT) or per bin
    (|d_k| <= eps[:, k], the clipped-frame kernel's fp64 DFT): carried with centred weights C_j - c_j through the squares
    (_quad / _quad_bins) over E - dE.  Float32 chroma stage: each class a sequential fma of its squared taps (gamma(taps +
    3)), sum X^2 at depth sum_depth(K) (gamma; covers the 16-lane sums of the solo kernel's Kp-padded rows, the deepest
    layout), and one division (DIV_REL covers IEEE division and __fdividef)."""
    K = X.shape[1]
    Et = (X ** 2).sum(axis=1)
    w = C[None] - cj[:, :, None]                                               # [T, 12, K]
    if eps is None:
        dEt = _quad(np.ones(K), X, e0, eb)
        num = _quad(w, X[:, None, :], e0[:, None], eb[:, None])
    else:
        dEt = _quad_bins(np.ones(K), X, eps)
        num = _quad_bins(w, X[:, None, :], eps[:, None, :])
    dc_t = num / _ratio_den(np.where(Et == 0, O_EPS, Et), dEt)[:, None]
    dc_a = MARGIN * cj * (gamma((C > 0).sum(axis=1) + 3)[None, :] + gamma(sum_depth(K)) + DIV_REL)
    return dc_t + dc_a


class FeatureBounds:
    """feature_bounds' result for one clip: ``ref`` [F, T] float64 reference, ``bound`` [F, T] per-entry bound (inf where
    unbounded), ``roll`` [2, T] admissible rolloff quanta (lo, hi) of every frame, ``unbounded`` {reason: count} and
    ``K``."""

    def __init__(self, ref, bound, roll, unbounded, K):
        self.ref, self.bound, self.roll, self.unbounded, self.K = ref, bound, roll, unbounded, K


_TABLES = {}


def _tables(fs, K):
    from oracle import st_oracle as O
    if (fs, K) not in _TABLES:
        _TABLES[(fs, K)] = (O.mel_filterbank(fs, K), O.dct_matrix(), O.chroma_operator(fs, K))
    return _TABLES[(fs, K)]


def clip_norm(x):
    """(a, bp, ambiguity) of the kernels' normalisation y = a (x - m) + bp in float64: a = 1 / (max |x - mean| +
    2^15 1e-10), m the clip centre exact in float (the rounded mean of int16, the float32 mean of float32), bp = a (m -
    mean)."""
    xd = np.asarray(x, dtype=np.float64)
    mean = xd.sum() / xd.size
    a = 1.0 / (max(xd.max() - mean, mean - xd.min()) + 32768.0 * 1e-10)
    m = float(np.rint(mean)) if np.asarray(x).dtype == np.int16 else float(np.float32(mean))
    return a, a * (m - mean)


def feature_bounds(x, fs, w, s, deltas=False):
    """The float64 reference of every short-term feature of clip x at (fs, w, s) and a per-entry bound on what a float32
    kernel may return: the spectrum bound of spectrum_reference carried through each feature, plus the float32
    arithmetic of the feature stage.  Derivation and error model: tests/test_feature_bounds_cpu.py."""
    from oracle import st_oracle as O
    x = np.asarray(x)
    f32 = x.dtype == np.float32
    K = w // 2
    T = O.frame_count(len(x), w, s)
    starts = s * np.arange(T)
    X, eb, e0, flat = spectrum_reference(x, starts, w)
    eb = np.where(flat, 0.0, eb)                       # a constant frame's bins 1 .. K-1 are exactly zero
    y = O.normalize_clip(x.astype(np.float64))
    fr = np.stack([y[a:a + w] for a in starts])
    ref = O.base_features_from_frames(fr, X, fs)
    M, D, C = _tables(fs, K)
    bound = np.zeros_like(ref)
    unb = {}
    ebc, e0c = eb[:, None], e0[:, None]
    gK = gamma(sum_depth(K))
    k1 = np.arange(1, K + 1) / K

    def unbounded(rows, mask, reason):
        if mask.any():
            bound[np.ix_(rows, np.nonzero(mask)[0])] = np.inf
            unb[reason] = unb.get(reason, 0) + int(mask.sum()) * len(rows)

    # ---- time domain: per-sample error of y = a (x - m) + bp in float32 (a, bp rounded; x - m rounded for float32
    # input; the generic kernel rebuilds x - m as (x - m - d0) + d0), then float32 sums
    a, bp = clip_norm(x)
    beta = MARGIN * 4 * U32 * (np.abs(fr) + np.abs(fr[:, :1]) + abs(bp))
    dq = 2 * np.abs(fr) * beta + beta ** 2                                   # bound on |y'^2 - y^2| per sample
    E = (fr ** 2).sum(axis=1)
    dE = dq.sum(axis=1)
    gN = gamma(sum_depth(w))
    flips_amb = (np.abs(fr) <= beta).sum(axis=1) if f32 else 0              # samples whose sign class may differ
    bound[0] = 2 * U32 * np.abs(ref[0]) + flips_amb * 2.0 / (w - 1)
    bound[1] = MARGIN * (dE + gN * (E + dE)) / w + 2 * U32 * ref[1]
    L = w // 10
    blk = np.arange(w) // L if L > 0 else np.full(w, 10)
    sj = np.stack([(fr[:, blk == j] ** 2).sum(axis=1) for j in range(10)], axis=1) / (E + O_EPS)[:, None]
    ind = (blk[None, :] == np.arange(10)[:, None]).astype(np.float64)        # [10, w]
    num = np.einsum("jn,tn->tj", np.abs(ind), dq) + sj * dE[:, None]         # |1_B - s_j| <= 1_B + s_j
    ds = num / _ratio_den(E + O_EPS, dE)[:, None] + sj * (2 * gN + 6 * U32)
    bound[2] = _entropy_bound(sj, ds)

    # ---- spectral rows from |X|: sums, ratios, square roots
    S = X.sum(axis=1)
    dS = _lin(np.ones(K), e0, eb)
    Sd = _ratio_den(S, dS)
    cen = np.where(S > 0, (X * k1).sum(axis=1) / np.where(S > 0, S, 1), 0.0)
    dcen_t = _lin(k1[None, :] - cen[:, None], e0, eb) / Sd
    dcen_a = MARGIN * cen * (2 * gK + 7 * U32)
    bound[3] = np.where(S > 0, dcen_t + dcen_a, 0.0)
    V = np.where(S > 0, ((k1[None, :] - cen[:, None]) ** 2 * X).sum(axis=1) / np.where(S > 0, S, 1), 0.0)
    dV_t = _lin((k1[None, :] - cen[:, None]) ** 2 - V[:, None], e0, eb) / Sd + dcen_t ** 2
    eta = (math.ceil(K / 16) + 4) * U32              # drift of (k + 1) / K - cen stepped across a lane's bins
    sp = V * S
    extra = dcen_a ** 2 * S + eta ** 2 * S + 2 * eta * np.sqrt(sp * S) + 2 * dcen_a * eta * S
    dV_a = MARGIN * ((extra + gK * (sp + extra)) / np.where(S > 0, S, 1) + (gK + DIV_REL + U32) * (V + extra / np.where(S > 0, S, 1)))
    dV = dV_t + dV_a
    spr = np.sqrt(V)
    # both sides: where V < dV the interval is cut at 0 below and the side above is the larger one
    bound[4] = np.where(S > 0, np.maximum(np.sqrt(V + dV) - spr, spr - np.sqrt(np.maximum(V - dV, 0.0)))
                        + SQRT_REL * np.sqrt(V + dV), 0.0)
    # spectral entropy: 10 blocks of K // 10 bins over the total of all K bins
    P = X ** 2
    Et = P.sum(axis=1)
    dEt = _quad(np.ones(K), X, e0, eb)
    Lb = K // 10
    bblk = np.arange(K) // Lb if Lb > 0 else np.full(K, 10)
    Bm = (bblk[None, :] == np.arange(10)[:, None]).astype(np.float64)       # [10, K]
    sjs = (P @ Bm.T) / (Et + O_EPS)[:, None]
    ds = _quad(Bm[None] - sjs[:, :, None], X[:, None, :], e0c, ebc) / _ratio_den(Et + O_EPS, dEt)[:, None]
    bound[5] = _entropy_bound(sjs, ds + sjs * (2 * gK + 6 * U32))
    # flux: sqrt(flux) = |X / Sn - Xp / Sp|_2, Sn = S + K eps; each side moves by at most (|d|_2 + |X / Sn|_2 dS) / (Sn - dS)
    Sn = S + K * O_EPS
    nrm = np.linalg.norm(X, axis=1) / Sn
    Dt = (np.sqrt(e0 ** 2 + eb ** 2) + nrm * dS) / _ratio_den(Sn, dS) + MARGIN * (gK + 7 * U32) * nrm
    Dp = np.concatenate([Dt[:1], Dt[:-1]])
    rf = np.sqrt(ref[6])
    bound[6] = (rf + Dt + Dp) ** 2 * (1 + gK + 2 * U32) - ref[6]
    # rolloff: first k with g_k = cumsum_k(X^2) + eps - 0.9 E > 0; g_k is a weighted sum of squares with weights
    # 1[j <= k] - 0.9, plus the float32 prefix (lane chunks, a shuffle scan, one subtraction) and 0.90f
    Pc = np.cumsum(P, axis=1)
    g = Pc + O_EPS - 0.9 * Et[:, None]
    aX2 = 0.01 * (Pc - P[:, :1]) + 0.81 * (Et[:, None] - Pc)
    b = (0.1 * (2 * X[:, :1] * e0c + e0c ** 2) + 2 * np.sqrt(np.maximum(aX2, 0.0)) * ebc + 0.9 * ebc ** 2
         + MARGIN * (gamma(sum_depth(K) + 2) * (Pc + 0.9 * Et[:, None]) + U32 * 0.9 * Et[:, None]))
    first = lambda c: np.where(c.any(axis=1), np.argmax(c, axis=1), -1)
    lo, hi = first(g + b > 0), first(g - b > 0)
    lo = np.where((lo < 0) | (hi < 0), 0, lo)
    hi = np.where(hi < 0, K - 1, hi)
    roll = np.stack([lo, hi])
    # mfcc: mel bands (linear, non-negative taps; each tap sum sequential in float32), log10 (lg2.approx * log10(2) or
    # log10f, 2 ulp), DCT (float32 table and sums around a constant offset of the log-mel values)
    m = X @ M.T                                                                # [T, 40]
    dm = _lin(M[None], e0c, ebc) + MARGIN * gamma((M > 0).sum(axis=1) + 2)[None, :] * m
    lm = np.log10(m + O_EPS)
    lo_m = m - dm
    mel_unb = (dm > 0) & (lo_m <= 0)
    dL = np.where(mel_unb, 0.0, lm - np.log10(np.maximum(lo_m, 0.0) + O_EPS))
    l2 = np.maximum(1.0, np.abs(np.log2(np.maximum(lo_m, 0.0) + O_EPS)))
    dL = dL + math.log10(2.0) * LOG2_ABS * l2 + 3 * U32 * np.abs(lm)
    Lrange = lm.max(axis=1) - lm.min(axis=1)
    Lmax = np.abs(lm).max(axis=1)
    aD = np.abs(D)
    g48 = gamma(48)
    dmf = dL @ aD.T + g48 * aD.sum(axis=1)[None, :] * (Lrange + gamma(8) * Lmax)[:, None]
    dmf[:, 0] += g48 * 6.33 * Lmax
    bound[8:21] = dmf.T + F64_REL * (np.abs(lm) @ aD.T).T
    unbounded(list(range(8, 21)), mel_unb.any(axis=1), "a mel band's interval contains 0 (log10(m + eps))")
    cj = ref[21:33].T                                                          # [T, 12]
    dcj = chroma_bound(X, C, cj, e0=e0, eb=eb)
    bound[21:33] = dcj.T
    # chroma_std: 1-Lipschitz in the RMS norm, then its own float32 mean (12 terms), squares and square root
    mu_e = gamma(6) * cj.mean(axis=1)
    bound[33] = np.sqrt((dcj ** 2).mean(axis=1)) + MARGIN * (mu_e + (gamma(8) + SQRT_REL) * (ref[33] + mu_e))
    unbounded([3, 4, 6], np.isnan(Sd), "sum |X| interval contains 0")
    unbounded([5, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33], np.isnan(_ratio_den(Et + O_EPS, dEt)) & (Et > 0),
              "sum X^2 interval contains 0")
    bound = np.where(np.isnan(bound), np.inf, bound)
    bound += F64_REL * np.abs(ref)
    if deltas:
        d = np.zeros_like(ref)
        d[:, 1:] = ref[:, 1:] - ref[:, :-1]
        db = np.zeros_like(bound)
        db[:, 1:] = bound[:, 1:] + bound[:, :-1]
        db[:, 1:] += 2 * U32 * (np.abs(d[:, 1:]) + db[:, 1:])
        for reason in list(unb):
            unb["delta: " + reason] = unb[reason]
        ref, bound = np.concatenate([ref, d]), np.concatenate([bound, db])
    return FeatureBounds(ref, bound, roll, unb, K)


def check_feature_bounds(got, fb, what="", roll_slack=4 * U32):
    """Rows ``got`` [F, T] against a FeatureBounds: every bounded entry within its bound, rolloff (and its delta) a whole
    number of quanta inside the admissible range (within roll_slack of it), no exception lists and no flip allowance.  Returns ({row group:
    worst err / bound}, {reason: unbounded entries})."""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == fb.ref.shape, (what, got.shape, fb.ref.shape)
    assert np.isfinite(got).all(), what + ": non-finite output"
    F, T = got.shape
    K = fb.K
    err = np.abs(got - fb.ref)
    fin = np.isfinite(fb.bound)
    ratio = np.where(fin, err / np.where(fb.bound > 0, fb.bound, 1.0), 0.0)
    ratio = np.where(fin & (fb.bound == 0), np.where(err > 0, np.inf, 0.0), ratio)
    lo, hi = fb.roll
    for r in (ROLLOFF_ROW, ROLLOFF_ROW + 34):
        if r >= F:
            continue
        q = np.rint(got[r] * K)
        if r == ROLLOFF_ROW:
            qlo, qhi, scale = lo, hi, q
        else:
            qlo = np.concatenate([[0], lo[1:] - hi[:-1]])
            qhi = np.concatenate([[0], hi[1:] - lo[:-1]])
            scale = np.abs(fb.ref[ROLLOFF_ROW] * K) + np.abs(np.concatenate([[0], fb.ref[ROLLOFF_ROW, :-1] * K]))
        off = (q < qlo) | (q > qhi) | (np.abs(got[r] * K - q) > roll_slack * (scale + 1))
        if off.any():
            t = int(np.nonzero(off)[0][0])
            raise AssertionError("%s: row %d (rolloff) outside its admissible quanta in %d frames, first %d: %r quanta, "
                                 "admissible %d .. %d" % (what, r, int(off.sum()), t, got[r, t] * K, qlo[t], qhi[t]))
        ratio[r] = 0.0
    bad = ratio > 1.0
    if bad.any():
        rows, cols = np.nonzero(bad)
        k = int(np.argmax(ratio[bad]))
        raise AssertionError("%s: %d entries outside the feature bound, rows %s; worst (row %d, frame %d): %r vs %r, bound "
                             "%.3g (err / bound %.3g)" % (what, rows.size, np.unique(rows)[:12].tolist(), rows[k], cols[k],
                                                        got[rows[k], cols[k]], fb.ref[rows[k], cols[k]],
                                                        fb.bound[rows[k], cols[k]], ratio[rows[k], cols[k]]))
    worst = {name: float(ratio[[r for r in rows if r < F]].max()) if T else 0.0 for name, rows in ROW_GROUPS.items()}
    if F > 34:
        worst["deltas"] = float(ratio[34:].max()) if T else 0.0
    return worst, dict(fb.unbounded)


# ---------------------------------------------------------------------------------------------------------------------
# Per-entry bound of chromagram rows, full-frame and clipped (derivation: tests/test_chroma_bounds_cpu.py)
U64 = 2.0 ** -53        # unit round-off of float64
TWIDDLE_ABS = (4 + 2 * math.pi) * U64   # sincospi(2j / n), per component: 2 ulp (< 4 u64 on [-1, 1]) + the rounded quotient
REF_FFT_C = 8.0         # numpy's float64 FFT of the reference, the same form as SPECTRUM_C
ROW_FULL, ROW_CLIPPED, ROW_EMPTY = 0, 1, 2
ROW_CLASS_NAMES = {ROW_FULL: "full", ROW_CLIPPED: "clipped", ROW_EMPTY: "never filled"}


def gamma64(n):
    n = np.asarray(n, dtype=np.float64)
    return n * U64 / (1.0 - n * U64)


def chromagram_rows(n, w, s):
    """csrc/rows.cuh's chromagram rule restated: (R, n_it, n_full, refused) for a clip of n samples."""
    R = int((n - s - w) / s) + 1
    n_it = min(R, len(range(w, n - s, s))) if R > 0 else 0
    n_full = min(n_it, (n - 2 * w) // s + 1) if n >= 2 * w else 0
    refused = R <= 0 or n - s - w < 0 or (n_it > n_full and n - (w + (n_it - 1) * s) < w // 2)
    return R, n_it, n_full, refused


class ChromaBounds:
    """chromagram_bounds' result for one clip: ``ref`` [R, 12] float64 reference, ``bound`` [R, 12] per-entry bound (inf
    where unbounded), ``cls`` [R] row class (ROW_FULL, ROW_CLIPPED, ROW_EMPTY), ``refused`` (the single-clip entry point
    refuses the clip: no rows) and ``unbounded`` {reason: entries}."""

    def __init__(self, ref, bound, cls, refused, unbounded):
        self.ref, self.bound, self.cls, self.refused, self.unbounded = ref, bound, cls, refused, unbounded


def _exact_sum(v):
    """The exact sum of int16 / float32 values as a Fraction."""
    v = np.asarray(v)
    if v.dtype == np.int16:
        return Fraction(int(v.astype(np.int64).sum()))
    return sum(map(Fraction, v.astype(np.float64).tolist()), Fraction(0))


def clip_record_error(x):
    """(a, mean, mean_q, alpha, dmean) of the kernels' normalisation record of clip x: the float64 a of clip_norm at the
    rounded mean, that mean, the exact mean (a Fraction), the relative error alpha of the float32 record value a, and
    dmean, a bound on the error of the kernels' fp64 mean: an exact int64 sum divided once for int16 input (the same
    rounded quotient as here), a float64 sum in any order for float32.  The record's a is 1 / (maxdev + c) evaluated in
    fp64 from that mean (maxdev moves by dmean) and rounded to float32."""
    xd = np.asarray(x, dtype=np.float64)
    n = xd.size
    mean_q = _exact_sum(x) / n
    mean = float(mean_q)
    if np.asarray(x).dtype == np.int16:
        dmean = float(abs(Fraction(mean) - mean_q))
    else:
        dmean = float(gamma64(n)) * math.fsum(np.abs(xd)) / n + 2 * U64 * abs(mean)
    den = max(xd.max() - mean, mean - xd.min()) + 32768.0 * 1e-10
    a = 1.0 / den
    alpha = MARGIN * (U32 + dmean / den + 4 * U64)
    return a, mean, mean_q, alpha, dmean


def clipped_spectrum_reference(x, p, K, rec=None):
    """The clipped frame y[p:] of clip x (n = len(x) - p samples, K <= n): float64 |DFT|[0:K] / K of the normalised
    frame, and eps [K], a per-bin bound on |kernel - reference| for clipped_chroma_kernel's arithmetic (derivation:
    tests/test_chroma_bounds_cpu.py), the reference's own error included.  ``rec``: clip_record_error(x), if at hand."""
    xd = np.asarray(x, dtype=np.float64)
    f32 = np.asarray(x).dtype == np.float32
    a, mean, mean_q, alpha, dmean = rec or clip_record_error(x)
    fr = xd[p:]
    n = fr.size
    z = fr - fr[0]                                               # exact: a difference of two int16 / float32 values
    z1 = np.abs(z).sum()
    D = np.abs(np.fft.fft(z)[:K])                                # |DFT z|, bins k >= 1 of the frame's DFT
    S = float(_exact_sum(np.asarray(x)[p:]) - n * mean_q)         # sum of x - mean over the frame, rounded once
    D[0] = abs(S)
    X = a * D / K
    # |m - mean| of the record's centre: for int16 the kernels round the same fp64 mean to the nearest integer, for float32
    # input they round their own fp64 mean (within dmean) to float
    dm = U32 * (abs(mean) + dmean) + dmean if f32 else abs(float(np.rint(mean)) - mean) + dmean
    # bins k >= 1: (re, im) err by (gamma64(n + 2) + twiddle) |z|_1 each; a * sqrt(re^2 + im^2) by 4 u64 more and a's alpha
    dft = math.sqrt(2.0) * (float(gamma64(n + 2)) + TWIDDLE_ABS) * z1
    eps = a * (alpha * D + (1 + alpha) * dft + 4 * U64 * D)
    # DC: a re + n (a (x0 - m) + bp) in fp64 from the float32 record: (a' - a) sum(x - m) + n (bp' - bp), plus the sum
    # re (n additions) and the roundings of the expression
    dbp = a * ((U32 + alpha) * dm + dmean)
    eps[0] = (alpha * a * (abs(S) + n * dm) + n * dbp + a * float(gamma64(n + 2)) * z1
              + 8 * U64 * a * (z1 + n * (abs(fr[0] - mean) + dm)))
    # the reference's own error: numpy's FFT of z (bins), the rounding of S and of a S (DC), and a from the rounded mean
    ref_err = a * REF_FFT_C * U64 * max(1, math.ceil(math.log2(n))) * math.sqrt(n) * np.linalg.norm(z) + 4 * U64 * a * D
    ref_err[0] = 2 * U64 * a * abs(S)
    ref_err = ref_err + (2 * U64 * abs(mean) * a + 2 * U64) * a * D          # a = 1 / den moves by dmean / den
    eps = MARGIN * (eps + ref_err) / K
    # the float64 magnitude divided by K, rounded to float once
    eps = eps + U32 * (X + eps) + 2 * U64 * X
    return X, eps


def chromagram_bounds(x, fs, w, s):
    """The float64 reference of the chromagram rows of clip x at (fs, w, s), a per-entry bound on what the kernels may
    return, and the row class of each row.

    * full rows (frame at w + r s, all w samples): the spectrum_reference ball at those starts through chroma_bound;
    * clipped rows (n = len - (w + r s) samples, K <= n < w): clipped_spectrum_reference's per-bin bound through
      chroma_bound;
    * rows the reference's loop never fills: exactly 0.
    A frame whose spectrum is exactly 0 gets exactly 0 (the EPS branch) and a constant frame its DC bin's class weights,
    both up to the float32 chroma stage only.  Derivation: tests/test_chroma_bounds_cpu.py."""
    from oracle import st_oracle as O
    x = np.asarray(x)
    K = w // 2
    R, n_it, n_full, refused = chromagram_rows(x.size, w, s)
    if refused:
        return ChromaBounds(np.zeros((0, 12)), np.zeros((0, 12)), np.zeros(0, dtype=int), True, {})
    C = _tables(fs, K)[2]
    ref = np.zeros((R, 12))
    bound = np.zeros((R, 12))
    cls = np.full(R, ROW_EMPTY)
    unb = {}

    def classes(X):
        Et = (X ** 2).sum(axis=1)
        return (X ** 2) @ C.T / np.where(Et == 0, O_EPS, Et)[:, None]

    if n_full:
        starts = w + s * np.arange(n_full)
        X, eb, e0, flat = spectrum_reference(x, starts, w)
        eb = np.where(flat, 0.0, eb)                   # a constant frame's bins 1 .. K-1 are exactly zero
        cj = classes(X)
        ref[:n_full] = cj
        bound[:n_full] = chroma_bound(X, C, cj, e0=e0, eb=eb)
        cls[:n_full] = ROW_FULL
    if n_it > n_full:
        rows = np.arange(n_full, n_it)
        rec = clip_record_error(x)
        XE = [clipped_spectrum_reference(x, w + s * i, K, rec) for i in rows]
        X = np.stack([v[0] for v in XE])
        eps = np.stack([v[1] for v in XE])
        cj = classes(X)
        ref[rows] = cj
        bound[rows] = chroma_bound(X, C, cj, eps=eps)
        cls[rows] = ROW_CLIPPED
    nan = np.isnan(bound).any(axis=1)
    if nan.any():
        unb["sum X^2 interval contains 0"] = int(nan.sum()) * 12
    bound = np.where(np.isnan(bound), np.inf, bound)
    bound += F64_REL * np.abs(ref)
    return ChromaBounds(ref, bound, cls, False, unb)


def check_chromagram_bounds(got, cb, what=""):
    """Rows ``got`` [R, 12] against a ChromaBounds: every bounded entry within its bound (a zero bound: exactly equal),
    rows never filled exactly 0.  Returns ({row class name: worst err / bound}, {reason: unbounded entries})."""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == cb.ref.shape, (what, got.shape, cb.ref.shape)
    assert np.isfinite(got).all(), what + ": non-finite output"
    err = np.abs(got - cb.ref)
    fin = np.isfinite(cb.bound)
    ratio = np.where(fin, err / np.where(cb.bound > 0, cb.bound, 1.0), 0.0)
    ratio = np.where(fin & (cb.bound == 0), np.where(err > 0, np.inf, 0.0), ratio)
    bad = ratio > 1.0
    if bad.any():
        rows, cols = np.nonzero(bad)
        k = int(np.argmax(ratio[bad]))
        r, c = rows[k], cols[k]
        raise AssertionError("%s: %d entries outside the chromagram bound in rows %s; worst (%s row %d, class %d): %r vs %r, "
                             "bound %.3g (err / bound %.3g)" % (what, rows.size, np.unique(rows)[:12].tolist(),
                                                              ROW_CLASS_NAMES[int(cb.cls[r])], r, c, got[r, c], cb.ref[r, c],
                                                              cb.bound[r, c], ratio[r, c]))
    worst = {}
    for c, name in ROW_CLASS_NAMES.items():
        sel = cb.cls == c
        if sel.any():
            worst[name] = float(ratio[sel].max())
    return worst, dict(cb.unbounded)


# ---------------------------------------------------------------------------------------------------------------------
# Every clip of a batch under its spectrum bound, through each kernel kind
ODD = 3                 # sample offset of the unaligned view


@contextlib.contextmanager
def pair_dump(B, T, K):
    """A NaN-filled float32 [B, T, K] buffer the pair kernel writes its |X| rows into while the block runs.  The dump
    pointer is process-wide: it is cleared once the launches that may write through it are done, before the buffer is
    freed, however the block ends."""
    import torch
    from pyaudioanalysis_b200._lib import lib
    buf = torch.full((B, T, K), float("nan"), dtype=torch.float32, device="cuda")
    assert lib().b200aa_debug_set_dump(ctypes.c_void_p(buf.data_ptr())) == 0
    try:
        yield buf
    finally:
        torch.cuda.synchronize()
        lib().b200aa_debug_set_dump(None)


def pair_spectra(P, fs, w, s):
    """The bank plus odd_tail (int16 and float32) as ragged feature batches through the pair kernel, every frame's dumped
    |X| row under the spectrum bound, exactly the frames below each clip's frame count written.  Returns the
    (bins, DC) err / bound of every clip."""
    from oracle import st_oracle as O
    from pyaudioanalysis_b200._lib import Plan
    from tests import signals as SG
    pl = Plan(fs, w, s).prefer_kernel(PAIR)
    assert pl.kernel_kind() == PAIR
    K = w // 2
    ints = dict(SG.bank(fs, w, s), odd_tail=SG.odd_tail(fs, w, s))
    flts = dict(SG.float_bank(fs, w, s), odd_tail_f32=ints["odd_tail"].astype(np.float32) * np.float32(0.37) + np.float32(11.5))
    ratios = []
    for bank, dtype in ((ints, np.int16), (flts, np.float32)):
        names, clips = list(bank), list(bank.values())
        d, lens = ragged(clips, dtype)
        with pair_dump(len(clips), O.frame_count(d.shape[1], w, s), K) as buf:
            P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl)
        got = buf.cpu().numpy()
        for i, name in enumerate(names):
            Tb = O.frame_count(clips[i].size, w, s)
            what = "pair kernel |X| rows, fs=%d w=%d s=%d: %s (%d frames)" % (fs, w, s, name, Tb)
            assert not np.isnan(got[i, :Tb]).any(), what + ": a frame below T_b was not written"
            assert np.isnan(got[i, Tb:]).all(), what + ": a frame at or past T_b was written"
            ratios.append(check_spectrum(got[i, :Tb], clips[i], s * np.arange(Tb), w, what))
    return ratios


def row_spectra(P, pl, fs, w, s, kind_name, offset_view=False):
    """The bank (int16 and float32) as ragged batches through spectrogram_batch on plan pl, every clip's rows under the
    spectrum bound; with offset_view also the int16 batch as a view at an odd sample offset.  Returns
    {"int16" | "float32" | "odd offset": [(bins, DC) err / bound of every clip]}."""
    from tests import signals as SG
    ints, flts = SG.bank(fs, w, s), SG.float_bank(fs, w, s)
    ratios = {}
    for bank, dtype, offsets in ((ints, np.int16, (0, ODD) if offset_view else (0,)), (flts, np.float32, (0,))):
        names, clips = list(bank), list(bank.values())
        for off in offsets:
            d, lens = ragged(clips, dtype, offset=off)
            sp = P.spectrogram_batch(d, fs, w, s, plan=pl, lengths=lens).cpu().numpy()
            for i, name in enumerate(names):
                R = int((clips[i].size - w) / s) + 1
                what = "%s rows, fs=%d w=%d s=%d%s: %s" % (kind_name, fs, w, s, ", odd offset" if off else "", name)
                cls = "odd offset" if off else ("float32" if dtype == np.float32 else "int16")
                ratios.setdefault(cls, []).append(check_spectrogram_rows(sp[i, :R], clips[i], w, s, what))
    return ratios


def generic_spectra(P, fs, w, path):
    """sweep_clips through a force_generic plan (the int16 clips as a ragged batch, the float32 clip alone), every row
    under the spectrum bound.  Returns the (bins, DC) err / bound of every clip."""
    import torch
    from pyaudioanalysis_b200._lib import Plan
    from tests.signals import sweep_clips
    s, ints, flt = sweep_clips(w)
    pl = Plan(fs, w, s)
    pl.force_generic(True)
    d, lens = ragged(ints, np.int16)              # ragged row kernel
    sp = P.spectrogram_batch(d, fs, w, s, plan=pl, lengths=lens).cpu().numpy()
    ratios = [check_spectrogram_rows(sp[i], x, w, s, "generic rows, w=%d s=%d (%s): int16 clip %d" % (w, s, path, i))
              for i, x in enumerate(ints)]
    spf = P.spectrogram_batch(torch.from_numpy(flt).cuda()[None], fs, w, s, plan=pl).cpu().numpy()   # equal-length row kernel
    ratios.append(check_spectrogram_rows(spf[0], flt, w, s, "generic rows, w=%d s=%d (%s): float32 chirp" % (w, s, path)))
    return ratios


# ---------------------------------------------------------------------------------------------------------------------
# Clips that end in clipped chromagram frames
def prime_between(lo, hi):
    for n in range((lo + hi) // 2, hi):
        if n > 1 and all(n % d for d in range(2, int(n ** 0.5) + 1)):
            return n
    return None


def clipped_targets(w, s):
    """Lengths the last clipped frame of an accepted clip can have, picked at K, K + 1, a prime and w - 1 where each is
    reachable.  The loop's last start p < len - s leaves n = len - p in (s, 2 s], and the reference needs n >= K; the
    clipped frames before it have n + s, n + 2 s, ... < w samples."""
    lo, hi = max(w // 2, s + 1), min(2 * s, w - 1)
    out = [n for n in (w // 2, w // 2 + 1, prime_between(lo, hi + 1), w - 1, hi) if n is not None and lo <= n <= hi]
    return sorted(set(out))


def clipped_clips(fs, w, s, n_last):
    """{name: clip} whose last chromagram row transforms a clipped frame of n_last samples, after a few full rows and the
    other clipped rows of its chain.  Signals: noise; DC 20000 +- 3 LSB (the record's bp and the DC rebuild); quiet noise
    with a loud first sample in every clipped frame (x - x0); a tone with a whole number of cycles in the last clipped
    frame, off the w-point bins (its other classes are ~1e-10 of the total, where only an fp64 transform keeps them); +-1
    LSB dither; a last clipped frame that is a run at the clip's exact integer mean (exact zeros); float32 noise at offset
    11.5 and a float32 tone with noise at 1e-3 full scale."""
    L = w + (-(-w // s) + 2) * s + n_last
    _, n_it, n_full, refused = chromagram_rows(L, w, s)
    assert not refused and n_full >= 2 and L - (w + (n_it - 1) * s) == n_last, (w, s, n_last)
    rng = np.random.default_rng(w * 31 + s * 7 + n_last)
    p_last = L - n_last
    firsts = [w + i * s for i in range(n_full, n_it)]
    t = np.arange(L)
    cyc = max(3, round(n_last * 523.25 / fs))          # C5-ish, whole cycles over n_last samples
    out = {"noise": np.round(rng.normal(0, 3000.0, L)).astype(np.int16),
           "dc": (20000 + rng.integers(-3, 4, L)).astype(np.int16)}
    x = np.round(rng.normal(0, 30.0, L))
    x[firsts] = 30000.0
    out["loud_first"] = x.astype(np.int16)
    out["tone"] = np.round(20000.0 * np.sin(2 * np.pi * cyc * t / n_last + 0.3)).astype(np.int16)
    out["dither"] = rng.integers(-1, 2, L).astype(np.int16)
    x = rng.integers(-3000, 3001, L).astype(np.int64) + 7
    x[p_last:] = 7
    q, r = divmod(int(x.sum()) - 7 * L, w)
    x[:w] -= q                                          # samples in no row: the clip mean becomes exactly 7
    x[0] -= r
    assert x.sum() == 7 * L
    out["mean_run"] = x.astype(np.int16)
    F = np.float32
    out["noise_f32"] = (out["noise"].astype(F) * F(0.37) + F(11.5)).astype(F)
    out["small_f32"] = (rng.normal(0, 1e-3 / 3, L) + 1e-3 * np.sin(2 * np.pi * cyc * t / n_last)).astype(F)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Batches under the per-entry bounds: worst err / bound and unbounded counts per (kernel, input), printed as JSON
def note(acc, worst, unb):
    for k, v in worst.items():
        acc["worst"][k] = max(acc["worst"].get(k, 0.0), v)
    for k, v in unb.items():
        acc["unbounded"][k] = acc["unbounded"].get(k, 0) + v


def report(tag, accs):
    for key, acc in accs.items():
        print(json.dumps(dict(config=tag, kernel=key[0], input=key[1],
                              worst={k: round(v, 4) for k, v in acc["worst"].items()}, unbounded=acc["unbounded"])))


def check_rows(out, cbs, what, accs, key):
    """out [B, R, 12] of a ragged batch (or an equal-length one): clip i's rows under its bound, the rows past them
    zero; a refused clip has none."""
    for i, cb in enumerate(cbs):
        R = cb.ref.shape[0]
        assert not out[i, R:].any(), what[i] + ": rows past the clip's own"
        if cb.refused:
            continue
        note(accs.setdefault(key, {"worst": {}, "unbounded": {}}), *check_chromagram_bounds(out[i, :R], cb, what[i]))


def ragged_bounds(P, pl, clips, names, dtype, fs, w, s, tag, accs, key, cbs=None):
    """clips as one ragged chromagram batch through plan pl, every clip under its bound.  Returns the bounds."""
    d, lens = ragged(clips, dtype)
    cbs = cbs or [chromagram_bounds(x, fs, w, s) for x in clips]
    out = P.chromagram_batch(d, fs, w, s, plan=pl, lengths=lens).cpu().numpy()
    assert P.row_counts(lens, w, s, 1).cpu().tolist() == [0 if cb.refused else cb.ref.shape[0] for cb in cbs], tag
    check_rows(out, cbs, ["%s: %s" % (tag, n) for n in names], accs, key)
    return cbs


def batch_bounds(P, pl, clips, dtype, fs, w, s, what, acc):
    """clips as one ragged batch through plan pl, deltas on and off, every clip under its bound; rows past a clip's
    frame count stay zero."""
    d, lens = ragged(clips, dtype)
    fbs = [feature_bounds(x, fs, w, s, deltas=True) for x in clips]
    for deltas in (True, False):
        out = P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl, deltas=deltas).cpu().numpy()
        for i, fb in enumerate(fbs):
            T = fb.ref.shape[1]
            F = 68 if deltas else 34
            assert not out[i, :, T:].any(), what[i] + ": output past the clip's frames"
            if not deltas:
                fb = type(fb)(fb.ref[:34], fb.bound[:34], fb.roll, {k: v for k, v in fb.unbounded.items()
                                                                    if not k.startswith("delta")}, fb.K)
            note(acc, *check_feature_bounds(out[i, :F, :T], fb, what[i] + (", deltas" if deltas else ", no deltas")))


# ---------------------------------------------------------------------------------------------------------------------
# Kernel 0's clip record against exact arithmetic
A_EMPTY = np.float32(1.0 / (32768.0 * 1e-10))      # a of a clip without samples (max deviation 0)


def check_f32_clip(rec, x, what):
    a, bp, m, lo, hi = (float(v) for v in rec[:5])
    assert not rec[5:].any(), what + ": reserved words not cleared"
    L = x.size
    if L == 0:
        assert rec[0] == A_EMPTY and not rec[1:5].any(), what + ": record of an empty clip"
        return
    xd = x.astype(np.float64)
    total = math.fsum(xd.tolist())
    mean = total / L
    assert abs(m - mean) <= float(np.spacing(np.float32(abs(mean)))), "%s: m = %r, mean %r" % (what, m, mean)
    if m == mean:
        assert lo == hi == 0.0, "%s: mean %r is a float32 but lo / hi = %r / %r" % (what, mean, lo, hi)
    else:
        lo_abs, hi_abs = np.float32(m + lo), np.float32(m + hi)
        assert float(lo_abs) < mean < float(hi_abs) and np.nextafter(lo_abs, np.float32(np.inf)) == hi_abs, \
            "%s: [%r, %r] does not bracket the mean %r between neighbouring floats" % (what, m + lo, m + hi, mean)
    ra = 1.0 / (max(xd.max() - mean, mean - xd.min()) + 32768.0 * 1e-10)
    assert abs(a - ra) <= float(np.spacing(np.float32(ra))), "%s: a = %r, expected %r" % (what, a, ra)
    rbp = ra * (m - mean)
    assert abs(bp - rbp) <= 2.0 ** -24 * abs(rbp) + 2.0 ** -149 + ra * 2.0 ** -50 * float(np.abs(xd).sum()), \
        "%s: bp = %r, expected %r" % (what, bp, rbp)
    check_samples(rec, x, np.sign(xd - mean), what)


def check_samples(rec, x, sign, what):
    """lo / hi classify d = x - m (float32, as the kernels form it) exactly as sign(x - mean); fma(a, d, bp) is the
    reference's normalised sample to float32 resolution of the clip's full scale."""
    from oracle import st_oracle as O
    a, bp, m, lo, hi = (np.float32(v) for v in rec[:5])
    d = x.astype(np.float32) - m
    cls = (d > lo).astype(np.int64) - (d < hi).astype(np.int64)
    bad = cls != sign
    assert not bad.any(), "%s: sign(x - mean) wrong for %d samples, first at %d" % (what, int(bad.sum()), int(np.argmax(bad)))
    y = (np.float64(a) * d.astype(np.float64) + np.float64(bp)).astype(np.float32).astype(np.float64)
    ref = O.normalize_clip(x.astype(np.float64))
    tol = 8 * 2.0 ** -24 * np.abs(ref).max() + 1e-30
    err = np.abs(y - ref)
    assert err.max() <= tol, "%s: a (x - m) + bp off by %.3g (tolerance %.3g) at sample %d" % (what, err.max(), tol, int(np.argmax(err)))

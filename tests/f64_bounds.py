"""Error bounds of the float64 feature path (kernel 12): its magnitude spectrum, full-frame and clipped, and its chroma
classes, each against a float64 reference under a bound derived from kernel 12's own fp64 arithmetic.

u = 2^-53 throughout; gamma64(n) = n u / (1 - n u) (tests/parity.gamma64).

**Full frames** (``spectrum_bound``).  Kernel 12 transforms the normalised frame y itself (no y - y[0] shift), length N,
by Stockham passes of radices R_1 .. R_m (``radices``: 4s first, then primes ascending, csrc/tables.inl radix_list; a
prime window is one pass of R = N).  Every output of a pass is one R-term sum sum_r v_r t_r over R inputs v and R table
twiddles t (``f64::stockham_output``), each component an fma chain of 2 R steps: |err| <= gamma64(2 R) sum_r (|v_r.x t_r.x|
+ |v_r.y t_r.y|) <= gamma64(2 R) (1 + tw) sum_r |v_r| per component, sqrt(2) times that as a complex number.  The table is
cos / sin(a), a = fl(fl(-2 kPi j) / N): kPi, the product and the quotient round once each, so a is off by gamma64(3) |a|
< 2 pi gamma64(3), and cos / sin (at most 1 ulp, < 2 u on [-1, 1]) add 2 sqrt(2) u as a complex number:
tw = 2 pi gamma64(3) + 2 sqrt(2) u, the largest at j near N, which the passes reach.  A twiddle off by tw moves an output
by tw sum_r |v_r|.  So every output errs by eps_R sum_r |v_r| <= eps_R sqrt(R) |v_g|_2 with
    eps_R = tw + sqrt(2) gamma64(2 R) (1 + tw),
where v_g is the group of R inputs the output reads.  The R outputs of a group read the same R inputs, so the pass errs by
R eps_R |v|_2 in 2-norm; the exact pass is a DFT of length R times unit twiddles per group, which scales the 2-norm by
sqrt(R).  Carried through the later (scaled unitary) passes, the whole transform errs by
    |X' - X|_2 <= delta sqrt(N) |y|_2,      delta = prod_p (1 + sqrt(R_p) eps_R_p) - 1,
(each pass's error relative to the exact norm of its output, compounded), where sqrt(N) |y|_2 = |X|_2 (Parseval).  Then
|X[k]| / K: hypot (CUDA: 2 ulp, CUDA C++ Programming Guide, double-precision functions; the host's libm less) and the IEEE
division by K, gamma64(5) of each bin, at most gamma64(5) (1 + delta) sqrt(N) |y|_2 / K in 2-norm.

The reference is NumPy's FFT of the same y (kernel 12's y equals the oracle's bit for bit, tests/test_gpu_f64.py
test_rows_0_1_bit_for_bit), held in parity's form: REF_FFT_C u ceil(log2 N) sqrt(N) |y|_2 / K, plus 4 u of each bin
for np.abs and the division.  The bound on the 2-norm of the error over the K bins is the sum, times MARGIN (first-order
products of (1 + err) factors).  There is no fitted constant: every term above is a stated rounding count.

What it costs per pass, sqrt(R) eps_R ~ sqrt(R) (2.83 R + 21.7) u: 66 u for a radix 4, 52 u for 3, 80 u for 5, 110 u for
7; a whole 800-point transform (4, 4, 2, 5, 5) ~330 u, 44 100 points ~550 u, each a few 1e-14 of |X|_2.  A prime window's single direct
pass costs sqrt(N) (2.83 N + 21.7) u: the worst case of an N-term chain, far above its typical (random-walk) error, so
primes are held much more loosely than composite windows.  Twiddles built by recurrence drift by about j u, N u at the
end of the table (44 100 u at 1 s at 44.1 kHz); one bin of a tone off by 1e-12 of its size is outside the bound of a
composite window; both pass ``assert_allclose(rtol=1e-9, atol=1e-11)`` (tests/test_f64_bounds_cpu.py).

**Clipped frames** (``clipped_reference``): a chromagram frame of n samples, K <= n < w, is transformed directly: re / im of
bin k are sequential fmas over the n samples y_j with twiddles sincospi(2 j / n) (``TWIDDLE_ABS`` per component, parity),
so per component gamma64(n) (1 + TWIDDLE_ABS) |y|_1 + TWIDDLE_ABS |y|_1, sqrt(2) times that complex; then hypot and / K
(gamma64(5)).  The reference is NumPy's FFT of the n samples, bounded per bin by the whole ball above (a bin's error is at
most the 2-norm's).

**Chroma classes** (``chroma_bound64``): c_j = (C X^2)_j / E, E = sum X^2, as parity.chroma_bound derives it: with X'
within the ball (full frames) or per-bin eps (clipped frames), c_j' - c_j = sum_k (C_jk - c_j)(X'_k^2 - X_k^2) / E'.  Over
|d|_2 <= e: |sum_k a_k ((X_k + d_k)^2 - X_k^2)| <= 2 |a X|_2 e + max |a| e^2.  Plus the fp64 chroma stage of kernel 12
(``f64_chroma``: each class adds X^2 / share of its taps in sequence, gamma64(taps + 2); E is NumPy's pairwise sum,
gamma64(pairwise_depth(K)); one IEEE division, u) and the same stage of the reference (X^2, the matrix product over the
same taps with 1 / share rounded, np.sum, the division): twice the stage.

**Feature rows** (``feature_bounds64``).  X' (kernel) lies in the ball |X' - X|_2 <= e of ``spectrum_bound``; the bound of
each entry is the largest change of the reference's exact formula over the ball, plus kernel 12's float64 stage and the
reference's (both sides' roundings counted, so no "2 x" hides in a constant).  pK = pairwise_depth(K).
* Rows 0-1: bit for bit (bound 0).  Row 2: the samples are exact, so only the stage: s_j = B_j / (E + eps) off by
  gamma64(pairwise_depth(w / 10)) + gamma64(pairwise_depth(w)) + 2 u per side, then ``_entropy64``: the mean value
  theorem on h(s) = -s log2(s + eps), the logs (1 ulp CUDA, 4 ulp NumPy's SIMD loops), the products and 10-term sums.
* Row 3: with ind = fl((k + 1) fs / 2K) (the same double on both sides), cen = N / Dn, N = sum ind X, Dn = S + eps top,
  top = max X.  top moves by at most e, S by sqrt(K) e, so |cen' - cen| <= (|ind - cen|_2 e + cen eps e) / (Dn - sqrt(K) e
  - eps e), plus gamma64(2 pK + 6) cen per side.  Row 4: V = sum (ind - c)^2 X / Dn at the computed centroid c (within
  dc of row 3's): V moves by (|w|_2 e + V eps e) / Dn_lo, w_k = |(ind_k - c)^2 - V| + 2 |ind_k - c| dc + dc^2 + dVc,
  dVc = dc (dc S + 2 cen eps top) / Dn the change of V with c; the stage adds u |ind - c| per rounded difference and
  gamma64(2 pK + 8) V; then sqrt over [V - dV, V + dV] and the roundings of sqrt and / (fs / 2).
* Row 5: X'^2 - X^2 = 2 X d + d^2, so s_j moves by (2 |(1_Bj - s_j) X|_2 e + max |1_Bj - s_j| e^2) / (E + eps - 2 |X|_2 e
  - e^2), then ``_entropy64``.  Row 6: sqrt(flux) = |X / Sn - Xp / Snp|_2, Sn = S + K eps; each side moves by (e + |X /
  Sn|_2 sqrt(K) e) / (Sn - sqrt(K) e) =: D, so flux moves by (Dt + Dp)(2 sqrt(flux) + Dt + Dp); the stage's rounded
  difference errs by gamma64(pK + 2)(|a_k| + |b_k|) + u |a_k - b_k| per bin, carried through the squares and the sum.
* Row 7: g_k = cumsum_k(X^2) + eps - 0.9 E has weights 1[j <= k] - 0.9 on X^2: it moves by 2 (0.01 C_k + 0.81 (E -
  C_k))^(1/2) e + 0.9 e^2, plus per side gamma64(k + 3) C_k (the sequential cumsum), (gamma64(pK) + u) 0.9 E and u (C_k +
  eps).  The kernel's index lies between the first k with g + b > 0 and the first with g - b > 0; the value is k / K
  correctly rounded (``check_feature_bounds64``: within 4 u of a whole number of quanta).
* Rows 8-20: m = M X moves by |M_j|_2 e plus gamma64(taps_j + 1) m_j (the kernel's sequential taps) and gamma64(K + 1)
  m_j (the reference's BLAS product, order unknown).  Both sides' m are sums of non-negative terms, so log10(m + eps)
  stays in [log10(max(m - dm, 0) + eps), log10(m + dm + eps)]: finite for every frame, constant frames included (written
  with log1p, which does not cancel).  Plus the + eps roundings (u / ln 10 per side), the logs (5 ulp together) and both
  sides' 40-term DCT sums, gamma64(41) sum |D| |log10 m| each.
* Rows 21-32: ``chroma_bound64``.  Row 33: np.std is 1-Lipschitz in the RMS norm of the class errors, plus per side the
  stage of a 12-value mean, the differences, squares, sum, division and sqrt.
* Deltas: b[t] + b[t - 1] plus the rounding of both sides' differences; row 41 through the quanta of row 7.
"Unbounded" has one meaning: a denominator's interval reaches 0 (Dn - sqrt(K) e - eps e, Sn - sqrt(K) e, E + eps - dE
<= 0); each such entry is counted with its reason.  An exactly zero spectrum (e = 0, top = 0) is bounded by the stage
alone.
"""
import math

import numpy as np

from tests.kernels import GENERIC_SWEEP
from tests.parity import MARGIN, O_EPS, REF_FFT_C, TWIDDLE_ABS, U64, _quad_bins, _ratio_den, _tables, gamma64

TW_TABLE = 2 * math.pi * float(gamma64(3)) + 2 * math.sqrt(2.0) * U64      # cos / sin of a rounded angle below 2 pi
MAG = float(gamma64(5))         # hypot (2 ulp) and the division by K, per bin

# Windows of the float64 spectrum sweep: the generic kernel's GENERIC_SWEEP; lanes above K and the 20-entry buffer floor
# (2 .. 33); 882 and 2205; the primes 997 and 20 011; 5 785 and 5 786, the last window whose arrays fit the frame kernel's
# shared memory and the first that goes to global scratch (f64_warp_bytes = 40 w bytes against kSmemCap = 226 KiB); 1 s
# at 44.1 kHz.
SMEM_LAST, BIG_FIRST = 5785, 5786
SWEEP = sorted({c[1] for c in GENERIC_SWEEP}
               | {2, 3, 9, 19, 20, 21, 31, 32, 33, 882, 2205, 997, 20011, SMEM_LAST, BIG_FIRST, 44100})
KINDS = ("noise", "constant", "impulse", "alternating", "tone_on_bin", "tone_between_bins", "dc_offset")


def frame_kinds(N, seed=0):
    """{kind: N samples}: seeded noise, a constant, one impulse, alternating +-1, a tone on a bin and one between bins,
    a large DC offset with small noise.  Shapes only: callers scale them to their sample type."""
    rng = np.random.default_rng(seed * 7919 + N)
    t = np.arange(N)
    k0 = max(1, N // 7)
    imp = np.zeros(N)
    imp[N // 3] = 1.0
    return {"noise": rng.normal(0, 0.3, N), "constant": np.full(N, 0.37), "impulse": imp,
            "alternating": np.where(t % 2 == 0, 1.0, -1.0), "tone_on_bin": np.sin(2 * np.pi * k0 * t / N + 0.3),
            "tone_between_bins": np.sin(2 * np.pi * (k0 + 0.37) * t / N),
            "dc_offset": 0.9 + rng.normal(0, 1e-4, N)}


def kind_clip(w, dtype, seed=0):
    """A clip of 8 w samples whose spectrogram rows at hop w (frames at w, 2 w, .., 7 w) are the KINDS in order, after a
    noise segment; int16 at most full scale, float32 x 0.37 + 11.5, float64 with values float32 cannot hold."""
    fr = frame_kinds(w, seed)
    rng = np.random.default_rng(seed + 3 * w)
    x = np.concatenate([rng.normal(0, 0.3, w)] + [fr[k] for k in KINDS])
    i16 = np.clip(np.round(x * 30000.0), -32768, 32767).astype(np.int16)
    if dtype == np.int16:
        return i16
    if dtype == np.float32:
        return (i16.astype(np.float32) * np.float32(0.37) + np.float32(11.5)).astype(np.float32)
    return i16 * 1.000123e-3 + 0.25 + 1e-9 * rng.normal(size=i16.size)


def radices(n):
    """csrc/tables.inl radix_list: 4s first, then primes ascending (a window of 1: no pass)."""
    r = []
    while n % 4 == 0:
        r.append(4)
        n //= 4
    p = 2
    while p * p <= n:
        while n % p == 0:
            r.append(p)
            n //= p
        p += 1
    if n > 1:
        r.append(n)
    return r


def pass_cost(R):
    """sqrt(R) eps_R: one pass's error relative to the exact norm of its output."""
    return math.sqrt(R) * (TW_TABLE + math.sqrt(2.0) * float(gamma64(2 * R)) * (1 + TW_TABLE))


def transform_delta(N):
    """delta of the module docstring: the whole transform's 2-norm error over |X|_2."""
    d = 1.0
    for R in radices(N):
        d *= 1.0 + pass_cost(R)
    return d - 1.0


def ref_fft_rel(n):
    """NumPy's float64 FFT of length n: its 2-norm error over |X|_2, parity's REF_FFT_C form."""
    return REF_FFT_C * U64 * max(1, math.ceil(math.log2(max(n, 2))))


def spectrum_reference(frames):
    """frames [F, N] (normalised float64 samples): NumPy's |FFT|[0:K] / K [F, K] and the bound [F] on the 2-norm of
    kernel 12's error over those K bins."""
    frames = np.asarray(frames, dtype=np.float64)
    N = frames.shape[1]
    K = N // 2
    ref = np.abs(np.fft.fft(frames, axis=1)[:, :K]) / K
    return ref, spectrum_bound(frames)


def spectrum_bound(frames):
    frames = np.asarray(frames, dtype=np.float64)
    N = frames.shape[1]
    K = N // 2
    delta = transform_delta(N)
    scale = math.sqrt(N) * np.linalg.norm(frames, axis=1) / K            # |X|_2 on the output's scale
    return MARGIN * scale * (delta + MAG * (1 + delta) + ref_fft_rel(N) + 4 * U64)


def check_spectrum(got, frames, what=""):
    """Rows ``got`` [F, K] of kernel 12 for the normalised frames [F, N]: the 2-norm of every frame's error within its
    bound (a zero frame: exactly 0).  Returns the worst err / bound."""
    got = np.asarray(got, dtype=np.float64)
    ref, bound = spectrum_reference(frames)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.isfinite(got).all(), what + ": non-finite spectrum"
    err = np.linalg.norm(got - ref, axis=1)
    r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    bad = np.nonzero(r > 1.0)[0]
    if bad.size:
        j = bad[np.argmax(r[bad])]
        k = int(np.argmax(np.abs(got[j] - ref[j])))
        raise AssertionError("%s: %d of %d frames outside the float64 spectrum bound; worst frame %d: err / bound %.3g, "
                             "largest error in bin %d: %r vs %r" % (what, bad.size, len(r), j, r[j], k, got[j, k], ref[j, k]))
    return float(r.max()) if r.size else 0.0


def clipped_reference(fr, K):
    """A clipped frame fr (n normalised samples, K <= n): NumPy's |FFT|[0:K] / K and the per-bin bound [K] of kernel 12's
    direct DFT, the reference's own error included."""
    fr = np.asarray(fr, dtype=np.float64)
    n = fr.size
    X = np.abs(np.fft.fft(fr)[:K]) / K
    chain = math.sqrt(2.0) * (float(gamma64(n)) * (1 + TWIDDLE_ABS) + TWIDDLE_ABS) * np.abs(fr).sum() / K
    ref = (ref_fft_rel(n) * math.sqrt(n) * np.linalg.norm(fr)) / K + 4 * U64 * X
    eps = MARGIN * (chain + MAG * (X + chain) + ref)
    return X, eps


def pairwise_depth(n):
    """Roundings a term of NumPy's pairwise sum of n values passes through: below 8 terms a sequential sum; up to 128 eight
    sequential accumulators of n / 8 terms, their three-level tree and up to 7 leftover additions; above, one level per
    halving (kernel 12 splits the same tree across the lanes of a warp), the final 0 + s, and the term's own product."""
    n = max(int(n), 1)
    base = n if n < 8 else -(-min(n, 128) // 8) + 3 + 7
    return base + max(0, math.ceil(math.log2(n / 128.0))) + 2


def _classes(X, C):
    Et = (X ** 2).sum(axis=1)
    return (X ** 2) @ C.T / np.where(Et == 0, O_EPS, Et)[:, None]


def chroma_bound64(X, C, cj, e=None, eps=None):
    """Per-entry bound [T, 12] on kernel 12's chroma classes for frames whose float64 spectrum is X [T, K] and classes cj
    [T, 12]: either the spectrum ball (|d|_2 <= e [T]) or per-bin bounds eps [T, K]; nan where E's interval reaches 0."""
    K = X.shape[1]
    Et = (X ** 2).sum(axis=1)
    w = C[None] - cj[:, :, None]                                               # [T, 12, K]
    if eps is None:
        dEt = 2 * np.linalg.norm(X, axis=1) * e + e ** 2
        num = 2 * np.linalg.norm(w * X[:, None, :], axis=2) * e[:, None] + np.abs(w).max(axis=2) * (e ** 2)[:, None]
    else:
        dEt = _quad_bins(np.ones(K), X, eps)
        num = _quad_bins(w, X[:, None, :], eps[:, None, :])
    dc_t = num / _ratio_den(np.where(Et == 0, O_EPS, Et), dEt)[:, None]
    stage = gamma64((C > 0).sum(axis=1) + 2)[None, :] + gamma64(pairwise_depth(K)) + U64
    return MARGIN * (dc_t + 2 * stage * cj)


class Bounds:
    """``ref`` [R, 12] reference classes, ``bound`` [R, 12] (inf where unbounded), ``cls`` [R] row classes as in
    parity (ROW_FULL / ROW_CLIPPED / ROW_EMPTY), ``refused`` and ``unbounded`` {reason: entries}: the shape of
    parity.ChromaBounds, so parity.check_chromagram_bounds checks it."""

    def __init__(self, ref, bound, cls, refused, unbounded):
        self.ref, self.bound, self.cls, self.refused, self.unbounded = ref, bound, cls, refused, unbounded


def _finish(ref, bound, cls, refused):
    unb = {}
    nan = np.isnan(bound).any(axis=1)
    if nan.any():
        unb["sum X^2 interval contains 0"] = int(nan.sum()) * 12
    return Bounds(ref, np.where(np.isnan(bound), np.inf, bound), cls, refused, unb)


def chromagram_bounds(x, fs, w, s):
    """Kernel 12's chromagram rows of clip x at (fs, w, s): full rows (frame at w + r s) through the spectrum ball,
    clipped rows (n = len - (w + r s) samples, K <= n < w) through the per-bin clipped bound, rows the reference's loop
    never fills exactly 0."""
    from oracle import st_oracle as O
    from tests.parity import ROW_CLIPPED, ROW_EMPTY, ROW_FULL, chromagram_rows
    x = np.asarray(x)
    K = w // 2
    R, n_it, n_full, refused = chromagram_rows(x.size, w, s)
    if refused:
        return Bounds(np.zeros((0, 12)), np.zeros((0, 12)), np.zeros(0, dtype=int), True, {})
    C = _tables(fs, K)[2]
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    ref, bound, cls = np.zeros((R, 12)), np.zeros((R, 12)), np.full(R, ROW_EMPTY)
    if n_full:
        fr = np.stack([y[w + s * i:2 * w + s * i] for i in range(n_full)])
        X, e = spectrum_reference(fr)
        cj = _classes(X, C)
        ref[:n_full], bound[:n_full], cls[:n_full] = cj, chroma_bound64(X, C, cj, e=e), ROW_FULL
    if n_it > n_full:
        rows = np.arange(n_full, n_it)
        XE = [clipped_reference(y[w + s * i:], K) for i in rows]
        X = np.stack([v[0] for v in XE])
        cj = _classes(X, C)
        ref[rows], bound[rows], cls[rows] = cj, chroma_bound64(X, C, cj, eps=np.stack([v[1] for v in XE])), ROW_CLIPPED
    return _finish(ref, bound, cls, False)


def feature_chroma_bounds(x, fs, w, s):
    """Rows 21 .. 32 of kernel 12's feature matrix (the chroma classes of every frame t s) as a Bounds over [T, 12]."""
    from oracle import st_oracle as O
    from tests.parity import ROW_FULL
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    T = O.frame_count(y.size, w, s)
    C = _tables(fs, w // 2)[2]
    fr = np.stack([y[s * t:s * t + w] for t in range(T)])
    X, e = spectrum_reference(fr)
    cj = _classes(X, C)
    return _finish(cj, chroma_bound64(X, C, cj, e=e), np.full(T, ROW_FULL), False)


# ---------------------------------------------------------------------------------------------------------------------
# The 68 feature rows (derivation: "Feature rows" in the module docstring)
LOG_HOST_ULP = 4        # NumPy's float64 log2 / log10: its SIMD loops are documented to 4 ulp, libm's to 1
LOG_CUDA_ULP = 1        # CUDA's double-precision log2 / log10 (CUDA C++ Programming Guide, mathematical functions)
LOG_ULPS = LOG_HOST_ULP + LOG_CUDA_ULP
EPS = O_EPS


def rowsum(A):
    """np.sum of every row of A, each a contiguous 1-D reduction: NumPy's pairwise sum, kernel 12's order."""
    A = np.ascontiguousarray(A, dtype=np.float64)
    return np.array([np.sum(r) for r in A]) if A.shape[0] else np.zeros(0)


def _g(n):
    return float(gamma64(n))


def _entropy64(s, ds):
    """Bound on |H' - H|, H = sum_j h(s_j), h(s) = -s log2(s + eps), each s_j' within ds_j of s_j, both sides' stage
    included.  By the mean value theorem |h(s') - h(s)| <= ds max |h'| over [lo, hi] (lo = max(s - ds, 0), hi = s + ds),
    |h'(s)| = |log2(s + eps) + s / ((s + eps) ln 2)| <= max(|log2(lo + eps)|, |log2(hi + eps)|) + 1 / ln 2.  (parity's
    concave-h interval gives the same bound, but its endpoint differences h(s) - h(lo) cancel in float64 at these
    widths.)  Then the logs of both sides, LOG_ULPS ulp <= 2 LOG_ULPS u |log2|, times s; the products and the 10-term
    pairwise sums of both sides, 2 gamma64(pairwise_depth(10))."""
    lo = np.maximum(s - ds, 0.0)
    hi = s + ds
    lg = np.maximum(np.abs(np.log2(lo + EPS)), np.abs(np.log2(hi + EPS)))
    dev = ds * (lg + 1 / math.log(2.0)) + hi * 2 * LOG_ULPS * U64 * lg
    stage = 2 * _g(pairwise_depth(10)) * (np.abs(s * np.log2(s + EPS)) + dev)
    return MARGIN * (dev + stage).sum(axis=-1)


def _blocks(V, n_blocks=10):
    """[T, 10] block sums of squares of the rows of V: blocks of len // 10 values, NumPy's pairwise sum each."""
    blk = V.shape[1] // n_blocks
    return np.stack([rowsum(V[:, j * blk:(j + 1) * blk] ** 2) for j in range(n_blocks)], axis=1), blk


def feature_bounds64(x, fs, w, s, deltas=False):
    """The float64 reference of all 68 (34 without deltas) short-term feature rows of clip x at (fs, w, s), every frame,
    and a per-entry bound on what kernel 12 may return, as a parity.FeatureBounds (rolloff: admissible quanta)."""
    from oracle import st_oracle as O
    from tests.parity import FeatureBounds
    K = w // 2
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    T = O.frame_count(y.size, w, s)
    fr = np.stack([y[s * t:s * t + w] for t in range(T)])
    X, e = spectrum_reference(fr)
    ref = O.base_features_from_frames(fr, X, fs)
    ref[0] = [O._zcr(f) for f in fr]
    ref[1] = [O._energy(f) for f in fr]
    M, D, C = _tables(fs, K)
    u = U64
    bound = np.zeros_like(ref)
    unb = {}

    def unbounded(rows, mask, reason):
        if mask.any():
            bound[np.ix_(rows, np.nonzero(mask)[0])] = np.inf
            unb[reason] = unb.get(reason, 0) + int(mask.sum()) * len(rows)

    pK = pairwise_depth(K)
    # row 2: the samples are exact; both sides round the block sums, the total, + eps and the division
    Bt, blk = _blocks(fr)
    Et = rowsum(fr ** 2)
    sj = Bt / (Et + EPS)[:, None]
    bound[2] = _entropy64(sj, 2 * sj * (_g(pairwise_depth(blk)) + _g(pairwise_depth(w)) + 2 * u))

    # rows 3, 4: in Hz, ind = fl((k + 1) fs / (2 K)) the same value on both sides; cen = N / Dn with N = sum ind X and
    # Dn = S + eps top (X / top and sum + eps, top = max X); top moves by at most e
    ind = np.arange(1, K + 1) * (fs / (2.0 * K))
    half = fs / 2.0
    S = X.sum(axis=1)
    top = X.max(axis=1)
    Dn = S + EPS * top
    silent = (top == 0) & (e == 0)                       # an exactly zero spectrum: both sides compute 0 exactly
    Dlo = _ratio_den(Dn, math.sqrt(K) * e + EPS * e)
    Dlo = np.where(silent, 1.0, Dlo)
    c = ref[3] * half
    dc_t = (np.linalg.norm(ind[None, :] - c[:, None], axis=1) * e + c * EPS * e) / Dlo
    dc = MARGIN * (dc_t + 2 * _g(2 * pK + 6) * c)
    bound[3] = dc / half
    V = (ref[4] * half) ** 2
    Dsafe = np.where(silent, 1.0, Dn)
    dVc = dc * (dc * S + 2 * c * EPS * top) / Dsafe       # V at a centroid dc away
    dk = np.abs(ind[None, :] - c[:, None])
    wv = np.abs(dk ** 2 - V[:, None]) + 2 * dk * dc[:, None] + dc[:, None] ** 2 + dVc[:, None]
    dV_t = (np.linalg.norm(wv, axis=1) * e + (V + dVc) * EPS * e) / Dlo + dVc
    zeta = u * (dk + dc[:, None])                        # the rounded ind - cen
    dV_a = 2 * (((2 * dk * zeta + zeta ** 2) * X).sum(axis=1) / Dlo + _g(2 * pK + 8) * (V + dVc))
    dV = MARGIN * (dV_t + dV_a)
    sv = np.sqrt(V)
    up = np.where(dV > 0, dV / np.maximum(np.sqrt(V + dV) + sv, 1e-300), 0.0)
    down = np.where(V > dV, dV / np.maximum(sv + np.sqrt(np.maximum(V - dV, 0.0)), 1e-300), sv)
    bound[4] = (np.maximum(up, down) + 4 * u * np.sqrt(V + dV)) / half
    unbounded([3, 4], np.isnan(Dlo), "sum X interval contains 0 (centroid, spread)")

    # row 5: s_j = B_j / (E + eps) over blocks of K // 10 bins; X'^2 - X^2 = 2 X d + d^2
    P = X ** 2
    E = P.sum(axis=1)
    dE = 2 * np.linalg.norm(X, axis=1) * e + e ** 2
    Bs, blk = _blocks(X)
    sjs = Bs / (E + EPS)[:, None]
    Bm = np.zeros((10, K))
    for j in range(10):
        Bm[j, j * blk:(j + 1) * blk] = 1.0
    a = Bm[None] - sjs[:, :, None]                                             # [T, 10, K]
    Elo = _ratio_den(E + EPS, dE)
    ds = (2 * np.linalg.norm(a * X[:, None, :], axis=2) * e[:, None] + np.abs(a).max(axis=2) * (e ** 2)[:, None]) / Elo[:, None]
    bound[5] = _entropy64(sjs, ds + 2 * sjs * (_g(pairwise_depth(blk)) + _g(pK) + 2 * u))

    # row 6: sqrt(flux) = |X / Sn - Xp / Snp|_2, Sn = sum(X + eps); each side moves by (e + |X / Sn|_2 dSn) / (Sn - dSn)
    Sn = S + K * EPS
    dSn = math.sqrt(K) * e
    Snlo = _ratio_den(Sn, dSn)
    nrm = np.linalg.norm(X, axis=1) / Sn
    Dt = (e + nrm * dSn) / Snlo
    Dp = np.concatenate([Dt[:1], Dt[:-1]])
    Xn = X / Sn[:, None]
    Pn = np.concatenate([Xn[:1], Xn[:-1]])
    dd = np.abs(Xn - Pn)
    eta = _g(pK + 2) * (Xn + Pn) + u * dd                                      # one side's rounded difference
    sq = (2 * dd * eta + eta ** 2).sum(axis=1)
    rf = np.sqrt(ref[6])
    bound[6] = MARGIN * ((Dt + Dp) * (2 * rf + Dt + Dp) + 2 * (sq + _g(pK) * (ref[6] + sq)))
    unbounded([6], np.isnan(Snlo) | np.isnan(np.concatenate([Snlo[:1], Snlo[:-1]])), "sum (X + eps) interval contains 0")

    # row 7: first k with g_k = cumsum_k(X^2) + eps - 0.9 E > 0; weights 1[j <= k] - 0.9 on X^2; both sides' stage
    Pc = np.cumsum(P, axis=1)
    g = Pc + EPS - 0.9 * E[:, None]
    aX2 = 0.01 * Pc + 0.81 * np.maximum(E[:, None] - Pc, 0.0)
    kk = np.arange(K)[None, :]
    b = MARGIN * (2 * np.sqrt(aX2) * e[:, None] + 0.9 * (e ** 2)[:, None]
                  + 2 * (_g(1) * (kk + 3) * Pc + (_g(pK) + u) * 0.9 * E[:, None] + u * (Pc + EPS)))
    first = lambda cnd: np.where(cnd.any(axis=1), np.argmax(cnd, axis=1), -1)
    lo, hi = first(g + b > 0), first(g - b > 0)
    lo = np.where((lo < 0) | (hi < 0), 0, lo)
    hi = np.where(hi < 0, K - 1, hi)
    roll = np.stack([lo, hi])

    # rows 8 .. 20: mel bands m = M X (non-negative sums on both sides), log10(m + eps), the DCT
    m = X @ M.T
    taps = np.array([np.ptp(np.nonzero(r)[0]) + 1 if r.any() else 0 for r in M])
    dm = np.linalg.norm(M, axis=1)[None, :] * e[:, None] + (gamma64(taps + 1)[None, :] + _g(K + 1)) * m
    lm = np.log10(m + EPS)
    lo_m = np.maximum(m - dm, 0.0)
    dL = np.maximum(np.log1p((m - lo_m) / (lo_m + EPS)), np.log1p(dm / (m + EPS))) / math.log(10.0)
    dL = dL + 2 * u / math.log(10.0) + 2 * LOG_ULPS * u * np.abs(lm)
    aD = np.abs(D)
    bound[8:21] = MARGIN * (dL @ aD.T + 2 * _g(41) * (np.abs(lm) @ aD.T)).T

    # rows 21 .. 33: the chroma bound; chroma_std 1-Lipschitz in the RMS norm of the class errors, plus np.std's stage
    cj = ref[21:33].T
    dcj = chroma_bound64(X, C, cj, e=e)
    bound[21:33] = dcj.T
    mu_e = _g(pairwise_depth(12) + 1) * np.abs(cj).mean(axis=1)
    bound[33] = np.sqrt((dcj ** 2).mean(axis=1)) + 2 * MARGIN * (mu_e + (_g(pairwise_depth(12) + 4) + u) * (ref[33] + mu_e))
    unbounded([5] + list(range(21, 34)), np.isnan(Elo) | np.isnan(dcj).any(axis=1), "sum X^2 interval contains 0")
    bound = np.where(np.isnan(bound), np.inf, bound)
    bound[7] = 0.0
    if deltas:
        d = np.zeros_like(ref)
        d[:, 1:] = ref[:, 1:] - ref[:, :-1]
        db = np.zeros_like(bound)
        db[:, 1:] = bound[:, 1:] + bound[:, :-1]
        db[:, 1:] += 2 * u * (np.abs(d[:, 1:]) + db[:, 1:])
        for reason in list(unb):
            unb["delta: " + reason] = unb[reason]
        ref, bound = np.concatenate([ref, d]), np.concatenate([bound, db])
    return FeatureBounds(ref, bound, roll, unb, K)


def check_feature_bounds64(got, fb, what=""):
    """parity.check_feature_bounds at float64: the rolloff k / K within 4 u64 of a whole number of quanta."""
    from tests.parity import check_feature_bounds
    return check_feature_bounds(got, fb, what, roll_slack=4 * U64)


# ---------------------------------------------------------------------------------------------------------------------
# The stage model: kernel 12's feature stage (csrc/f64.cu f64_spectrum's time rows, f64_spectral) restated in NumPy in
# its documented order, logs correctly rounded
def _cr(fn, v):
    """fn (mpmath.log, base 2 or 10) of every value of v, correctly rounded to float64."""
    import mpmath
    v = np.asarray(v, dtype=np.float64)
    uq, inv = np.unique(v, return_inverse=True)
    with mpmath.workprec(160):
        out = np.array([float(fn(mpmath.mpf(float(a)))) if a > 0 else (-np.inf if a == 0 else np.nan) for a in uq])
    return out[inv].reshape(v.shape)


def cr_log2(v):
    import mpmath
    return _cr(lambda a: mpmath.log(a, 2), v)


def cr_log10(v):
    import mpmath
    return _cr(mpmath.log10, v)


def _entropy_stage(Bsum, tot):
    """-np.sum of s_j log2(s_j + eps), s_j = B_j / (tot + eps), with correctly rounded logs; and the margin of a kernel
    whose log2 is within LOG_CUDA_ULP ulp: its logs differ by at most 1.5 ulp <= 3 u |L|, so each term by 3 u |t| plus
    both products' roundings, and each 10-term sum lies within gamma64(pairwise_depth(10)) sum |t| of the exact sum."""
    s = Bsum / (tot + EPS)[:, None]
    t = s * cr_log2(s + EPS)
    H = -rowsum(t)
    at = np.abs(t).sum(axis=1)
    return H, MARGIN * (5 * U64 + 2 * _g(pairwise_depth(10))) * at


def stage_tables(exe, fs, K):
    """(mel [40, K], dct [13, 40]) as the host builds them for the plan (tests/f64_host.cu ``tables``)."""
    from tests.host_exe import floats, run
    v = floats(run(exe, "tables %d %d\n" % (fs, K))[0][1:])
    return v[:40 * K].reshape(40, K), v[40 * K:].reshape(13, 40)


class Stage:
    """stage_model's result: ``rows`` [34, T] (rows 0 .. 1 nan: the model starts from the spectra), ``margin`` [34, T]
    (0: bit for bit; rows 2, 5, 8 .. 20: the log margin) and the mask ``have`` [34] of the rows it states."""

    def __init__(self, rows, margin, have):
        self.rows, self.margin, self.have = rows, margin, have


def stage_model(X, Xp, fs, mel, dct, frames=None):
    """Kernel 12's rows 3 .. 33 (and row 2 from the frames' samples, when given) of frames whose spectra are X [T, K]
    and whose previous frames' spectra are Xp [T, K], in the order DESIGN section 4 (kernel 12) states: NumPy's pairwise
    sums (np.sum of a contiguous row), IEEE division and sqrt, a sequential cumsum, sequential mel taps and a sequential
    40-term DCT, the chroma fold in ascending slot order, np.std of the 12 classes."""
    from oracle import st_oracle as O
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xp = np.ascontiguousarray(Xp, dtype=np.float64)
    T, K = X.shape
    rows = np.full((34, T), np.nan)
    margin = np.zeros((34, T))
    have = np.zeros(34, dtype=bool)
    if frames is not None:
        Bt, _ = _blocks(np.asarray(frames, dtype=np.float64))
        rows[2], margin[2] = _entropy_stage(Bt, rowsum(np.asarray(frames, dtype=np.float64) ** 2))
        have[2] = True
    top = X.max(axis=1)
    dv = np.where(top == 0.0, EPS, top)
    Xt = X / dv[:, None]
    ind = np.arange(1, K + 1).astype(np.float64) * (fs / (2.0 * K))
    den = rowsum(Xt) + EPS
    cen = rowsum(ind[None, :] * Xt) / den
    spr = np.sqrt(rowsum(((ind[None, :] - cen[:, None]) ** 2) * Xt) / den)
    rows[3], rows[4] = cen / (fs / 2.0), spr / (fs / 2.0)
    tot = rowsum(X * X)
    Bs, _ = _blocks(X)
    rows[5], margin[5] = _entropy_stage(Bs, tot)
    d = X / rowsum(X + EPS)[:, None] - Xp / rowsum(Xp + EPS)[:, None]
    rows[6] = rowsum(d * d)
    over = np.cumsum(X * X, axis=1) + EPS > (0.90 * tot)[:, None]
    rows[7] = np.where(over.any(axis=1), np.argmax(over, axis=1) / float(K), 0.0)
    acc = np.zeros((T, 40))
    for i in range(40):
        nz = np.nonzero(mel[i])[0]
        if nz.size:
            for k in range(nz[0], nz[-1] + 1):
                acc[:, i] = acc[:, i] + mel[i, k] * X[:, k]
    lm = cr_log10(acc + EPS)
    mf = np.zeros((T, 13))
    for n in range(40):
        mf = mf + dct[None, :, n] * lm[:, n:n + 1]
    rows[8:21] = mf.T
    margin[8:21] = (MARGIN * (5 * U64 + 2 * _g(41)) * (np.abs(lm) @ np.abs(dct).T)).T
    semis, share = O.chroma_tables(fs, K)
    wrap = lambda j: j + K if j < 0 else j
    winner = {}
    for k in range(K):
        winner[wrap(int(semis[k]))] = k
    ch = np.zeros((T, 12))
    for cl in range(12):
        for j in range(cl, K, 12):
            if j in winner:
                b = winner[j]
                ch[:, cl] = ch[:, cl] + (X[:, b] * X[:, b]) / share[wrap(int(semis[j]))]
    ch = ch / np.where(tot == 0.0, EPS, tot)[:, None]
    rows[21:33] = ch.T
    rows[33] = [np.std(r) for r in ch]
    have[3:34] = True
    return Stage(rows, margin, have)


EXACT_ROWS = (3, 4, 6, 7) + tuple(range(21, 34))
LOG_ROWS = (2, 5) + tuple(range(8, 21))


def check_stage(got, st, what="", rows=None):
    """Kernel rows ``got`` [34, T] against a Stage: rows 3, 4, 6, 7, 21 .. 33 equal (+0 == -0), rows 2, 5, 8 .. 20 within
    the log margin.  ``rows``: the subset to check (default: every row the model states).  Returns the worst
    |got - model| / margin of the log rows."""
    got = np.asarray(got, dtype=np.float64)
    rows = [r for r in (rows if rows is not None else range(34)) if st.have[r]]
    assert np.isfinite(got[rows]).all(), what + ": non-finite rows"
    worst = 0.0
    for r in rows:
        if r in EXACT_ROWS:
            bad = got[r] != st.rows[r]
            if bad.any():
                t = int(np.nonzero(bad)[0][0])
                raise AssertionError("%s: row %d differs from the stage model in %d frames, first %d: %r vs %r"
                                     % (what, r, int(bad.sum()), t, got[r, t], st.rows[r, t]))
        else:
            err = np.abs(got[r] - st.rows[r])
            bad = err > st.margin[r]
            if bad.any():
                t = int(np.nonzero(bad)[0][0])
                raise AssertionError("%s: row %d outside the stage model's log margin in %d frames, first %d: %r vs %r, "
                                     "margin %.3g" % (what, r, int(bad.sum()), t, got[r, t], st.rows[r, t], st.margin[r, t]))
            if err.size:
                worst = max(worst, float(np.max(np.where(err > 0, err / np.where(st.margin[r] > 0, st.margin[r], 1), 0))))
    return worst


def check_deltas(F, T, what=""):
    """Rows 34 .. 67 of a [68, >= T] feature block: column 0 zero, column t the kernel's own row difference, in bits."""
    F = np.asarray(F, dtype=np.float64)[:, :T]
    d = np.zeros((34, T))
    d[:, 1:] = F[:34, 1:] - F[:34, :-1]
    same = (F[34:] == d) | (np.isnan(F[34:]) & np.isnan(d))
    same &= np.signbit(F[34:]) == np.signbit(d)
    if not same.all():
        r, t = (int(v[0]) for v in np.nonzero(~same))
        raise AssertionError("%s: delta row %d frame %d is %r, the row difference %r" % (what, 34 + r, t, F[34 + r, t], d[r, t]))

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

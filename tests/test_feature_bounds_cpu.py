"""The per-entry feature bound of ``tests/parity.feature_bounds``: its derivation, and a float32 emulation of the kernels'
feature path held to it on the adversarial bank (no device needed).

**What is bounded.**  Every short-term feature is a function of the magnitude spectrum |X| / K of a frame (rows 3..33)
or of the frame's normalised samples y (rows 0..2).  ``spectrum_reference`` bounds what a float32 transform may return
for a frame: the 2-norm of the error over bins 1 .. K-1 within eps_b, the DC bin within eps_0 (a constant frame's bins
1 .. K-1 exactly zero).  The bound of a feature entry is the sum of (a) the largest change of the float64 feature over
that ball of spectra, carried rigorously, and (b) the error of evaluating the feature in float32 from the spectrum the
kernel holds.

**(a) Transform error.**  Over |d_0| <= eps_0, |d_1..K-1|_2 <= eps_b:
* a linear functional sum a_k X_k moves by at most |a_0| eps_0 + |a_1..|_2 eps_b (sum X, sum (k+1) X / K, the 40 mel
  bands);
* a weighted sum of squares sum a_k X_k^2 by at most 2 |a X|_2 eps_b + max |a| eps_b^2 (DC likewise): sum X^2, the
  spectral-entropy blocks, the chroma classes, the rolloff prefixes.
Ratios A / B are carried with centred weights: A'/B' - A/B = sum (a_k - A/B) d_k / B' (the squares' form for sums of
squares), B' >= B - |dB|; where that interval of B reaches 0 the entry is unbounded.  Then:
* centroid c: weights (k+1)/K - c.  Spread: V = spr^2 = sum w_k X_k / S with w_k = ((k+1)/K - c)^2 at the exact c; since c'
  minimises the second moment about any point, V' = sum w_k X'_k / S' - (c' - c)^2, so |V' - V| <= the centred ratio bound
  with weights w_k - V, plus dc^2; sqrt(V) moves by at most sqrt(V) - sqrt(max(V - dV, 0)).
* entropy (spectral and energy): each share s_j = e_j / E within its interval, h(s) = -s log2(s + eps) is concave with its
  maximum near 1/e, so its range over the interval is read off the endpoints and that maximum; the ten deviations add.
* flux: sqrt(flux) = |X / Sn - Xp / Snp|_2 with Sn = S + K eps; each side moves by at most (|d|_2 + |X / Sn|_2 dS) /
  (Sn - dS) (triangle inequality), and flux by (sqrt(flux) + D)^2 - flux.
* rolloff: g_k = cumsum_k X^2 + eps - 0.9 E has weights 1[j <= k] - 0.9.  The admissible quanta run from the first k whose
  g_k may be > 0 to the first k whose g_k must be; where the float64 prefixes clear the threshold by more than their bound
  that range is one quantum, and there is no count allowance anywhere.
* mfcc: |dlog10 m_i| <= log10((m_i + eps) / (m_i - dm_i + eps)); a band whose interval contains 0 makes the frame's 13
  mfcc entries unbounded (reported with that reason, never skipped).  Then |dmfcc_j| <= sum_i |D_ji| |dlog10 m_i|.
* chroma_std is 1-Lipschitz in the RMS norm: it moves by at most the RMS of its twelve classes' bounds.
* time domain: the kernels compute y = fma(a, x - m, bp) with a, bp rounded to float32 (and x - m rounded for float32
  input; the generic kernel rebuilds x - m as (x - m - d0) + d0), so each sample is within beta_n = 4 u (|y_n| + |y_0| +
  |bp|) of the float64 y; energy and the energy-entropy shares take sum over the samples of 2 |y| beta + beta^2.  zcr of
  int16 input is an exact count (one rounding); for float32 input a sample with |y_n| <= beta_n may change sign class,
  and each such sample may change the count by 2 flips (2 / (w - 1)).
* deltas: b(t) + b(t - 1) plus the rounding of the float32 subtraction.

**(b) Float32 feature stage.**  One model for every kernel kind (u = 2^-24, gamma_n = n u / (1 - n u)):
* a sum over n bins or samples passes each term through at most ceil(n / 16) + 12 roundings: per-lane sequential chunks
  (16-lane layouts hold at most ceil(n / 16) terms per lane), at most 5 shuffle levels, entropy parts, and the fma of the
  term; sums of non-negative terms err by gamma of that depth times the sum (Higham, Accuracy and Stability of Numerical
  Algorithms, 2nd ed., section 3.1).  A mel band or chroma class sums its taps sequentially: gamma(taps + 2 or 3);
* ``fdiv`` (``__fdividef``): 2 ulp (CUDA C++ Programming Guide, "Intrinsic Functions", for divisors in [2^-126, 2^126],
  which every divisor here is: sums plus eps); IEEE division is inside that;
* ``flog2`` (``lg2.approx.ftz.f32``, the instruction behind ``__log2f``): absolute error 2^-22 on [0.5, 2], otherwise 2 ulp
  (Programming Guide, ``__log2f``; the ftz form only flushes subnormal inputs, and every input here is >= eps);
  ``log10f`` and ``log2f``: 2 and 1 ulp (Programming Guide, single-precision mathematical functions); the kernels'
  0.30103 * flog2 adds two roundings;
* ``fsqrt_pos`` (x * ``rsqrt.approx.ftz.f32``): 2 ulp for rsqrt (Programming Guide, ``rsqrtf``) plus the product;
  ``sqrtf`` is within that.  The pair and solo kernels' ``sqrt.approx.ftz.f32`` sits in the magnitude |X| itself, inside
  the spectrum bound's per-bin allowance; its 2 ulp is an ASSUMPTION (the PTX ISA gives no figure for it);
* the spread's offsets (k + 1) / K - c are stepped across a lane's bins by repeated adds: each drifts by at most
  (ceil(K / 16) + 4) u, which enters the spread's sum through sum |d| X <= sqrt(spr^2 S) S^(1/2);
* the DCT: float32 table, a constant offset subtracted from the log-mel values (m_0 or their mean) and at most 48
  roundings per term: gamma_48 sum |D_j| (range of log m + gamma_8 max |log m|), row 0 also 6.33 gamma_48 max |log m|;
* products of (1 + relative error) factors are kept to first order with a 1 % margin, and the float64 reference's own
  round-off is allowed 1e-12 relative.

**Soundness** (``test_emulation_within_bound``): the bank, int16 and float32, at every window of the adversarial feature
configs, through a float32 emulation: scipy's float32 FFT of z = y_frame - y_frame[0] (DC from float64), then every
feature in float32 the way the generic kernel orders it, rolloff by lane chunks and a scan.  A spectrum moved by the full
eps_b along the worst direction of a linear functional (sum X, sum (k+1) X, the most sensitive mel band) must stay inside
too (``test_worst_direction_within_bound``).

**Sensitivity.**  Defects planted in the emulation by hand (not committed), over the 399 clips of the 19 windows above:
* bin 5 floor(K / 10) counted in spectral-entropy block 4 instead of 5: the bound fails on 360 clips, the flat check on 367;
* one sample moved across an energy-entropy block boundary: both fail on all 399;
* rolloff one quantum late when the crossing falls on a lane chunk's first bin: both fail on the same 294;
* the spread as a one-pass float32 E[k^2] - c^2: NEITHER fails.  Its error (a few u times E[k^2] / spr) stays below the
  bound, whose worst direction puts the spectrum error on the bins farthest from the centroid, and below the
  arithmetic allowance for the kernels' own stepped offsets (k + 1) / K - c.  The bound cannot tell that defect from
  the error a float32 transform is allowed, so it is not a test of it.
The flat check misses none of the three that the bound catches; the bound's gain is elsewhere: it holds every entry to
its own float32 error, with no exception list, no absolute floor and no rolloff flip allowance.
"""
import numpy as np
import pytest
import scipy.fft

from oracle import st_oracle as O
from tests import signals as SG
from tests.parity import check_feature_bounds, clip_norm, feature_bounds

# the (fs, window, hop) of tests/test_gpu_adversarial.py FEATURE_CONFIGS
FEATURE_WINDOWS = [(16000, 320, 160), (16000, 480, 240), (16000, 512, 256), (16000, 640, 320), (16000, 800, 400),
                   (48000, 960, 480), (16000, 1024, 512), (16000, 800, 800), (16000, 800, 200), (16000, 800, 333),
                   (16000, 1024, 300), (44100, 882, 441), (44100, 882, 300), (16000, 400, 160), (16000, 400, 200),
                   (8000, 600, 300), (22050, 551, 200), (16000, 883, 300), (16000, 2048, 1024)]
F = np.float32
EPS32 = F(O.EPS)


def emulate_spectrum(x, w, s):
    """(y frames in float32 as the kernels stage them, |X| / K in float32): the transform of d - d0 in float32 (d = x - m),
    scaled by a / K; the DC bin from float64."""
    x = np.asarray(x)
    a, bp = clip_norm(x)
    xd = x.astype(np.float64)
    m = np.rint(xd.mean()) if x.dtype == np.int16 else float(F(xd.mean()))
    d = (x.astype(F) - F(m)).astype(F)
    T = O.frame_count(len(x), w, s)
    idx = s * np.arange(T)[:, None] + np.arange(w)[None, :]
    dfr = d[idx]
    yfr = (F(a) * dfr.astype(np.float64) + F(bp)).astype(F)
    z = (dfr - dfr[:, :1]).astype(F)
    K = w // 2
    X = (np.abs(scipy.fft.fft(z, axis=1))[:, :K] * F(F(a) / F(K))).astype(F)
    y = O.normalize_clip(xd)[idx]
    X[:, 0] = np.abs(y.sum(axis=1)) / K
    return yfr, X


def _blocks(v, n):
    L = v.shape[1] // 10
    return np.stack([v[:, j * L:(j + 1) * L].sum(axis=1, dtype=F) for j in range(10)], axis=1)


def _entropy(parts, tot):
    sj = (parts / (tot + EPS32)[:, None]).astype(F)
    return (-(sj * np.log2(sj + EPS32))).sum(axis=1, dtype=F)


def emulate_features(yfr, X, fs, deltas=True):
    """The 34 (68) rows in float32 from the float32 frames and spectra."""
    T, w = yfr.shape
    K = X.shape[1]
    out = np.zeros((34, T), dtype=F)
    sg = np.sign(yfr)
    out[0] = F(np.abs(np.diff(sg, axis=1)).sum(axis=1) * 0.5) / F(w - 1)
    E = (yfr * yfr).sum(axis=1, dtype=F)
    out[1] = E / F(w)
    out[2] = _entropy(_blocks(yfr * yfr, w), E)
    kk = (np.arange(1, K + 1, dtype=F) * F(1.0 / K)).astype(F)
    S = X.sum(axis=1, dtype=F)
    Sk = (X * np.arange(1, K + 1, dtype=F)).sum(axis=1, dtype=F)
    cen = np.where(S > 0, (Sk / np.where(S > 0, S, 1)) * F(1.0 / K), 0).astype(F)
    dv = (kk[None, :] - cen[:, None]).astype(F)
    sp = (dv * dv * X).sum(axis=1, dtype=F)
    out[3] = cen
    out[4] = np.where(S > 0, np.sqrt(sp / np.where(S > 0, S, 1)), 0)
    P = (X * X).astype(F)
    Et = P.sum(axis=1, dtype=F)
    out[5] = _entropy(_blocks(P, K), Et)
    nx = (F(1) / (S + F(K) * EPS32)).astype(F)
    Xn = (X * nx[:, None]).astype(F)
    Xp = np.vstack([Xn[:1], Xn[:-1]])
    out[6] = ((Xn - Xp) ** 2).sum(axis=1, dtype=F)
    # rolloff: lanes of c = odd(ceil(K / 32)) consecutive bins, an inclusive scan of the lane parts, then each lane walks
    # its chunk from the exclusive prefix incl - part
    c = -(-K // 32) | 1
    Pp = np.zeros((T, 32 * c), dtype=F)
    Pp[:, :K] = P
    ch = Pp.reshape(T, 32, c)
    part = ch.sum(axis=2, dtype=F)
    incl = np.cumsum(part, axis=1, dtype=F)
    run = np.cumsum(np.concatenate([(incl - part)[:, :, None], ch], axis=2), axis=2, dtype=F)[:, :, 1:]
    thr = (F(0.9) * Et - EPS32).astype(F)
    over = run.reshape(T, -1)[:, :K] > thr[:, None]
    out[7] = np.where(over.any(axis=1), np.argmax(over, axis=1), 0).astype(F) * F(1.0 / K)
    M, D, C = (t.astype(F) for t in (O.mel_filterbank(fs, K), O.dct_matrix(), O.chroma_operator(fs, K)))
    lm = np.log10(X @ M.T + EPS32).astype(F)
    mbar = lm.mean(axis=1, dtype=F)
    mf = ((lm - mbar[:, None]) @ D.T).astype(F)
    mf[:, 0] = F(6.324555320336759) * mbar
    out[8:21] = mf.T
    chv = ((P @ C.T) / np.where(Et == 0, EPS32, Et)[:, None]).astype(F)
    out[21:33] = chv.T
    out[33] = chv.std(axis=1, dtype=F)
    if not deltas:
        return out
    d = np.zeros_like(out)
    d[:, 1:] = out[:, 1:] - out[:, :-1]
    return np.concatenate([out, d])


def bank_clips(fs, w, s):
    return list(SG.bank(fs, w, s).items()) + list(SG.float_bank(fs, w, s).items())


@pytest.mark.parametrize("fs,w,s", FEATURE_WINDOWS, ids=["%d-%d-%d" % c for c in FEATURE_WINDOWS])
def test_emulation_within_bound(fs, w, s):
    worst = {}
    unb = {}
    for name, x in bank_clips(fs, w, s):
        fb = feature_bounds(x, fs, w, s, deltas=True)
        got = emulate_features(*emulate_spectrum(x, w, s), fs)
        r, u = check_feature_bounds(got, fb, "float32 emulation, fs=%d w=%d s=%d: %s" % (fs, w, s, name))
        for k, v in r.items():
            worst[k] = max(worst.get(k, 0.0), v)
        for k, v in u.items():
            unb[k] = unb.get(k, 0) + v
    print("fs=%d w=%d s=%d: worst err / bound %s; unbounded entries %s" % (fs, w, s, worst, unb))


def _worst_directions(x, fs, w, s):
    """Per frame, unit directions over bins 1 .. K-1 (DC kept) of the linear functionals sum X, sum (k+1) X and the mel
    band with the largest eps_b |M_i|_2 / m_i among those whose interval stays above 0."""
    from tests.parity import _tables, spectrum_reference
    K = w // 2
    T = O.frame_count(len(x), w, s)
    X, eb, _, flat = spectrum_reference(x, s * np.arange(T), w)
    M = _tables(fs, K)[0]
    m = X @ M.T
    sens = np.linalg.norm(M[:, 1:], axis=1)[None, :] * eb[:, None] / np.where(m > 0, m, np.inf)
    sens = np.where(sens < 1, sens, -1)
    band = M[np.argmax(sens, axis=1)]                                            # [T, K]
    dirs = [np.ones((T, K)), np.broadcast_to(np.arange(1, K + 1) / K, (T, K)), band]
    out = []
    for a in dirs:
        a = np.array(a, dtype=np.float64)
        a[:, 0] = 0
        out.append(a / np.linalg.norm(a, axis=1, keepdims=True))
    return X, np.where(flat, 0.0, eb), out


@pytest.mark.parametrize("fs,w,s", FEATURE_WINDOWS[::3], ids=["%d-%d-%d" % c for c in FEATURE_WINDOWS[::3]])
def test_worst_direction_within_bound(fs, w, s):
    """Every frame's spectrum moved by the full eps_b along a linear functional's worst direction (both signs, magnitudes
    kept >= 0, which only shortens the move): all 68 float64 rows stay inside the bound."""
    for name, x in bank_clips(fs, w, s):
        fb = feature_bounds(x, fs, w, s, deltas=True)
        y = O.normalize_clip(x.astype(np.float64))
        T = fb.ref.shape[1]
        fr = y[s * np.arange(T)[:, None] + np.arange(w)[None, :]]
        X, eb, dirs = _worst_directions(x, fs, w, s)
        for j, a in enumerate(dirs):
            for sign in (1.0, -1.0):
                Xq = np.maximum(X + sign * eb[:, None] * a, 0.0)
                base = O.base_features_from_frames(fr, Xq, fs)
                got = np.concatenate([base, np.diff(base, axis=1, prepend=base[:, :1])])
                check_feature_bounds(got, fb, "fs=%d w=%d s=%d %s: direction %d, sign %+d" % (fs, w, s, name, j, sign))

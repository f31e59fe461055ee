"""Deterministic adversarial signals for the short-term feature kernels.

Every signal targets one mechanism that broadband, evenly loud test clips (``st_oracle.synth_clip``) cannot reach:
per-frame scaling of quiet frames next to loud ones, the block-energy ring, the one- and two-mask zero-crossing
counts, the int16 load, exactly constant frames.  All are int16 and about one second long, each of a different
length so that a batch of them is ragged.

Some inputs make the reference's own answer float64 round-off: a frame whose samples are all equal has an exactly
zero spectrum beyond DC, its mel bands become ``log10(round-off + eps)`` and its spectral spread is round-off.
``noise_defined_frames`` marks those frames; ``patch_noise_defined`` puts the exact values of a DC-only spectrum into
those rows of a reference matrix, and every row is then compared as usual.  The bank
avoids the other inputs of that kind (tones exactly on a bin, periods that divide the window, Nyquist alternation)
and keeps the spectral range inside each frame to about 60 dB; the range between frames is large on purpose.
"""
import math

import numpy as np

from oracle import st_oracle as O

SPREAD_ROW = 4
MFCC_ROWS = np.arange(8, 21)         # mfcc_1..13 of the 34 base rows


def _i16(x):
    return np.round(np.clip(x, -32768, 32767)).astype(np.int16)


def _frames_per_span(window, hop):
    return -(-window // hop)         # hop-length blocks a frame touches


def loud_quiet(rng, n, fs, window, hop):
    """Hop-length blocks: one loud block (full-scale off-bin tone + noise) then quiet N(0, 2) blocks, with a period of
    frames-per-window + 2 blocks, so that frames are loud or quiet and pairs (2q, 2q + 1) meet loud / quiet in both
    orders."""
    period = _frames_per_span(window, hop) + 2
    t = np.arange(n)
    f = fs * (37.37 / window)                   # 37.37 bins: off-bin
    loud = 22000.0 * np.sin(2 * np.pi * f * t / fs) + rng.normal(0, 2000.0, n)
    quiet = rng.normal(0, 2.0, n)
    return _i16(np.where((t // hop) % period == 0, loud, quiet))


def level_ramp(rng, n):
    return _i16(rng.normal(0, 8000.0, n) * 10.0 ** (-90.0 / 20.0 * np.arange(n) / n))


def triangle(rng, n):
    """The symmetric +-2000 triangle (period 8000) plus integer noise v - reverse(v), whose sum is exactly 0: the clip mean
    stays exactly 0.  The noise (about 5 LSB rms) holds the spectral range of frames around a corner, where the
    triangle's spectrum falls as 1/k^2, to about 60 dB; the noise-free wave goes beyond 100 dB there, below float32
    resolution of the transform."""
    sym = np.concatenate([np.arange(-2000, 2000), np.arange(2000, -2000, -1)])
    x = np.tile(sym, max(1, int(round(n / sym.size))))
    v = rng.integers(-6, 7, x.size)
    return (x + v - v[::-1]).astype(np.int16)


def integer_mean(rng, n, m=7):
    x = np.round(m + rng.normal(0, 300.0, n)).astype(np.int64)
    x[rng.random(n) < 0.4] = m
    r = int(x.sum() - m * n)                   # move the sum onto m * n with the last samples
    k = max(1, -(-abs(r) // 1000))
    x[n - k:] -= r // k
    x[-1] -= int(x.sum() - m * n)
    assert x.sum() == m * n and np.abs(x).max() < 32767
    return x.astype(np.int16)


def rails(rng, n):
    return _i16(rng.normal(0, 30000.0, n))


def dc_offset(rng, n):
    return (20000 + rng.integers(-3, 4, n)).astype(np.int16)


def edge_impulses(rng, n, window, hop):
    """Low noise with +-20000 impulses on the first sample of frames 5j and on the last sample of frames 5j + 2."""
    x = rng.normal(0, 2.0, n)
    T = O.frame_count(n, window, hop)
    for t in range(0, T, 5):
        x[t * hop] = 20000.0
    for t in range(2, T, 5):
        x[t * hop + window - 1] = -20000.0
    return _i16(x)


def constant_runs(rng, n, window, hop):
    """Noise in the first and last fifth, the constant 1000 in between, where every (frames-per-window + 1)-th frame gets
    one differing sample at its first, middle or last position in turn (no frame touches two of them).  Frames touching
    no differing sample are exactly constant."""
    x = rng.normal(0, 3000.0, n)
    a, b = n // 5, n - n // 5
    x[a:b] = 1000.0
    t0 = -(-a // hop)
    T = O.frame_count(n, window, hop)
    pos = (0, window // 2, window - 1)
    j = 0
    for t in range(t0 + 1, T, _frames_per_span(window, hop) + 1):
        p = t * hop + pos[j % 3]
        if p + window > b:
            break
        x[p] = 1000.0 + (1 if j % 2 else -1) * 9000.0
        j += 1
    return _i16(x)


def dither(rng, n):
    return rng.integers(-1, 2, n).astype(np.int16)


def chirp(rng, n, fs):
    t = np.arange(n) / fs
    f0, f1, dur = 50.0, 0.45 * fs, n / fs
    k = math.log(f1 / f0) / dur
    return _i16(20000.0 * np.sin(2 * np.pi * f0 * (np.exp(k * t) - 1) / k) + rng.normal(0, 300.0, n))


# name -> one-line note on the mechanism the signal targets
NOTES = {
    "loud_quiet": "80 dB loud / quiet hop blocks: per-frame scale sa / sb, separation, block-energy ring",
    "level_ramp": "noise on an exponential ramp down to -90 dB: per-frame scaling over the whole range",
    "triangle": "symmetric triangle + zero-sum noise, clip mean exactly 0: two-mask zcr, spectrum falling 1/k^2",
    "integer_mean": "40 % of samples equal the integer clip mean: two-mask zcr, zeros between sign changes",
    "rails": "noise clipped to -32768 and 32767: x ^ 0x8000 load, min / max of the clip statistics",
    "dc_offset": "DC 20000 with +-3 LSB: centring, the bp offset of the normalisation",
    "edge_impulses": "impulses on a frame's first sample (the x - x[0] subtraction) and on its last",
    "constant_runs": "constant frames (exact zero spectrum) and frames with one differing sample (must not be zeroed)",
    "dither": "+-1 LSB dither: smallest non-zero level",
    "chirp": "log chirp 50 Hz .. 0.45 fs: every bin in turn",
}


def bank(fs, window, hop):
    """{name: int16 clip} for one (fs, window, hop); lengths differ by a few samples per signal."""
    out = {}
    for i, name in enumerate(NOTES):
        rng = np.random.default_rng(9000 + 17 * i)
        n = fs + 37 * i + 11
        if name == "loud_quiet":
            x = loud_quiet(rng, n, fs, window, hop)
        elif name == "level_ramp":
            x = level_ramp(rng, n)
        elif name == "triangle":
            x = triangle(rng, n)
        elif name == "integer_mean":
            x = integer_mean(rng, n)
        elif name == "rails":
            x = rails(rng, n)
        elif name == "dc_offset":
            x = dc_offset(rng, n)
        elif name == "edge_impulses":
            x = edge_impulses(rng, n, window, hop)
        elif name == "constant_runs":
            x = constant_runs(rng, n, window, hop)
        elif name == "dither":
            x = dither(rng, n)
        else:
            x = chirp(rng, n, fs)
        out[name] = x
    return out


def float_bank(fs, window, hop):
    """float32 variants: every int16 signal x 0.37 + 11.5, and one clip at 1e-3 full scale."""
    out = {name + "_f32": (x.astype(np.float32) * np.float32(0.37) + np.float32(11.5)) for name, x in bank(fs, window, hop).items()}
    rng = np.random.default_rng(9999)
    out["small_f32"] = (rng.normal(0, 1e-3 / 3, fs + 5) + 1e-3 * np.sin(np.arange(fs + 5) * 0.0371)).astype(np.float32)
    return out


def constant_frames(x, window, starts):
    """Boolean per frame start: every sample of x[s : s + window] equals x[s]."""
    x = np.asarray(x)
    eq = np.concatenate([[0], np.cumsum(x[1:] != x[:-1])])       # number of changes up to each sample
    starts = np.asarray(starts, dtype=np.int64)
    return eq[starts + window - 1] == eq[starts]


def noise_defined_frames(x, window, hop):
    """Frames of feature_extraction whose mfcc rows are float64 round-off in the reference."""
    return constant_frames(x, window, hop * np.arange(O.frame_count(len(x), window, hop)))


def zero_spectrum_rows():
    """(rows, values) of a frame with no energy outside DC: spectral_spread 0 (the reference's is eps-sized round-off),
    and mfcc_1..13 of log10(eps) in every mel band (the mel bank never reaches bin 0)."""
    return np.concatenate([[SPREAD_ROW], MFCC_ROWS]), np.concatenate([[0.0], O.dct_matrix() @ np.full(O.N_MEL, math.log10(O.EPS))])


def patch_noise_defined(F, x, window, hop):
    """The oracle / reference matrix F with the noise-defined rows of constant frames replaced by the exact values of a
    DC-only spectrum (deltas recomputed).  Returns (patched copy, mask of noise-defined frames)."""
    F = np.array(F, dtype=np.float64)
    bad = noise_defined_frames(x, window, hop)
    if bad.any():
        rows, vals = zero_spectrum_rows()
        F[rows[:, None], np.nonzero(bad)[0][None, :]] = vals[:, None]
        if F.shape[0] == 2 * O.N_BASE:
            F[O.N_BASE:, 1:] = F[:O.N_BASE, 1:] - F[:O.N_BASE, :-1]
            F[O.N_BASE:, 0] = 0.0
    return F, bad

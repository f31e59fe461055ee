"""GPU: the magnitude spectrum |X[k]| / K of every kernel against a float64 DFT, under a bound derived from float32 FFT
arithmetic.

Spectral features, mel bands, MFCCs, chroma and spectrogram rows are all built from this spectrum, and the feature checks
see it only through sums, logs and ratios, where an error in a few bins or in a quiet frame mostly cancels.  Here the
spectrum itself is the thing under test, everywhere it is computed:

* pair kernel (windows 32 R): the |X| rows it dumps through ``b200aa_debug_set_dump`` during a feature launch;
* solo and CTA kernels: their spectrogram rows (the row modes run the same transform code as the feature paths), the
  CTA kernel also on a view with an odd sample offset, which selects its other staging variant;
* generic kernel: spectrogram rows of a ``force_generic`` plan at the windows of ``tests.kernels.GENERIC_SWEEP``, each
  chosen for the code path it reaches (radix passes, packed / unpacked transform, frames per CTA group, global scratch).

**Reference and bound** (``tests/parity.spectrum_reference``).  Reference: |DFT(y_frame)|[0:K] / K in float64, y the
normalised clip.  Every kernel transforms z = y_frame - y_frame[0] (so that a constant frame gives exact zeros), and the
float32 error of a transform is relative to the norm of what it transforms.  By Parseval nu = sqrt(N) |z|_2 / K is the
2-norm of z's whole spectrum on the output's scale, and per frame

    |got - ref|_2 over bins 1 .. K-1  <=  C u ceil(log2 N) nu,        u = 2^-24,

the DC bin (a plain sum, then N times the first sample added back) within C u (|z|_1 + N |y_frame[0]|) / K, and a
constant frame's bins 1 .. K-1 exactly zero.  For float32 input, x - x[0] is rounded once per sample: u |y_frame|_2 is
added to |z|_2.  The pair kernel's bound uses each frame's OWN z, never its partner's: that its per-frame scale keeps
either spectrum's error relative to its own level (DESIGN section 4) is what this checks.

**Choosing C = 8** (fixed before any GPU measurement).  For a radix-2 FFT of length n in floating point with twiddles
of relative error mu, Higham (Accuracy and Stability of Numerical Algorithms, 2nd ed., Theorem 24.2) gives
|err|_2 <= log2(n) eta / (1 - log2(n) eta) |y|_2 with eta = mu + gamma_4 (sqrt 2 + mu), gamma_4 = 4u / (1 - 4u): one
butterfly level costs eta.  Float32 twiddles rounded from float64 have mu <= u, so eta ~ (1 + 4 sqrt 2) u = 6.7 u.  A
radix-r codelet (4, 3, 5, 7) does the work of log2 r levels with the same per-operation rounding, so a mixed-radix
transform costs log2 n levels in all; the packed-real form (N/2 complex points, then one split per bin) spends the
level its half-length transform saved on that split.  The final scale by a / K, the two squares and their sum and the
square root add about 3u relative per bin.  So |err| <= (6.7 log2 N + 3) u nu <= 8 ceil(log2 N) u nu for every N >= 5
(smaller windows have K = 1: only the DC bin).  The generic kernel's direct pass for a prime radix above 7 sums p
terms per output; in float32 that sum errs by about sqrt(p) u of its terms' size, outside the model, so it
accumulates in fp64 and only its float32 inputs and twiddles round (accumulated in float32, the DC bin of the window
20 011 missed its bound by 3.5x: the partial sums of x - x[0] grow with the offset of x[0]).  The pass is still outside
the worst case: p twiddles each off by u give an error up to u |z|_1 per output, sqrt(p) u relative to the spectrum
(141 u at p = 20 011, against C ceil(log2 N) = 120 u).  It stays inside the bound because those p rounding errors are
independent and of either sign, so they add up like a random walk, about u relative.  The pair kernel
transforms two frames as one complex sequence, where the partner adds at most a factor sqrt(5) to the worst case
(per-frame scales are powers of two, so the two scaled energies are within a factor 4).  The worst-case bound is far
above the typical error (rounding errors add up like a random walk, about u sqrt(log2 N)), while one wrong bin among
K bins of similar size gives about 1 / sqrt(K): thousands of times the bound.  The worst measured err / bound per
kernel kind and window class is recorded in DESIGN section 6.
"""
import pytest

from tests.kernels import CTA, CTA_CONFIGS, GENERIC_SWEEP, PAIR_CONFIGS, SOLO, SOLO_CONFIGS
from tests.parity import generic_spectra, pair_spectra, row_spectra

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


@pytest.mark.parametrize("fs,w,s", PAIR_CONFIGS, ids=["%d-%d-%d" % c for c in PAIR_CONFIGS])
def test_pair_kernel_spectra(P, fs, w, s):
    pair_spectra(P, fs, w, s)


@pytest.mark.parametrize("fs,w,s", SOLO_CONFIGS, ids=["%d-%d-%d" % c for c in SOLO_CONFIGS])
def test_solo_kernel_spectra(P, fs, w, s):
    from pyaudioanalysis_b200._lib import Plan
    pl = Plan(fs, w, s).prefer_kernel(SOLO)
    assert pl.kernel_kind() == SOLO
    row_spectra(P, pl, fs, w, s, "solo")


@pytest.mark.parametrize("fs,w,s", CTA_CONFIGS, ids=["%d-%d-%d" % c for c in CTA_CONFIGS])
def test_cta_kernel_spectra(P, fs, w, s):
    from pyaudioanalysis_b200._lib import Plan
    pl = Plan(fs, w, s).prefer_kernel(CTA)
    assert pl.kernel_kind() == CTA
    row_spectra(P, pl, fs, w, s, "CTA", offset_view=True)


@pytest.mark.parametrize("fs,w,G,path", GENERIC_SWEEP, ids=["w%d" % c[1] for c in GENERIC_SWEEP])
def test_generic_kernel_spectra(P, fs, w, G, path):
    generic_spectra(P, fs, w, path)

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
import contextlib
import ctypes

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import CTA, GENERIC_SWEEP, PAIR, SOLO, ragged
from tests.parity import check_spectrogram_rows, check_spectrum

pytestmark = pytest.mark.gpu

# pair kernel: every window at hop N / 2 (shared halves), and the independent-frame path at other hops
PAIR_CONFIGS = [(16000, 320, 160), (16000, 480, 240), (16000, 512, 256), (16000, 640, 320), (16000, 800, 400),
                (48000, 960, 480), (16000, 1024, 512), (16000, 800, 200), (16000, 800, 333), (16000, 800, 800),
                (16000, 1024, 300)]
SOLO_CONFIGS = [(44100, 882, 441), (44100, 882, 300), (16000, 400, 200), (16000, 400, 160), (8000, 600, 300)]
CTA_CONFIGS = [(16000, 320, 160), (16000, 400, 200), (16000, 480, 240), (8000, 600, 300), (16000, 640, 320),
               (16000, 800, 400), (16000, 800, 200), (16000, 800, 333), (44100, 882, 441)]
ODD = 3                 # sample offset of the unaligned view


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


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


def odd_tail(fs, w, s):
    """A clip with an odd frame count whose last frame (paired with itself) is loud in its first half and 80 dB quieter in
    its second: with shared halves the partner's energy is not the frame's own, and a scale taken from it buries the
    frame under its copy."""
    rng = np.random.default_rng(w + s)
    T = 2 * (fs // (2 * s)) + 1
    n = w + (T - 1) * s
    x = rng.normal(0, 2.0, n)
    a = (T - 1) * s
    t = np.arange(w // 2)
    x[a:a + w // 2] = 20000.0 * np.sin(2 * np.pi * 37.37 * t / w) + rng.normal(0, 300.0, w // 2)
    x = np.round(x).astype(np.int16)
    assert O.frame_count(n, w, s) == T and T % 2 == 1
    return x


def pair_spectra(P, fs, w, s):
    """The bank plus odd_tail (int16 and float32) as ragged feature batches through the pair kernel, every frame's dumped
    |X| row under the spectrum bound, exactly the frames below each clip's frame count written.  Returns the
    (bins, DC) err / bound of every clip."""
    from pyaudioanalysis_b200._lib import Plan
    pl = Plan(fs, w, s).prefer_kernel(PAIR)
    assert pl.kernel_kind() == PAIR
    K = w // 2
    ints = dict(SG.bank(fs, w, s), odd_tail=odd_tail(fs, w, s))
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


@pytest.mark.parametrize("fs,w,s", PAIR_CONFIGS, ids=["%d-%d-%d" % c for c in PAIR_CONFIGS])
def test_pair_kernel_spectra(P, fs, w, s):
    pair_spectra(P, fs, w, s)


def row_spectra(P, pl, fs, w, s, kind_name, offset_view=False):
    """The bank (int16 and float32) as ragged batches through spectrogram_batch on plan pl, every clip's rows under the
    spectrum bound; with offset_view also the int16 batch as a view at an odd sample offset.  Returns
    {"int16" | "float32" | "odd offset": [(bins, DC) err / bound of every clip]}."""
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


def sweep_clips(w):
    """Two int16 clips (noise; noise with a loud first sample in every other frame) and one float32 clip (a chirp),
    long enough for five full spectrogram rows and a few rows past them."""
    s = max(1, w // 2)
    n = 2 * w + 5 * s + 3
    rng = np.random.default_rng(w)
    noise = np.round(rng.normal(0, 3000.0, n)).astype(np.int16)
    edges = np.round(rng.normal(0, 30.0, n))
    edges[w::2 * s] = 20000.0
    t = np.arange(n)
    chirp = (0.3 * np.sin(2 * np.pi * (0.01 + 0.4 * t / n) * t) + rng.normal(0, 0.01, n)).astype(np.float32)
    return s, [noise, edges.astype(np.int16)], chirp


def generic_spectra(P, fs, w, path):
    """sweep_clips through a force_generic plan (the int16 clips as a ragged batch, the float32 clip alone), every row
    under the spectrum bound.  Returns the (bins, DC) err / bound of every clip."""
    import torch
    from pyaudioanalysis_b200._lib import Plan
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


@pytest.mark.parametrize("fs,w,G,path", GENERIC_SWEEP, ids=["w%d" % c[1] for c in GENERIC_SWEEP])
def test_generic_kernel_spectra(P, fs, w, G, path):
    generic_spectra(P, fs, w, path)

"""Kernel kinds and the configurations the tests run them at, shared by the test modules and the golden generators: the
kernel kinds a plan reaches, the (fs, window, hop) lists of each sweep, the specialised windows and sample rates, and
ragged batches on the device."""
import numpy as np

PAIR, SOLO, CTA, GENERIC = 2, 3, 1, 0
KIND_NAMES = {PAIR: "pair", SOLO: "solo", CTA: "CTA", GENERIC: "generic"}

# Feature configs of the adversarial bank (tests/test_gpu_adversarial.py, tests/test_gpu_feature_bounds.py): (fs, window,
# hop) and the kernel kinds a plan reaches through prefer_kernel / force_generic
FEATURE_CONFIGS = [
    (16000, 320, 160, {PAIR, CTA, GENERIC}), (16000, 480, 240, {PAIR, CTA, GENERIC}), (16000, 512, 256, {PAIR, GENERIC}),
    (16000, 640, 320, {PAIR, CTA, GENERIC}), (16000, 800, 400, {PAIR, CTA, GENERIC}), (48000, 960, 480, {PAIR, GENERIC}),
    (16000, 1024, 512, {PAIR, GENERIC}), (16000, 800, 800, {PAIR, CTA, GENERIC}), (16000, 800, 200, {PAIR, CTA, GENERIC}),
    (16000, 800, 333, {PAIR, CTA, GENERIC}), (16000, 1024, 300, {PAIR, GENERIC}),
    (44100, 882, 441, {SOLO, CTA, GENERIC}), (44100, 882, 300, {SOLO, CTA, GENERIC}), (16000, 400, 160, {SOLO, CTA, GENERIC}),
    (16000, 400, 200, {SOLO, CTA, GENERIC}), (8000, 600, 300, {SOLO, CTA, GENERIC}),
    (22050, 551, 200, {GENERIC}), (16000, 883, 300, {GENERIC}), (16000, 2048, 1024, {GENERIC}),
]
# Row configs (spectrogram / chromagram) of the adversarial bank and the chromagram bounds
ROW_CONFIGS = [(16000, 800, 400), (16000, 800, 333), (44100, 882, 441), (16000, 400, 160), (8000, 600, 300)]
# Spectrum checks per kernel kind (tests/test_gpu_spectra.py, scripts/spectrum_ratios.py).
# pair kernel: every window at hop N / 2 (shared halves), and the independent-frame path at other hops
PAIR_CONFIGS = [(16000, 320, 160), (16000, 480, 240), (16000, 512, 256), (16000, 640, 320), (16000, 800, 400),
                (48000, 960, 480), (16000, 1024, 512), (16000, 800, 200), (16000, 800, 333), (16000, 800, 800),
                (16000, 1024, 300)]
SOLO_CONFIGS = [(44100, 882, 441), (44100, 882, 300), (16000, 400, 200), (16000, 400, 160), (8000, 600, 300)]
CTA_CONFIGS = [(16000, 320, 160), (16000, 400, 200), (16000, 480, 240), (8000, 600, 300), (16000, 640, 320),
               (16000, 800, 400), (16000, 800, 200), (16000, 800, 333), (44100, 882, 441)]

# Windows of the generic kernel's spectrum sweep (tests/test_gpu_spectra.py), each chosen for the code path it reaches:
# (fs, window, frames per CTA group, path).  The group size G (8, 4, 2, 1; 0 = global scratch) is what launch_generic
# picks (csrc/generic_kernel.cuh: generic_group) with the tables blob the plan for (fs, window) builds, which grows with
# the window (the mel taps: about 0.84 K + 900 words at 16 kHz); tests/test_smem_budget_cpu.py holds each claim to the
# budget formula at that blob and at 256 words either side of it.
# Even windows transform N/2 packed points, odd windows N real points; radices are 4s first, then primes ascending.
GENERIC_SWEEP = [
    (16000, 2, 8, "Nc = 1: empty radix list; K = 1"),
    (16000, 3, 8, "K = 1, odd: one radix-3 pass, unpacked"),
    (16000, 5, 8, "small odd window: radix 5"),
    (16000, 7, 8, "small odd window: radix 7"),
    (16000, 9, 8, "small odd window: radix 3, 3"),
    (16000, 8, 8, "4^n: one radix-4 pass"),
    (16000, 486, 8, "radix 3 alone (Nc = 3^5)"),
    (16000, 686, 8, "radix 7 alone (Nc = 7^3)"),
    (16000, 882, 8, "radix 3 and 7 mixed (Nc = 3^2 7^2)"),
    (16000, 630, 8, "radix 3, 5, 7 mixed (Nc = 3^2 5 7)"),
    (16000, 22, 8, "prime above 7: direct radix-11 pass"),
    (16000, 26, 8, "prime above 7: direct radix-13 pass"),
    (16000, 242, 8, "repeated prime above 7: two radix-11 passes"),
    (16000, 1688, 4, "4 and a prime above 7 mixed (Nc = 4 211)"),
    (16000, 1994, 4, "large prime: one direct radix-997 pass"),
    (16000, 441, 8, "odd composite (3^2 7^2), unpacked; last G = 8 odd window"),
    (16000, 1000, 8, "even, radix 4, 5 mixed; last G = 8 even window"),
    (16000, 883, 4, "odd prime, direct radix-883 pass; first G = 4 odd window"),
    (16000, 1250, 4, "radix 5 alone (Nc = 5^4); first G = 4 even window"),
    (16000, 1009, 4, "odd prime, direct radix-1009 pass"),
    (16000, 1323, 4, "odd composite (3^3 7^2)"),
    (16000, 2048, 4, "4^5"),
    (16000, 4096, 4, "4^5 2; last G = 4 even window"),
    (16000, 2401, 4, "odd, radix 7 alone (7^4); last G = 4 odd window"),
    (16000, 6000, 2, "first G = 2 even window"),
    (16000, 3375, 2, "odd, radix 3, 5 (3^3 5^3); first G = 2 odd window"),
    (16000, 9000, 2, "radix 4, 3, 5 (Nc = 4 3^2 5^3); last G = 2 even window"),
    (16000, 5103, 2, "odd, radix 3, 7 (3^6 7); last G = 2 odd window"),
    (16000, 11000, 1, "prime 11 among 4s and 5s; first G = 1 even window"),
    (16000, 6561, 1, "odd, radix 3 alone (3^8); first G = 1 odd window"),
    (16000, 15360, 1, "radix 4, 2, 3, 5 (Nc = 4^4 2 3 5); last G = 1 even window"),
    (16000, 10125, 1, "odd, radix 3, 5 (3^4 5^3); last G = 1 odd window"),
    (16000, 20000, 0, "global scratch, even"),
    (16000, 12005, 0, "global scratch, odd (5 7^4)"),
    (16000, 20011, 0, "global scratch, odd prime: one direct radix-20011 pass (its float32 DC sum missed the bound)"),
    (44100, 11025, 0, "0.25 s at 44.1 kHz, odd: global scratch with its blob of ~2 560 words (G = 1 below ~1 700)"),
]


# Sample rates of the specialised kernels (tests/test_gpu_rates.py; their tables: tests/test_rates_cpu.py).  The rate reaches a
# kernel only through its tables, whose layout changes with fs: (fs, window, hop, kernel kinds plans() reaches, what).
# The mel bank is refused below 6 854 Hz at every specialised window; just above it the last filter reaches bin K - 1, the
# only place where build_pair_blob moves a four-tap group back inside the row ("clamped").  Layouts: tests/test_rates_cpu.py.
RATE_CONFIGS = [
    (48000, 480, 240, {PAIR, CTA, GENERIC}, "10 ms at 48 kHz: 4 empty mel filters"),
    (44100, 320, 160, {PAIR, CTA, GENERIC}, "9 empty mel filters"),
    (44100, 512, 256, {PAIR, GENERIC}, "3 empty mel filters, chroma lists of 9 taps"),
    (24000, 320, 160, {PAIR, CTA, GENERIC}, "1 empty mel filter"),
    (8000, 800, 400, {PAIR, CTA, GENERIC}, "12 mel steps per lane"),
    (8000, 1024, 512, {PAIR, GENERIC}, "15 mel steps per lane"),
    (7000, 960, 480, {PAIR, GENERIC}, "17 mel steps per lane"),
    (6854, 1024, 512, {PAIR, GENERIC}, "the lowest accepted rate: 18 mel steps per lane (the largest pair blob), a clamped group"),
    (6854, 800, 400, {PAIR, CTA, GENERIC}, "the lowest accepted rate: a clamped group"),
    (11025, 1024, 512, {PAIR, GENERIC}, "11.025 kHz: 11 mel steps per lane"),
    (96000, 960, 480, {PAIR, GENERIC}, "96 kHz: 4 empty mel filters, chroma lists of 9 taps"),
    (192000, 1024, 512, {PAIR, GENERIC}, "192 kHz: 14 empty mel filters, chroma lists of 10 taps"),
    (44100, 400, 200, {SOLO, CTA, GENERIC}, "6 empty mel filters"),
    (48000, 600, 300, {SOLO, CTA, GENERIC}, "2 empty mel filters"),
    (8000, 882, 441, {SOLO, CTA, GENERIC}, "13 mel steps per lane"),
    (7000, 600, 300, {SOLO, CTA, GENERIC}, "11 mel steps per lane"),
    (6854, 600, 300, {SOLO, CTA, GENERIC}, "the lowest accepted rate: a clamped group"),
    (96000, 882, 441, {SOLO, CTA, GENERIC}, "96 kHz: 6 empty mel filters"),
    (16000, 800, 1000, {PAIR, CTA, GENERIC}, "hop longer than the window"),
    (16000, 800, 1600, {PAIR, CTA, GENERIC}, "hop longer than the window: the CTA kernel hands it to the generic kernel"),
    (16000, 320, 400, {PAIR, CTA, GENERIC}, "hop longer than the window"),
    (44100, 882, 1323, {SOLO, CTA, GENERIC}, "hop longer than the window"),
    (16000, 600, 900, {SOLO, CTA, GENERIC}, "hop longer than the window"),
]


# The (fs, window) sweep of the specialised kernels' tables (tests/test_rates_cpu.py, tests/golden/rates.npz): every
# specialised window at every rate of FINE and RATES.
PAIR_WINDOWS = [320, 480, 512, 640, 800, 960, 1024]
SOLO_WINDOWS = [400, 600, 882]
CTA_WINDOWS = [320, 400, 480, 600, 640, 800, 882]
WINDOWS = sorted(set(PAIR_WINDOWS + SOLO_WINDOWS + CTA_WINDOWS))
FINE = list(range(6300, 7101))               # the mel bank's refusal boundary at every specialised window
RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000]
# (window, hop) whose CTA staging exceeds its cap: the launcher returns unsupported and the generic kernel runs instead.
# With run staging (hop a multiple of 8) the 800-sample window crosses the cap from hop 1 200 (6 854 Hz) .. 1 232 (16 kHz).
CTA_FALLBACK = {(800, 1600)}


def plans(fs, w, s):
    """[(kind, Plan)] for every kernel kind a plan for (fs, w, s) reaches, the default choice first."""
    from pyaudioanalysis_b200._lib import Plan
    out = [(Plan(fs, w, s).kernel_kind(), Plan(fs, w, s))]
    for kind in (PAIR, SOLO, CTA):
        pl = Plan(fs, w, s).prefer_kernel(kind)
        if pl.kernel_kind() == kind:
            out.append((kind, pl))
    pg = Plan(fs, w, s)
    pg.force_generic(True)
    assert pg.kernel_kind() == GENERIC
    out.append((GENERIC, pg))
    return out


def ragged(clips, dtype, offset=0, pad=0):
    """[B, Nmax] CUDA batch of the clips and their lengths; samples past a clip's length are ``pad``.  offset 0: a view
    of a buffer with 16-byte aligned rows (a row stride that is a multiple of 8 samples); offset > 0: a view into a wider
    buffer whose rows start ``offset`` samples in and whose row stride is not a multiple of 8 samples.  ``pad`` may be
    an array: it is tiled over each row's padding."""
    import torch
    n = max(x.size for x in clips)
    width = -(-(n + offset) // 8) * 8 + (1 if offset else 0)
    buf = np.empty((len(clips), width), dtype=dtype)
    fill = np.resize(np.asarray(pad, dtype=dtype), width)
    for i, x in enumerate(clips):
        buf[i] = fill
        buf[i, offset:offset + x.size] = x
    d = torch.from_numpy(buf).cuda()[:, offset:offset + n]
    lens = torch.tensor([x.size for x in clips], dtype=torch.int64, device="cuda")
    return d, lens

"""GPU: mid-term pooling (kernel 2) and the long-term mean against float64, at the kernel and through the mid-term path.

Kernel level: mid_pool_batch on float32 [B, F, t_stride] rows that are NaN past n_frames, for window ratios and steps
around the warp width, one frame, the whole row and beyond it, zero and negative ratios (Python slices, as in the
reference).  Rows: noise, constants, 1e4 + 1e-3 noise (defeats a one-pass variance), values around -99 (silent mfcc),
cancelling signs, one row with a single NaN.  The reference is st_oracle.mid_pool of the same float32 values in float64;
every output must be within one float32 ulp of it.

Path level: the adversarial bank (tests/signals.py) through MidTermFeatures.mid_feature_extraction (host entry point)
and mid_feature_extraction_batch (device path): both bit-equal, the mid-term matrix equal to float64 pooling of the
returned short-term matrix, and within the propagated tolerance (tests/parity.check_mid_propagated) of pooling of the
oracle's short-term matrix.  The reference's own mid-term matrices at ratio 0 / -1 and the other unusual ratios of
tests/golden_cases.MID_CASES (tests/golden/mid_edges.npz) are held to the same propagated tolerance.
"""
import warnings

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests import golden_cases as EDGES
from tests.conftest import load_golden
from tests.parity import check_features, check_mid_propagated, exception_bounds, mid_slices
from tests.signals import ROW_KINDS, oracle_st, rows

pytestmark = pytest.mark.gpu

T_VALUES = [1, 2, 31, 32, 33, 65, 399, 143999]
LONG = 143999            # one hour at 50 / 25 ms
SHAPES = [(1, 1), (34, 3), (68, 1), (1, 3), (34, 1), (68, 3)]       # (F, B), taken in turn


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    pkg.ShortTermFeatures.PRINT_SPECTROGRAM_SHAPE = False
    return pkg


def pool64(st, ratio, stepr):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)         # mean of an empty slice, NaN rows
        return O.mid_pool(np.asarray(st, dtype=np.float64), ratio, stepr)


def st_batch(T, F, B, seed):
    """([B, F, T + 3] CUDA tensor, NaN past T), its [B, F, T] host values."""
    import torch
    rng = np.random.default_rng(seed)
    host = np.stack([rows(rng, F, T, b) for b in range(B)])
    buf = np.full((B, F, T + 3), np.nan, dtype=np.float32)
    buf[:, :, :T] = host
    return torch.from_numpy(buf).cuda(), host


def within_ulp(got, ref, what):
    """Every entry within one float32 ulp of the float64 value; exact zeros stay exact."""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.isfinite(got).all(), what + ": non-finite output"
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    bad = np.abs(got - ref) > ulp
    if bad.any():
        i = np.unravel_index(np.argmax(np.abs(got - ref) / ulp), ref.shape)
        raise AssertionError("%s: %d entries off by more than one float32 ulp, worst at %s: %r vs %r"
                             % (what, int(bad.sum()), i, got[i], ref[i]))


def kernel_cases(T):
    ratios = [1, 2, 31, 32, 33, 39, T, T + 7, 0, -1, -(T + 3)]
    steps = [1, 2, 39, 40, T, T + 1]
    for ratio in dict.fromkeys(ratios):
        for stepr in dict.fromkeys(steps):
            if T == LONG and stepr < 39:
                continue            # 72 000+ windows: one-hour pooling at step 40 is test_config4_at_size's
            if T == LONG and ratio >= T and stepr < T:
                continue            # every window the rest of the hour: quadratic work for both sides
            yield ratio, stepr


@pytest.mark.parametrize("T", T_VALUES)
def test_mid_pool_kernel_float64(P, T):
    from pyaudioanalysis_b200.batch import mid_pool_batch
    cache = {}
    for n, (ratio, stepr) in enumerate(kernel_cases(T)):
        F, B = SHAPES[n % len(SHAPES)]
        if (F, B) not in cache:
            cache[F, B] = st_batch(T, F, B, 1000 * T + F + B)
        st, host = cache[F, B]
        what = "T=%d ratio=%d step=%d F=%d B=%d" % (T, ratio, stepr, F, B)
        mid = mid_pool_batch(st, ratio, stepr, n_frames=T).cpu().numpy()
        win = mid_slices(T, ratio, stepr)
        assert mid.shape == (B, 2 * F, len(win)), what
        for b in range(B):
            ref = pool64(host[b], ratio, stepr)
            within_ulp(mid[b], ref, what + " clip %d" % b)
            # windows of one frame, and of a constant row, have a standard deviation of exactly 0
            for j, (a, e) in enumerate(win):
                if e - a == 1:
                    assert not mid[b, F:, j].any(), what + ": std of a one-frame window"
            const = [f for f in range(F) if (b + f) % ROW_KINDS == 1]
            assert not mid[b, [F + f for f in const]].any(), what + ": std of a constant row"
            # the NaN's windows are 0 / 0 (np.nan_to_num), every other window is finite and unaffected (within_ulp)
            for f in range(F):
                if (b + f) % ROW_KINDS == 5:
                    hit = [j for j, (a, e) in enumerate(win) if a <= T // 2 < e]
                    assert not mid[b, f, hit].any() and not mid[b, F + f, hit].any(), what + ": window holding a NaN"


@pytest.mark.parametrize("M", [1, 31, 32, 33, 3600])
def test_long_term_mean_float64(P, M):
    import torch
    from pyaudioanalysis_b200.batch import long_term_mean_batch
    rng = np.random.default_rng(M)
    B, R = 3, 136
    x = np.stack([rows(rng, R, M, b) for b in range(B)])
    x[np.isnan(x)] = 0.5
    got = long_term_mean_batch(torch.from_numpy(x).cuda()).cpu().numpy().astype(np.float64)
    ref = x.astype(np.float64).mean(axis=2)
    scale = np.abs(x.astype(np.float64)).mean(axis=2)
    bad = np.abs(got - ref) > 2.0 ** -23 * scale
    assert not bad.any(), ("M=%d: long-term means off" % M, np.argwhere(bad)[:5])
    for b in range(B):
        for r in range(R):
            if (b + r) % ROW_KINDS == 1:
                assert got[b, r] == 3.25, (M, b, r, got[b, r])


# (fs, short window, short hop, mid window, mid step): ratio, step ratio in the comment
PATH_CONFIGS = [
    (16000, 800, 400, 3200, 1600),       # 7, 4
    (44100, 882, 441, 8820, 4410),       # 19, 10
    (16000, 400, 160, 8000, 4000),       # 48.5 -> 48 (half to even), 25
    (22050, 551, 200, 4410, 2205),       # 20, 11: generic kernel
    (16000, 800, 400, 32000, 16000),     # 79, 40: one window longer than the clip
]


@pytest.mark.parametrize("fs,w,s,mw,ms", PATH_CONFIGS, ids=["%d-%d-%d-%d-%d" % c for c in PATH_CONFIGS])
def test_mid_path_on_bank(P, fs, w, s, mw, ms):
    import torch
    from pyaudioanalysis_b200._lib import get_plan
    ratio, stepr = O.mid_ratios(mw, ms, w, s)
    kind = get_plan(fs, w, s).kernel_kind()
    for name, x in SG.bank(fs, w, s).items():
        what = "fs=%d %d/%d mid %d/%d (ratio %d, step %d): %s" % (fs, w, s, mw, ms, ratio, stepr, name)
        mid, st, _ = P.MidTermFeatures.mid_feature_extraction(x, fs, mw, ms, w, s)
        dmid, dst = P.mid_feature_extraction_batch(torch.from_numpy(x).cuda()[None], fs, mw, ms, w, s)
        assert np.array_equal(mid, dmid[0].cpu().numpy()) and np.array_equal(st, dst[0].cpu().numpy()), \
            what + ": host entry point and device path differ"
        within_ulp(mid, pool64(st, ratio, stepr), what + ", pooling of the returned short-term matrix")
        ref = oracle_st(x, fs, w, s)
        allow = exception_bounds(name, kind)
        check_features(st, ref, w // 2, what, allow=allow)
        check_mid_propagated(mid, st, ref, ratio, stepr, w // 2, what, allow=allow)


@pytest.mark.parametrize("signal", EDGES.SIGNALS)
def test_mid_edges_against_reference(P, signal):
    """Ratio 0 and -1, the half-to-even ties, a window longer than the clip, a step above the window: the reference's own
    mid-term matrices (tests/golden/mid_edges.npz)."""
    g = load_golden("mid_edges.npz")
    x = EDGES.clip(signal)
    fs, w, s = EDGES.FS, EDGES.W, EDGES.S
    ref_st = oracle_st(x, fs, w, s)
    for name, (mw, ms, ratio, stepr) in EDGES.MID_CASES.items():
        what = "%s, %s" % (signal, name)
        mid, st, _ = P.MidTermFeatures.mid_feature_extraction(x, fs, mw, ms, w, s)
        ref = g[EDGES.mid_key(signal, name, "mid")]
        assert mid.shape == ref.shape, what
        check_mid_propagated(mid, st, ref_st, ratio, stepr, w // 2, what, ref_mid=ref)
        if ratio <= 0:
            assert not mid[:, 1:].any(), what

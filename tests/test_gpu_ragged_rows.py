"""GPU: ragged spectrogram / chromagram batches (spectrogram_batch / chromagram_batch with lengths=, row_counts) and the
kernel that transforms every clipped chromagram frame of a batch in one launch.

The adversarial bank, uncut, runs as one ragged batch through every row kernel kind a plan reaches, against the oracle
and bit for bit against each clip alone through the equal-length entry points; padding values and an odd-offset view do
not change a bit.  Lengths around every edge of the row arithmetic (csrc/rows.cuh) check the per-clip row counts, which
rows the C ABI writes, and the refusals.  A ragged chromagram is the row kernel plus one clipped-frame launch however
many clipped lengths it holds, and a 1 s window's clipped frames (large-window form of the kernel) match the oracle.
"""
import ctypes

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import PAIR, KIND_NAMES, plans, ragged
from tests.parity import check_close, check_spectrogram_rows
from tests.test_gpu_adversarial import ROW_CONFIGS

pytestmark = pytest.mark.gpu

CONFIGS = ROW_CONFIGS + [(16000, 800, 200)]
ODD = 3


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


def bits(t):
    return np.ascontiguousarray(t.cpu().numpy(), dtype=np.float32).view(np.uint32)


def alone(P, fn, x, fs, w, s, pl):
    import torch
    return fn(torch.from_numpy(np.ascontiguousarray(x)).cuda()[None], fs, w, s, plan=pl)[0]


def oracle_chromagram(x, fs, w, s):
    """The oracle's chromagram, None where the single-clip entry point refuses the clip (the oracle raises for a clipped
    frame shorter than K; a clip shorter than w + s is refused as well)."""
    if len(x) - s - w < 0:
        return None
    try:
        return O.chromagram(x, fs, w, s)[0]
    except ValueError:
        return None


@pytest.mark.parametrize("fs,w,s", CONFIGS, ids=["%d-%d-%d" % c for c in CONFIGS])
def test_bank_ragged_every_kernel(P, fs, w, s):
    import torch
    ints = SG.bank(fs, w, s)
    flts = SG.float_bank(fs, w, s)
    names, clips = list(ints), list(ints.values())
    fclips = list(flts.values())
    d, lens = ragged(clips, np.int16)
    dodd, _ = ragged(clips, np.int16, offset=ODD)
    drail, _ = ragged(clips, np.int16, pad=[32767, -32768])
    df, flens = ragged(fclips, np.float32)
    dfnan, _ = ragged(fclips, np.float32, pad=np.nan)
    rs = P.row_counts(lens, w, s, 0).cpu().tolist()
    rc = P.row_counts(lens, w, s, 1).cpu().tolist()
    frs, frc = P.row_counts(flens, w, s, 0).cpu().tolist(), P.row_counts(flens, w, s, 1).cpu().tolist()
    sp_ref = [O.spectrogram(x, fs, w, s)[0] for x in clips]
    ch_ref = [oracle_chromagram(x, fs, w, s) for x in clips]
    fch_ref = [oracle_chromagram(x.astype(np.float64), fs, w, s) for x in fclips]
    for kind, pl in plans(fs, w, s):
        if kind == PAIR:
            continue                      # the pair kernel has no row mode: the CTA kernel serves these rows
        tag = "%s rows, fs=%d w=%d s=%d" % (KIND_NAMES[kind], fs, w, s)
        sp = P.spectrogram_batch(d, fs, w, s, plan=pl, lengths=lens)
        ch = P.chromagram_batch(d, fs, w, s, plan=pl, lengths=lens)
        for i, name in enumerate(names):
            what = "%s: %s" % (tag, name)
            assert rs[i] == sp_ref[i].shape[0], what
            check_spectrogram_rows(sp[i, :rs[i]].cpu().numpy(), clips[i], w, s, "spectrogram " + what)
            assert not sp[i, rs[i]:].any() and not ch[i, rc[i]:].any(), what + ": rows past the clip's own"
            assert np.array_equal(bits(alone(P, P.spectrogram_batch, clips[i], fs, w, s, pl)), bits(sp[i, :rs[i]])), \
                "spectrogram " + what + ": differs from the clip alone"
            if ch_ref[i] is None:
                assert rc[i] == 0, what
                with pytest.raises(ValueError):
                    alone(P, P.chromagram_batch, clips[i], fs, w, s, pl)
                continue
            assert rc[i] == ch_ref[i].shape[0], what
            check_close(ch[i, :rc[i]].cpu().numpy(), ch_ref[i], "chromagram " + what, atol=1e-6)
            assert np.array_equal(bits(alone(P, P.chromagram_batch, clips[i], fs, w, s, pl)), bits(ch[i, :rc[i]])), \
                "chromagram " + what + ": differs from the clip alone"
        for view, label in ((dodd, "odd-offset view"), (drail, "rail padding")):
            assert torch.equal(P.spectrogram_batch(view, fs, w, s, plan=pl, lengths=lens), sp), "%s: %s" % (tag, label)
            assert torch.equal(P.chromagram_batch(view, fs, w, s, plan=pl, lengths=lens), ch), "%s: %s" % (tag, label)
        fsp = P.spectrogram_batch(df, fs, w, s, plan=pl, lengths=flens)
        fch = P.chromagram_batch(df, fs, w, s, plan=pl, lengths=flens)
        for i, name in enumerate(flts):
            what = "%s: %s" % (tag, name)
            assert frs[i] == int((fclips[i].size - w) / s) + 1, what
            check_spectrogram_rows(fsp[i, :frs[i]].cpu().numpy(), fclips[i], w, s, "spectrogram " + what)
            if fch_ref[i] is None:
                assert frc[i] == 0 and not fch[i].any(), what
            else:
                check_close(fch[i, :frc[i]].cpu().numpy(), fch_ref[i], "chromagram " + what, atol=1e-6)
        assert torch.equal(P.spectrogram_batch(dfnan, fs, w, s, plan=pl, lengths=flens), fsp), tag + ": NaN padding"
        assert torch.equal(P.chromagram_batch(dfnan, fs, w, s, plan=pl, lengths=flens), fch), tag + ": NaN padding"


def clipped_lengths(n, w, s):
    """Lengths of the clipped frames of chromagram()'s loop over n samples (ShortTermFeatures.py:349-355)."""
    return [n - p for p in range(w, n - s, s) if p + w > n]


def edge_lengths(w, s):
    """Lengths at and around w - s, w, w + s (len - s - w = 0), 2w, and clips with 0, 1, 2 and 3 clipped frames."""
    out = set()
    for e in (w - s, w, w + s, 2 * w):
        out.update(e + d for d in (-2, -1, 0, 1, 2) if e + d >= 0)
    by_count = {}
    for n in range(2 * w, 6 * w):
        by_count.setdefault(len(clipped_lengths(n, w, s)), []).append(n)
    for c in (0, 1, 2, 3):
        picks = by_count.get(c, [])
        out.update(picks[:: max(1, len(picks) // 3)][:3])
    return sorted(out)


@pytest.mark.parametrize("fs,w,s", [(16000, 800, 200), (16000, 800, 333), (16000, 800, 400), (44100, 882, 441), (16000, 400, 160)])
def test_edge_lengths(P, fs, w, s):
    import torch
    from pyaudioanalysis_b200._lib import lib, get_plan
    lengths = edge_lengths(w, s)
    rng = np.random.default_rng(w * 7 + s)
    clips = [rng.normal(0, 3000, n).round().astype(np.int16) for n in lengths]
    d, lens = ragged(clips, np.int16)
    B, N = d.shape
    norm = P.clip_stats(d, lens)
    pl = get_plan(fs, w, s)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for which, fn, rows_of, width, entry in ((0, P.spectrogram_batch, lib().b200aa_spectrogram_rows, w // 2, lib().b200aa_spectrogram_ragged),
                                             (1, P.chromagram_batch, lib().b200aa_chromagram_rows, 12, lib().b200aa_chromagram_ragged)):
        counts = P.row_counts(lens, w, s, which).cpu().tolist()
        R = rows_of(N, w, s)
        raw = torch.full((B, R, width), float("nan"), device="cuda")
        assert entry(pl.handle, ctypes.c_void_p(d.data_ptr()), 0, B, N, d.stride(0), ctypes.c_void_p(lens.data_ptr()),
                     ctypes.c_void_p(norm.data_ptr()), ctypes.c_void_p(raw.data_ptr()), stream) == 0
        seen = set()
        for i, n in enumerate(lengths):
            what = "%s, w=%d s=%d, clip of %d samples (clipped frames %s)" % (["spectrogram", "chromagram"][which], w, s, n,
                                                                              clipped_lengths(n, w, s))
            try:
                ref = alone(P, fn, clips[i], fs, w, s, pl)
            except ValueError:
                ref = None
            if ref is None:
                assert counts[i] == 0, what + ": a refused clip counts 0 rows"
                assert torch.isnan(raw[i]).all(), what + ": a refused clip gets nothing written"
                seen.add("refused")
                continue
            assert counts[i] == rows_of(n, w, s) == ref.shape[0] >= 1, what
            assert not torch.isnan(raw[i, :counts[i]]).any() and torch.isnan(raw[i, counts[i]:]).all(), what + ": rows written"
            assert np.array_equal(bits(raw[i, :counts[i]]), bits(ref)), what + ": differs from the clip alone"
            seen.add(len(clipped_lengths(n, w, s)) if which else "ok")
        assert "refused" in seen


def test_one_clipped_launch_for_any_number_of_clipped_lengths(P):
    import torch
    from pyaudioanalysis_b200._lib import lib
    fs, w, s = 16000, 800, 400             # one clipped frame of any length in [K, w) per clip
    K = w // 2
    firsts = {}
    for n in range(2 * w, 8 * w):
        cl = clipped_lengths(n, w, s)
        if cl and min(cl) >= K:
            firsts.setdefault(cl[0], n)
    assert len(firsts) >= 200

    def launches(ns):
        rng = np.random.default_rng(len(ns))
        d, lens = ragged([rng.normal(0, 3000, n).round().astype(np.int16) for n in ns], np.int16)
        norm = P.clip_stats(d, lens)
        torch.cuda.synchronize()
        c0 = lib().b200aa_launch_count()
        out = P.chromagram_batch(d, fs, w, s, norm=norm, lengths=lens)
        c1 = lib().b200aa_launch_count()
        for i, n in enumerate(ns[:3]):
            check_close(out[i, :lib().b200aa_chromagram_rows(n, w, s)].cpu().numpy(), O.chromagram(d[i, :n].cpu().numpy(), fs, w, s)[0],
                        "clip of %d samples" % n, atol=1e-6)
        return c1 - c0
    ns = list(firsts.values())
    assert launches(ns[:2]) == launches(ns[:200]) == 2, "the row kernel plus one clipped-frame launch"


def test_large_window_clipped_frames(P):
    import torch
    fs, w, s = 16000, 16000, 8000
    lengths = [45000, 41000, 50500, 39000, 47999]
    rng = np.random.default_rng(5)
    clips = [rng.normal(0, 3000, n).round().astype(np.int16) for n in lengths]
    assert all(clipped_lengths(n, w, s) for n in lengths)
    d, lens = ragged(clips, np.int16)
    ch = P.chromagram_batch(d, fs, w, s, lengths=lens)
    counts = P.row_counts(lens, w, s, 1).cpu().tolist()
    for i, n in enumerate(lengths):
        ref = O.chromagram(clips[i], fs, w, s)[0]
        assert counts[i] == ref.shape[0]
        check_close(ch[i, :counts[i]].cpu().numpy(), ref, "1 s window, clip of %d samples" % n, atol=1e-6)
        one = P.chromagram_batch(torch.from_numpy(clips[i]).cuda()[None], fs, w, s)[0]
        assert torch.equal(one, ch[i, :counts[i]]), "clip of %d samples differs from the clip alone" % n

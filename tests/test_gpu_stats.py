"""GPU: kernel 0's clip record against exact arithmetic, no kernel reading past a clip's length, and the output
contract of the batched entry points.

Every feature kernel starts from the 32-byte record b200aa_clip_norm (include/b200aa.h), read here as float32[B, 8] =
(a, bp, m, lo, hi, 0, 0, 0).  The features are nearly scale invariant, so a wrong a or bp mostly cancels in them; this
module holds the record itself to values computed on the host from the exact clip sum (int64 sums for int16,
math.fsum for float32), and checks what the record is for: lo / hi classify every sample's x - m exactly as
sign(x - mean), and a (x - m) + bp equals the reference's x / 2^15 + dc_normalize to float32 resolution.

Ragged batches are padded with poison past each length (int16: alternating rails, float32: NaN): records must equal
those of each clip alone, and every feature kernel must give what it gives on the zero-padded batch.

The output contract: feature_extraction_batch writes exactly the columns below each clip's own frame count of an ``out``
wider than T (odd row stride), and nothing else; spectrogram_batch writes every element of ``out``.
"""
import math

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import KIND_NAMES, plans, ragged
from tests.parity import check_features

pytestmark = pytest.mark.gpu

LENGTHS = [0, 1, 7, 8, 9, 31, 33, 4095, 4097, 32767, 32769, 160000]
ODD_LENGTH = 160001          # per = ceil(L / chunks) is odd: chunk starts fall off the 16-byte boundary
RAILS = np.array([32767, -32768], dtype=np.int16)
A_EMPTY = np.float32(1.0 / (32768.0 * 1e-10))      # a of a clip without samples (max deviation 0)


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


def with_sum(x, target):
    """x (int64) with its last samples moved so that its sum is exactly ``target``."""
    x = x.copy()
    r = int(x.sum() - target)
    k = max(1, min(x.size, -(-abs(r) // 1000)))
    x[x.size - k:] -= r // k
    x[-1] -= int(x.sum() - target)
    assert x.sum() == target and np.abs(x).max() < 32767
    return x


def i16_clips():
    """Clips of every length of LENGTHS (non-integer means of both signs), rails, an integer mean, a k + 1/2 mean."""
    rng = np.random.default_rng(4242)
    out = {}
    for i, L in enumerate(LENGTHS):
        out["len%d" % L] = (rng.integers(-3000, 3001, L) + (-1) ** i * (137 * i + 0.3 * L) % 1000).astype(np.int16)
    out["all_min"] = np.full(999, -32768, dtype=np.int16)
    out["all_max"] = np.full(1001, 32767, dtype=np.int16)
    out["alt_rails"] = np.resize(RAILS, 2000)                         # mean exactly -1/2
    out["int_mean"] = SG.integer_mean(rng, 3001, m=-23)
    out["half_mean"] = with_sum(np.round(12 + rng.normal(0, 300, 1000)).astype(np.int64), 12 * 1000 + 500).astype(np.int16)
    return out


def f32_clips():
    rng = np.random.default_rng(4343)
    out = {}
    for i, L in enumerate(LENGTHS):
        out["len%d" % L] = (rng.normal(0, 3000, L) * 0.37 + 11.5 - 7 * i).astype(np.float32)
    tiny = np.array([0.0, -0.0, 1e-45, -1e-45, 3e-40, -7e-41, 1.1754942e-38, -0.0], dtype=np.float32)
    out["zeros_subnormals"] = np.resize(tiny, 1003)
    big = (rng.normal(0, 1.0, 2049)).astype(np.float32)
    big[700] = 1e30
    out["plus_1e30"] = big
    neg = (rng.normal(0, 1.0, 1537)).astype(np.float32)
    neg[3] = -1e30
    out["minus_1e30"] = neg
    return out


# ---------------------------------------------------------------------------------------------------- record checks
def check_i16_records(rec, sums, lens, mins, maxs, what):
    """Vectorised over clips: rec float32 [B, 8]; exact int64 sums, lengths, minima and maxima of every clip."""
    rec = np.asarray(rec)
    S, L = np.asarray(sums, np.int64), np.asarray(lens, np.int64)
    a, bp, m, lo, hi = (rec[:, k].astype(np.float64) for k in range(5))
    assert not rec[:, 5:].any(), what + ": reserved words not cleared"
    e = L == 0
    assert (rec[e, 0] == A_EMPTY).all() and not rec[e, 1:5].any(), what + ": record of an empty clip"
    v = ~e
    S, L, a, bp, m, lo, hi = S[v], L[v], a[v], bp[v], m[v], lo[v], hi[v]
    mn, mx = np.asarray(mins, np.float64)[v], np.asarray(maxs, np.float64)[v]
    assert (m == np.round(m)).all(), what + ": m is not an integer"
    mi = m.astype(np.int64)
    bad = 2 * np.abs(mi * L - S) > L
    assert not bad.any(), "%s: |m - mean| > 1/2 for clips %s" % (what, np.nonzero(v)[0][bad][:8])
    fl, ce = S // L, -((-S) // L)
    bad = (lo != fl - mi) | (hi != ce - mi)
    assert not bad.any(), "%s: lo / hi are not floor / ceil(mean) - m for clips %s" % (what, np.nonzero(v)[0][bad][:8])
    mean = S / L
    ra = 1.0 / (np.maximum(mx - mean, mean - mn) + 32768.0 * 1e-10)
    bad = np.abs(a - ra) > np.spacing(ra.astype(np.float32)).astype(np.float64)
    assert not bad.any(), "%s: a off by more than one float32 ulp for clips %s" % (what, np.nonzero(v)[0][bad][:8])
    rbp = ra * (mi * L - S) / L
    bad = np.abs(bp - rbp) > 2.0 ** -24 * np.abs(rbp) + ra * 2.0 ** -50 * np.abs(mean)
    assert not bad.any(), "%s: bp is not a (m - mean) for clips %s" % (what, np.nonzero(v)[0][bad][:8])


def check_i16_clip(rec, x, what):
    """One int16 clip: the record, then lo / hi and a, bp against every sample."""
    x64 = x.astype(np.int64)
    L = x.size
    check_i16_records(rec[None], [x64.sum()], [L], [x64.min() if L else 0], [x64.max() if L else 0], what)
    if L:
        check_samples(rec, x, np.sign(x64 * L - x64.sum()), what)


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


def stats(P, d, lens=None):
    import torch
    return P.clip_stats(d, lens).view(torch.float32).cpu().numpy()


# ---------------------------------------------------------------------------------------------------- record tests
def test_int16_records_exact(P):
    import torch
    clips = i16_clips()
    for name, x in clips.items():
        if x.size:              # the empty clip is in the batches below (an empty tensor has no device address)
            check_i16_clip(stats(P, torch.from_numpy(x).cuda()[None])[0], x, "int16 %s alone" % name)
    x = np.resize(np.arange(-5000, 5000, 7, dtype=np.int16), ODD_LENGTH)
    check_i16_clip(stats(P, torch.from_numpy(x).cuda()[None])[0], x, "int16 length %d" % ODD_LENGTH)
    # views at sample offsets 1..7 with row strides that are not multiples of 8: scalar loads, unaligned chunk starts
    some = [clips[k] for k in ("len4097", "len33", "len32769", "half_mean", "alt_rails")]
    for off in range(1, 8):
        d, lens = ragged(some, np.int16, offset=off, pad=RAILS)
        assert d.stride(0) % 8 != 0
        rec = stats(P, d, lens)
        for i, x in enumerate(some):
            check_i16_clip(rec[i], x, "int16 view at offset %d, clip %d" % (off, i))


def test_float32_records_exact(P):
    import torch
    for name, x in f32_clips().items():
        if x.size:
            check_f32_clip(stats(P, torch.from_numpy(x).cuda()[None])[0], x, "float32 %s alone" % name)
    x = (np.arange(ODD_LENGTH) % 1013).astype(np.float32) * np.float32(0.37)
    check_f32_clip(stats(P, torch.from_numpy(x).cuda()[None])[0], x, "float32 length %d" % ODD_LENGTH)
    some = list(f32_clips().values())[6:]
    for off in (1, 3, 6):
        d, lens = ragged(some, np.float32, offset=off, pad=np.nan)
        rec = stats(P, d, lens)
        for i, x in enumerate(some):
            check_f32_clip(rec[i], x, "float32 view at offset %d, clip %d" % (off, i))


def test_poisoned_padding_records(P):
    """Ragged batches with poison past every length: the same records as each clip alone (int16: bit for bit)."""
    import torch
    clips = list(i16_clips().values())
    d, lens = ragged(clips, np.int16, pad=RAILS)
    rec = stats(P, d, lens)
    for i, x in enumerate(clips):
        check_i16_clip(rec[i], x, "int16 poisoned batch, clip %d" % i)
        if x.size:
            alone = stats(P, torch.from_numpy(x).cuda()[None])[0]
            assert np.array_equal(alone.view(np.int32), rec[i].view(np.int32)), "int16 clip %d: batch record differs from alone" % i
    fclips = list(f32_clips().values())
    d, lens = ragged(fclips, np.float32, pad=np.nan)
    rec = stats(P, d, lens)
    for i, x in enumerate(fclips):
        check_f32_clip(rec[i], x, "float32 NaN-padded batch, clip %d" % i)


def test_grid_y_split(P):
    """40 000 clips: more than one launch along the grid's y dimension (32 768 clips each)."""
    import torch
    rng = np.random.default_rng(31)
    B, N = 40000, 64
    x = rng.integers(-20000, 20001, (B, N)).astype(np.int16)
    x += (np.arange(B) % 997).astype(np.int16)[:, None]
    L = rng.integers(1, N + 1, B)
    L[[0, 32767, 32768, 39999]] = (N, 1, 37, N)
    valid = np.arange(N)[None, :] < L[:, None]
    xp = np.where(valid, x, RAILS[np.arange(N) % 2][None, :]).astype(np.int16)
    rec = stats(P, torch.from_numpy(xp).cuda(), torch.from_numpy(L).cuda())
    x64 = x.astype(np.int64)
    S = np.where(valid, x64, 0).sum(axis=1)
    mn = np.where(valid, x64, 1 << 20).min(axis=1)
    mx = np.where(valid, x64, -(1 << 20)).max(axis=1)
    check_i16_records(rec, S, L, mn, mx, "40 000 clips")
    for b in (0, 32767, 32768, 39999):
        check_i16_clip(rec[b], x[b, :L[b]], "40 000 clips, clip %d" % b)


# ---------------------------------------------------------------------------------------------------- feature kernels
POISON_CONFIGS = [(16000, 800, 400), (44100, 882, 441), (16000, 400, 160), (16000, 1024, 300), (22050, 551, 200)]


@pytest.mark.parametrize("fs,w,s", POISON_CONFIGS, ids=["%d-%d-%d" % c for c in POISON_CONFIGS])
def test_no_kernel_reads_past_a_clip(P, fs, w, s):
    """The bank as a ragged batch padded with poison: every kernel kind gives what it gives on the zero-padded batch
    (int16: bit for bit; float32 NaN padding: bit for bit with the zero-padded batch's records, finite and within the
    tolerance with its own)."""
    import torch
    clips = list(SG.bank(fs, w, s).values())
    fclips = list(SG.float_bank(fs, w, s).values())
    d0, lens = ragged(clips, np.int16)
    dp, _ = ragged(clips, np.int16, pad=RAILS)
    f0, flens = ragged(fclips, np.float32)
    fp, _ = ragged(fclips, np.float32, pad=np.nan)
    fnorm = P.clip_stats(f0, flens)
    T = [O.frame_count(x.size, w, s) for x in fclips]
    for kind, pl in plans(fs, w, s):
        tag = "%s kernel, fs=%d w=%d s=%d" % (KIND_NAMES[kind], fs, w, s)
        ref = P.feature_extraction_batch(d0, fs, w, s, lengths=lens, plan=pl)
        got = P.feature_extraction_batch(dp, fs, w, s, lengths=lens, plan=pl)
        assert torch.equal(got, ref), tag + ": int16 output depends on the samples past a clip's length"
        fref = P.feature_extraction_batch(f0, fs, w, s, lengths=flens, plan=pl, norm=fnorm)
        fgot = P.feature_extraction_batch(fp, fs, w, s, lengths=flens, plan=pl, norm=fnorm)
        assert torch.equal(fgot, fref), tag + ": float32 output depends on the samples past a clip's length"
        own = P.feature_extraction_batch(fp, fs, w, s, lengths=flens, plan=pl).cpu().numpy()
        assert np.isfinite(own).all(), tag + ": NaN padding reached the float32 output"
        fr = fref.cpu().numpy()
        for i in range(len(fclips)):
            check_features(own[i, :, :T[i]], fr[i, :, :T[i]], w // 2, "%s: NaN-padded float32 clip %d" % (tag, i))


# ---------------------------------------------------------------------------------------------------- output contract
CONTRACT_CONFIGS = [(16000, 800, 400), (44100, 882, 441), (22050, 551, 200)]
NAN_BITS = np.array([np.nan], dtype=np.float32).view(np.int32)[0]


@pytest.mark.parametrize("fs,w,s", CONTRACT_CONFIGS, ids=["%d-%d-%d" % c for c in CONTRACT_CONFIGS])
def test_output_contract(P, fs, w, s):
    """``out`` prefilled with NaN, [B, F, T + 5] (an odd row stride); the batch is ragged and holds a clip of no samples
    and one of window - 1 samples between full ones.  Every kernel kind, deltas on and off: columns below a clip's frame
    count are finite and bit-equal to the default call, every other element keeps its NaN bit pattern.  A record passed
    as ``norm=`` gives the same bits."""
    import torch
    clips = list(SG.bank(fs, w, s).values())
    clips = clips[:3] + [np.zeros(0, np.int16), clips[3][:w - 1]] + clips[3:]
    d, lens = ragged(clips, np.int16, pad=RAILS)
    Tc = [O.frame_count(x.size, w, s) for x in clips]
    assert Tc[3] == Tc[4] == 0
    T = O.frame_count(d.shape[1], w, s)
    norm = P.clip_stats(d, lens)
    for kind, pl in plans(fs, w, s):
        for deltas in (True, False):
            tag = "%s kernel, fs=%d w=%d s=%d, deltas %s" % (KIND_NAMES[kind], fs, w, s, deltas)
            F = 68 if deltas else 34
            ref = P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl, deltas=deltas)
            assert ref.shape == (len(clips), F, T)
            out = torch.full((len(clips), F, T + 5), float("nan"), device="cuda")
            got = P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl, deltas=deltas, out=out)
            assert got.data_ptr() == out.data_ptr()
            bits = got.view(torch.int32).cpu().numpy()
            g, r = got.cpu().numpy(), ref.cpu().numpy()
            for i, t in enumerate(Tc):
                assert np.isfinite(g[i, :, :t]).all(), "%s: clip %d has non-finite frames" % (tag, i)
                assert np.array_equal(g[i, :, :t].view(np.int32), r[i, :, :t].view(np.int32)), "%s: clip %d differs from the default call" % (tag, i)
                rest = bits[i, :, t:]
                assert (rest == NAN_BITS).all(), "%s: clip %d wrote %d elements at or past its frame count %d (first column %d)" % (
                    tag, i, int((rest != NAN_BITS).sum()), t, t + int(np.nonzero((rest != NAN_BITS).any(axis=0))[0][0]))
            again = P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl, deltas=deltas, norm=norm)
            assert torch.equal(again, ref), tag + ": norm= record gives other bits"


@pytest.mark.parametrize("fs,w,s", CONTRACT_CONFIGS[:2], ids=["%d-%d-%d" % c for c in CONTRACT_CONFIGS[:2]])
def test_spectrogram_writes_every_element(P, fs, w, s):
    """spectrogram_batch(out=...) into a NaN-filled tensor writes every element, the reference's zero rows included."""
    import torch
    bank = SG.bank(fs, w, s)
    n = min(x.size for x in bank.values())
    d = torch.from_numpy(np.stack([x[:n] for x in bank.values()])).cuda()
    for kind, pl in plans(fs, w, s):
        ref = P.spectrogram_batch(d, fs, w, s, plan=pl)
        out = torch.full(tuple(ref.shape), float("nan"), device="cuda")
        got = P.spectrogram_batch(d, fs, w, s, plan=pl, out=out)
        assert torch.isfinite(got).all(), "%s kernel: spectrogram left %d elements unwritten" % (KIND_NAMES[kind], int((~torch.isfinite(got)).sum()))
        assert torch.equal(got, ref), "%s kernel: spectrogram into out= differs" % KIND_NAMES[kind]
